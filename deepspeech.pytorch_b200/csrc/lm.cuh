// ARPA n-gram language model on the device (row N6): the layout of the buffer that ds2_lm_build (csrc/lm.cu)
// writes and the lookups that the beam search (csrc/beam_decode.cu, rule L2) makes in it.  This header is the one
// place the layout is defined; lm.cu fills it, beam_decode.cu reads it.
//
// Buffer (every part 256-byte aligned, offsets in the header):
//   LmHeader
//   slots   int32[S]      open-addressed hash, S = power of two >= 2 E; 0 = empty, else entry index + 1
//   keys    ulonglong2[E] the exact 128-bit key of each n-gram: order in bits 120..122, then up to five 24-bit word ids
//   vals    float2[E]     (log10 p, log10 backoff) as the ARPA file writes them, parsed to fp32; an unwritten backoff
//                         is 0
//   mask    uint64[NT]    vocabulary trie: child mask over labels,
//   first   int32[NT]       index of the first child (children are contiguous, in label order),
//   word    int32[NT]       word id of the node's prefix, -1 if the prefix is not a word of V
// A key holds every word id of its n-gram, so a lookup compares whole keys: a hash collision costs a probe, never a
// wrong value.  The slot claims are atomicCAS in any order; with distinct keys and linear probing without deletion, a
// lookup finds the key's own entry or an empty slot whatever the insertion order was, so its result does not depend
// on that order.
#pragma once
#include <stdint.h>

namespace ds2 {

constexpr int LM_MAX_ORDER = 5;
constexpr int LM_MAX_WORDS = 1 << 24;
constexpr unsigned LM_MAGIC = 0x364e4c44u;
// lm value of a word outside the ARPA vocabulary (rule L2), before alpha multiplies it
constexpr double LM_OOV = -1000.0;
// factor from the ARPA's log10 values to the lm value of rule L2.  1: the log10 value is used unconverted, which is
// how we read ctcdecode's get_log_cond_prob; that reading is not verifiable here.  If ctcdecode converts to natural
// log, this is ln 10 = 2.302585092994046 (and LM_SCALE in oracle/lm_oracle.py with it).
constexpr double LM_SCALE = 1.0;

struct LmHeader {
  unsigned magic;
  int order, n_words, bos;
  long long n_entries, n_slots, n_nodes;
  long long off_slots, off_keys, off_vals, off_mask, off_first, off_word, bytes;
};

struct LmView {
  const int* slots;
  const ulonglong2* keys;
  const float2* vals;
  const unsigned long long* mask;
  const int* first;
  const int* word;
  unsigned long long slot_mask;
  int bos;
};

__host__ __device__ __forceinline__ ulonglong2 lm_key(int n, const int* ids) {
  unsigned long long w[LM_MAX_ORDER] = {0ull, 0ull, 0ull, 0ull, 0ull};
  for (int k = 0; k < n; ++k) w[k] = (unsigned long long)(unsigned)ids[k];
  ulonglong2 key;
  key.x = w[0] | (w[1] << 24) | ((w[2] & 0xffffull) << 48);
  key.y = (w[2] >> 16) | (w[3] << 8) | (w[4] << 32) | ((unsigned long long)n << 56);
  return key;
}

__host__ __device__ __forceinline__ unsigned long long lm_hash(ulonglong2 k) {
  unsigned long long h = k.x ^ (k.y * 0x9e3779b97f4a7c15ull);
  h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
  return h;
}

#ifdef __CUDACC__
__device__ __forceinline__ LmView lm_view(const void* buf) {
  const LmHeader* h = static_cast<const LmHeader*>(buf);
  const char* b = static_cast<const char*>(buf);
  LmView v;
  v.slots = reinterpret_cast<const int*>(b + h->off_slots);
  v.keys = reinterpret_cast<const ulonglong2*>(b + h->off_keys);
  v.vals = reinterpret_cast<const float2*>(b + h->off_vals);
  v.mask = reinterpret_cast<const unsigned long long*>(b + h->off_mask);
  v.first = reinterpret_cast<const int*>(b + h->off_first);
  v.word = reinterpret_cast<const int*>(b + h->off_word);
  v.slot_mask = (unsigned long long)h->n_slots - 1ull;
  v.bos = h->bos;
  return v;
}

// entry index of the n-gram `ids` (n words, oldest first), or -1
__device__ __forceinline__ int lm_find(const LmView& v, int n, const int* ids) {
  const ulonglong2 key = lm_key(n, ids);
  unsigned long long s = lm_hash(key) & v.slot_mask;
  for (;;) {
    const int e = v.slots[s];
    if (e == 0) return -1;
    const ulonglong2 k = v.keys[e - 1];
    if (k.x == key.x && k.y == key.y) return e - 1;
    s = (s + 1) & v.slot_mask;
  }
}

// rule L2: lm(w | ctx) for an order-N model, ctx = the N-1 context word ids, oldest first (<s>-padded).  The longest
// listed n-gram ending in w, plus the backoffs of the longer contexts, summed in fp64 from the longest context down.
__device__ __forceinline__ double lm_logp(const LmView& v, int N, const int* ctx, int w) {
  int ids[LM_MAX_ORDER];
  double acc = 0.0;
  for (int n = N; n >= 1; --n) {
    for (int k = 0; k < n - 1; ++k) ids[k] = ctx[N - n + k];
    ids[n - 1] = w;
    const int e = lm_find(v, n, ids);
    if (e >= 0) return __dmul_rn(LM_SCALE, __dadd_rn(acc, (double)v.vals[e].x));
    if (n > 1) {
      const int eb = lm_find(v, n - 1, ids);          // the context as an (n-1)-gram: its backoff, 0 if unlisted
      if (eb >= 0) acc = __dadd_rn(acc, (double)v.vals[eb].y);
    }
  }
  return LM_OOV;
}
#endif

}  // namespace ds2
