// ds2_lm_bytes / ds2_lm_build (row N6): the ARPA n-gram tables and the vocabulary trie of a language model, written
// into a caller buffer in the layout of lm.cuh for ds2_beam_decode_lm.

#include "common.cuh"
#include "lm.cuh"

namespace ds2 {

namespace {

constexpr int LM_THREADS = 256;

bool lm_layout(int order, const int64_t* counts, int64_t n_nodes, LmHeader* h) {
  if (order < 1 || order > LM_MAX_ORDER || !counts || n_nodes < 1) return false;
  long long E = 0;
  for (int n = 0; n < order; ++n) {
    if (counts[n] < 0) return false;
    E += counts[n];
  }
  long long S = 2;
  while (S < 2 * E) S <<= 1;
  memset(h, 0, sizeof(*h));
  h->magic = LM_MAGIC;
  h->order = order;
  h->n_entries = E;
  h->n_slots = S;
  h->n_nodes = n_nodes;
  size_t off = align_up(sizeof(LmHeader), 256);
  h->off_slots = (long long)off;  off += align_up((size_t)S * 4, 256);
  h->off_keys = (long long)off;   off += align_up((size_t)E * 16, 256);
  h->off_vals = (long long)off;   off += align_up((size_t)E * 8, 256);
  h->off_mask = (long long)off;   off += align_up((size_t)n_nodes * 8, 256);
  h->off_first = (long long)off;  off += align_up((size_t)n_nodes * 4, 256);
  h->off_word = (long long)off;   off += align_up((size_t)n_nodes * 4, 256);
  h->bytes = (long long)off;
  return true;
}

__global__ void lm_header_kernel(LmHeader h, LmHeader* out) { *out = h; }

__global__ void __launch_bounds__(LM_THREADS)
lm_insert_kernel(int n, long long count, long long base, const int32_t* __restrict__ ids,
                 const float* __restrict__ logp, const float* __restrict__ bo, int* slots, ulonglong2* keys,
                 float2* vals, unsigned long long slot_mask) {
  const long long r = (long long)blockIdx.x * LM_THREADS + threadIdx.x;
  if (r >= count) return;
  const ulonglong2 key = lm_key(n, ids + r * n);
  const long long e = base + r;
  keys[e] = key;
  vals[e] = make_float2(logp[r], bo ? bo[r] : 0.f);
  unsigned long long s = lm_hash(key) & slot_mask;
  while (atomicCAS(&slots[s], 0, (int)(e + 1)) != 0) s = (s + 1) & slot_mask;
}

}  // namespace
}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_lm_bytes(int order, const int64_t* counts, int64_t n_nodes) {
  LmHeader h;
  if (!lm_layout(order, counts, n_nodes, &h)) return 0;
  return (size_t)h.bytes;
}

int ds2_lm_build(int order, const int64_t* counts, const int32_t* const* ids, const float* const* logp,
                 const float* const* backoff, int n_words, int bos, int64_t n_nodes, const uint64_t* trie_mask,
                 const int32_t* trie_first, const int32_t* trie_word, void* buffer, size_t buffer_bytes,
                 void* stream) {
  LmHeader h;
  DS2_REQUIRE(lm_layout(order, counts, n_nodes, &h), "ds2_lm_build: bad order=%d (1..%d), counts or n_nodes", order,
              LM_MAX_ORDER);
  DS2_REQUIRE(n_words >= 1 && n_words < LM_MAX_WORDS && counts[0] == n_words,
              "ds2_lm_build: n_words=%d must equal the unigram count and be < 2^24", n_words);
  DS2_REQUIRE(h.n_entries < (1ll << 31) - 1, "ds2_lm_build: %lld n-grams is too many", h.n_entries);
  DS2_REQUIRE(bos >= 0 && bos < n_words, "ds2_lm_build: bos=%d outside [0, %d)", bos, n_words);
  DS2_REQUIRE(ids && logp && backoff && trie_mask && trie_first && trie_word && buffer, "ds2_lm_build: null pointer");
  for (int n = 0; n < order; ++n)
    DS2_REQUIRE(counts[n] == 0 || (ids[n] && logp[n]), "ds2_lm_build: null pointer for the %d-grams", n + 1);
  DS2_REQUIRE(buffer_bytes >= (size_t)h.bytes, "ds2_lm_build: buffer too small (%zu < %lld bytes)", buffer_bytes,
              h.bytes);
  h.n_words = n_words;
  h.bos = bos;
  cudaStream_t st = as_stream(stream);
  char* b = static_cast<char*>(buffer);
  int* slots = reinterpret_cast<int*>(b + h.off_slots);
  DS2_CHECK_CUDA(cudaMemsetAsync(slots, 0, (size_t)h.n_slots * 4, st));
  DS2_LAUNCH(lm_header_kernel, 1, 1, 0, st, h, reinterpret_cast<LmHeader*>(b));
  long long base = 0;
  for (int n = 1; n <= order; ++n) {
    const long long cnt = counts[n - 1];
    if (cnt > 0)
      DS2_LAUNCH(lm_insert_kernel, cdiv(cnt, LM_THREADS), LM_THREADS, 0, st, n, cnt, base, ids[n - 1], logp[n - 1],
                 backoff[n - 1], slots, reinterpret_cast<ulonglong2*>(b + h.off_keys),
                 reinterpret_cast<float2*>(b + h.off_vals), (unsigned long long)h.n_slots - 1ull);
    base += cnt;
  }
  DS2_CHECK_CUDA(cudaMemcpyAsync(b + h.off_mask, trie_mask, (size_t)n_nodes * 8, cudaMemcpyDeviceToDevice, st));
  DS2_CHECK_CUDA(cudaMemcpyAsync(b + h.off_first, trie_first, (size_t)n_nodes * 4, cudaMemcpyDeviceToDevice, st));
  DS2_CHECK_CUDA(cudaMemcpyAsync(b + h.off_word, trie_word, (size_t)n_nodes * 4, cudaMemcpyDeviceToDevice, st));
  return DS2_OK;
}

}  // extern "C"
