// Prefix beam search for CTC without a language model (row N5): what the reference's BeamCTCDecoder
// (decoder.py:56-118) gets from ctcdecode.CTCBeamDecoder with an empty lm_path, on the GPU.
//
// The decoder is defined by these rules (oracle/beam_oracle.py and DESIGN.md §5.7 carry the same text; ctcdecode's
// algorithm with ext_scorer == nullptr, deviating only where its behaviour is order-dependent or degenerate, (!)):
//
// All path arithmetic is in float64 log space, with lp[c] = log((double) p[c]) and log 0 = -inf.  lse(a, b) is a
// log-sum-exp that returns -inf when both arguments are -inf, and never NaN.  (!) ctcdecode keeps path probabilities
// in fp32; fp64 here makes GPU and oracle agree to rounding of the last bits, so list order can be tested exactly.
//  1. State.  An ordered list of at most W prefixes, each with log_b, log_nb and score = lse(log_b, log_nb).  Before
//     frame 0 the list is {empty prefix: log_b = 0, log_nb = -inf}.
//  2. Prefix identity is by content: the same label sequence is never in the list twice.  A prefix that falls out of
//     the list and is produced again later is the same prefix: its probabilities restart from the new contributions,
//     but it keeps its timestep record (rule 7) -- ctcdecode's trie node coming back with exists_ = true.  A prefix's
//     parent is its sequence minus the last label.
//  3. Character pruning per frame.  If cutoff_prob < 1 or cutoff_top_n < C: order the characters by (p desc, index
//     asc).  With cutoff_prob < 1, take characters in that order, accumulating p in fp64, until the cumulative sum is
//     >= cutoff_prob or cutoff_top_n characters are taken; otherwise take the first cutoff_top_n characters.  In all
//     other cases the kept set K is every character.  The blank can be pruned; it then contributes nothing that frame.
//  4. Candidates at frame t.  For each listed prefix j, with last label l_j, and its parent pi if the parent is in the
//     list, the stay candidate is  b' = lp[blank] + score_j if blank in K, else -inf;
//     nb' = lse(lp[l_j] + nb_j, lp[l_j] + (b_pi if l_pi = l_j else score_pi)), each term present only if l_j in K, and
//     the second only if pi is listed (the empty prefix has no nb terms).  For each listed prefix i and each c in K,
//     c != blank, where i + c is not in the list, the new candidate is  b' = -inf, nb' = lp[c] + (b_i if c = l_i else
//     score_i).
//  5. Selection.  Drop candidates whose score is -inf ((!) ctcdecode can return -inf prefixes when fewer than W finite
//     ones exist).  Order the rest by (score desc, origin asc), the origin being (j, -1) for the stay candidate of list
//     position j and (i, c) for a new candidate ((!) a total order, so ties are defined).  The first W candidates
//     become the new list, in that order.
//  6. Output.  Per utterance, the final list in its order, with each prefix's labels and per-label timesteps; its
//     reported score is -lse(log_b, log_nb) (ctcdecode's sign: a negative log-likelihood, lower is better).
//     n_beams[b] <= W; unused slots have length 0 and score +inf.  sizes[b] = 0 gives one empty beam with score 0.
//  7. Timesteps.  A label's timestep is the frame at which its prefix was first created, with best = that frame's lp.
//     It moves to a later frame t when, at t, the listed parent is extended by the same label with a strictly larger
//     lp than the recorded best (ctcdecode's get_path_trie rule as we read it; not verifiable here).
// Read where the rules leave room (as the oracle does): "created" = first entry into the list; the rule-7 move is
// checked for listed prefixes with a listed parent and l_j in K (the stay candidate's second term), whether or not the
// stay survives selection, and a returning prefix keeps its record unchanged; reported timesteps are the records of
// the prefix's ancestors at the end of the utterance (ctcdecode's get_path_vec walk).  NaN scores count as -inf.
//
// Kernel: one CTA per utterance, the list in shared memory.  Per frame:
//  A. warp 0 loads the C <= 64 probabilities, takes logs and prunes (ranks by (p desc, index asc); the cutoff_prob
//     sum is one sequential fp64 loop in that order, as in the oracle, so both round alike);
//  B. every candidate gets a 64-bit key at a dense position e = i * S + s (S = 1 + |K \ {blank}|, s = 0 the stay of i,
//     s >= 1 the s-th kept non-blank character in ascending index), so e ascending IS origin ascending.  The key is the
//     order-reversing 64-bit image of the fp64 score (ascending key = descending score), all ones for a dropped
//     candidate.  "Is i + c listed?" is a per-slot 64-bit child mask rebuilt each frame from the parent slots;
//  C. the W smallest (key, e) pairs are found by an MSB-first radix select (8 bits per pass over the key, then 7 + 7
//     over e; it stops as soon as the boundary bucket is taken whole, usually after 2-4 passes), then ranked by
//     counting (<= W^2 comparisons) into list order;
//  D. the new list: a new candidate looks up (parent node, label) in the utterance's hash, so a returning prefix finds
//     its old node (rule 2); otherwise it takes the next node of the pool (ids in list order).  Parent slots and child
//     masks of the new list come from a W x W node comparison.
// Nothing is decided by an atomic: shared atomics only count (histograms, compaction before the rank sort, child
// masks), and the hash's slot claims do not change what a lookup returns.  The final beams are written by walking
// parent pointers through the pool.
//
// With an ARPA n-gram language model (row N6, ds2_beam_decode_lm), rules 1-7 hold with these additions: ctcdecode's
// algorithm with a word-level Scorer (PaddlePaddle's ctc_beam_search_decoder with ext_scorer set,
// fill_dictionary(true), OOV_SCORE = -1000).  Parity with ctcdecode and KenLM is unpinned: neither is available here.
//  L0. Model.  An ARPA text file, plain or gzip'd; values parsed to fp32 (as KenLM stores them), an unwritten backoff
//      is 0; word ids in the file's unigram order.  Refused (host side, deepspeech.pytorch_b200/lm.py): a missing
//      file, a file that is not ARPA (a KenLM binary), counts that differ from the \data\ header, duplicate n-grams,
//      order > 5 or >= 2^24 words, no <s> unigram, labels without ' ', a character-based model (every word one
//      character), and a model none of whose words can be spelled with the labels.
//  L1. Vocabulary V and dictionary constraint.  V = the unigrams other than <s>, </s>, <unk> whose every character is
//      a label other than the blank's and the space's ((!) ctcdecode would also map the blank's character).  A prefix
//      splits at spaces into completed words and its partial word (the run after the last space, maybe empty).  A new
//      candidate (i, c), c != blank, exists only if c != space and partial(i)+c is a prefix of a word of V, or
//      c = space and partial(i) is in V.  Leading and double spaces are impossible.  (!) ctcdecode's FST matcher also
//      rejects the first character after a space in the frame where it resets its state; which character that hits
//      depends on the visiting order, so it is not reproduced.
//  L2. LM value.  lm(w | u_1..u_k) is the ARPA conditional log10 probability of w with the context the last N-1 items
//      of (<s>^(N-1), u_1, ..., u_k): the longest listed n-gram plus the backoffs of the longer unlisted contexts (0 for
//      a context that is not listed), the fp32 values summed in fp64 from the longest context down.  A word outside
//      the ARPA vocabulary gets lm = -1000 (LM_OOV).  a(w) = alpha * lm + beta.  (!) The value is used in log10,
//      unconverted (LM_SCALE, lm.cuh): how we read ctcdecode's get_log_cond_prob, not verifiable here.
//  L3. a(w) enters on the path from "...w" to "...w ": the new candidate (i, space) has
//      nb' = lp[space] + score_i + a(partial(i) | ctx(i)), and a listed prefix ending in a space whose parent pi is
//      listed adds it to the second nb term of its stay candidate.  The first nb term gets none.  Scores carry every
//      LM term from then on.
//  L4. Full-beam filter (ctcdecode's min_cutoff).  When the list holds W prefixes at the start of frame t, let
//      m = score of the last listed prefix + log p[blank] - max(0, beta), p[blank] unpruned.  Every contribution from a
//      prefix x through a character c with lp[c] + score_x < m is dropped: the blank term of a stay (x = j), both nb
//      terms of a stay (x = j, then x = pi, c = l_j), a new candidate (x = i).  A dropped contribution does not move a
//      timestep under rule 7.
//  L5. End of utterance.  Each listed prefix that is non-empty and does not end in a space gets
//      score += a(partial | ctx), lm = -1000 for a partial word not in V.  The list is reordered by (score desc, list
//      position asc) and -score is reported.  (!) ctcdecode orders by this score but reports an "approx_ctc" that
//      subtracts beta per character and alpha times a sentence probability including </s>, a term the search never
//      added; here the reported score is the one the beams are ordered by.  sizes[b] = 0 gives one empty beam, 0.
// Kernel (LM = true): per list slot in shared memory the trie node of the partial word, the allowed-extension mask
// (trie children, plus the space when the node is a word) and the N-1 context word ids; per pool node the lm value of
// its partial word, so a returning prefix needs no new lookup.  Pass B drops a new candidate that fails L1 or L4 with
// KEY_DROPPED and adds a(w) to a space candidate; pass D looks up lm for each new node whose partial is a word (<= W
// lookups per frame, each <= 2N - 1 hash probes runs).  The L5 term and the reorder (a W x W counting rank) happen
// before the beams are written.  a(w) is computed with __dmul_rn / __dadd_rn, never contracted, so it rounds as the
// oracle's does.

#include <math_constants.h>

#include <cmath>

#include "common.cuh"
#include "lm.cuh"

namespace ds2 {

namespace {

constexpr int BEAM_THREADS = 512;
constexpr int BEAM_MAX_W = 128, BEAM_MAX_C = 64;
constexpr unsigned long long KEY_DROPPED = ~0ull;

// Per-utterance node pool (NP = T*W + 1 nodes, node 0 = the empty prefix) and (parent, label) -> node hash.
struct BeamPool {
  int* parent;
  int* label;
  int* ts;
  int* depth;
  double* best;
  unsigned long long* hkey;   // 0 = empty slot
  int* hval;
  double* lm;                 // LM only: lm value of the node's partial word (rule L2), if that word is in V
  long long NP, HC;           // HC: power of two >= 2 NP
};

// LM only: the tables of ds2_lm_build and the scorer's parameters
struct BeamLm {
  const void* tables;
  int order, space;
  double alpha, beta;
};

constexpr int LM_CTX = LM_MAX_ORDER - 1;   // context word ids per list slot

void pool_sizes(int T, int W, long long* NP, long long* HC) {
  *NP = (long long)T * W + 1;
  long long h = 1;
  while (h < 2 * *NP) h <<= 1;
  *HC = h;
}

size_t dyn_smem_bytes(int W, int C, bool lm) {
  return (size_t)W * C * 8          // keys
         + (size_t)W * 8 * 8        // lb, lnb, sc, sb, snb, b2, nb2, child masks
         + (size_t)W * 4 * 10       // lab, node, pnode, pslot, lab2, node2, pnode2, sel, rnk, ord
         + (lm ? (size_t)W * (8 + 8 + 4 + 4 * LM_CTX) : 0);   // LM: amask, lmv, tn, ctx
}

// a(w) = alpha * lm + beta (rule L2), rounded as written
__device__ __forceinline__ double lm_term(const BeamLm& L, double lm) {
  return __dadd_rn(__dmul_rn(L.alpha, lm), L.beta);
}

__device__ __forceinline__ double lse(double a, double b) {
  const double m = fmax(a, b);
  if (m == -CUDART_INF) return -CUDART_INF;
  return m + log1p(exp(-fabs(a - b)));
}

// ascending key = descending score; +0 and -0 map alike
__device__ __forceinline__ unsigned long long score_key(double s) {
  if (!(s > -CUDART_INF)) return KEY_DROPPED;                      // -inf and NaN are dropped (rule 5)
  const unsigned long long u = (unsigned long long)__double_as_longlong(s + 0.0);
  const unsigned long long asc = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
  return ~asc;
}

__device__ __forceinline__ unsigned long long hash_key(int pnode, int c) {
  return (((unsigned long long)pnode << 6) | (unsigned)c) + 1ull;
}
__device__ __forceinline__ long long hash_slot(unsigned long long k, long long HC) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (long long)(k & (unsigned long long)(HC - 1));
}

// Streaming (ds2_beam_decode_stream): the beam list of a session between calls, one record per pool slot.  Record:
// n_list, pool_next, frames decoded so far, 0 (4 ints) | lb, lnb, sc, lmv (W doubles each) | kids, amask (W u64 each) |
// lab, node, pnode, pslot, tn (W ints each) | ctx (W * LM_CTX ints); every array 16-byte aligned.
size_t stream_rec_bytes(int W) {
  return align_up(16 + (size_t)W * (4 * 8 + 2 * 8 + 5 * 4) + (size_t)W * LM_CTX * 4, 256);
}

// The session a streaming CTA runs: items[5 * s ..] = {row0, n_frames, slot, flags, out_row}; flags bit 0: the session's
// first call (clear its hash, start from the empty prefix), bit 1: final (write all W beams, else only the best);
// probability rows [row0, row0 + n_frames) of the packed (rows, C) array; beams to rows out_row.. of (rows, Tout).
struct StreamArgs {
  const int32_t* items;
  unsigned char* recs;
  size_t rec_bytes;
  int Tout;
};

// One beam search: utterance u, in pool slot `slot`, written to output row `out`.  TOP = false writes every beam
// (rule 6) at out = u; TOP = true writes only the best beam: labels row `out` of (rows, T) and lengths[out] (the grid
// entry, where timesteps, scores and n_beams are NULL).  Both kernels below run this body.
template <bool LM, bool TOP, bool STREAM = false>
__device__ __forceinline__ void beam_search_item(int u, int slot, int out, int T, int C,
                                                 const float* __restrict__ probs, const int32_t* __restrict__ out_len,
                                                 int blank, int W, int top_n, float cutoff_prob,
                                                 int32_t* __restrict__ labels, int32_t* __restrict__ timesteps,
                                                 int32_t* __restrict__ lengths, double* __restrict__ scores,
                                                 int32_t* __restrict__ n_beams, const BeamPool& pool,
                                                 const BeamLm& lmp, const StreamArgs sa = StreamArgs{}) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* key = reinterpret_cast<unsigned long long*>(smem_raw);
  double* lb = reinterpret_cast<double*>(key + (size_t)W * C);
  double* lnb = lb + W;
  double* sc = lnb + W;
  double* sb = sc + W;
  double* snb = sb + W;
  double* b2 = snb + W;
  double* nb2 = b2 + W;
  unsigned long long* kids = reinterpret_cast<unsigned long long*>(nb2 + W);
  int* lab = reinterpret_cast<int*>(kids + W);
  int* node = lab + W;
  int* pnode = node + W;
  int* pslot = pnode + W;
  int* lab2 = pslot + W;
  int* node2 = lab2 + W;
  int* pnode2 = node2 + W;
  int* sel = pnode2 + W;
  int* rnk = sel + W;
  int* ord = rnk + W;
  // LM only (rules L1-L5): per slot the allowed extensions, the lm value of the partial word, its trie node, and
  // the N-1 context word ids (oldest first)
  unsigned long long* amask = reinterpret_cast<unsigned long long*>(ord + W);
  double* lmv = reinterpret_cast<double*>(amask + W);
  int* tn = reinterpret_cast<int*>(lmv + W);
  int* ctx = tn + W;

  __shared__ double lp[BEAM_MAX_C];
  __shared__ float pf[BEAM_MAX_C];
  __shared__ int ordc[BEAM_MAX_C];
  __shared__ int knb[BEAM_MAX_C];
  __shared__ int hist[256];
  __shared__ unsigned warp_new[BEAM_MAX_W / 32];
  __shared__ unsigned long long kmask, pre_hi;
  __shared__ int n_list, nK, n_valid, n_sel, need, passes, done, pre_e, pool_next, t_base;

  const long long NP = pool.NP, HC = pool.HC;
  int* P_par = pool.parent + (size_t)slot * NP;
  int* P_lab = pool.label + (size_t)slot * NP;
  int* P_ts = pool.ts + (size_t)slot * NP;
  int* P_depth = pool.depth + (size_t)slot * NP;
  double* P_best = pool.best + (size_t)slot * NP;
  unsigned long long* hk = pool.hkey + (size_t)slot * HC;
  int* hv = pool.hval + (size_t)slot * HC;

  // streaming: the session's item and its saved list (a resumed call loads it instead of starting afresh)
  const int32_t* it = STREAM ? sa.items + 5 * (size_t)u : nullptr;
  const bool resume = STREAM && !(it[3] & 1);
  unsigned char* rec = STREAM ? sa.recs + (size_t)slot * sa.rec_bytes : nullptr;
  double* R_lb = reinterpret_cast<double*>(rec + 16);
  double* R_lnb = R_lb + W;
  double* R_sc = R_lnb + W;
  double* R_lmv = R_sc + W;
  unsigned long long* R_kids = reinterpret_cast<unsigned long long*>(R_lmv + W);
  unsigned long long* R_amask = R_kids + W;
  int* R_lab = reinterpret_cast<int*>(R_amask + W);
  int* R_node = R_lab + W;
  int* R_pnode = R_node + W;
  int* R_pslot = R_pnode + W;
  int* R_tn = R_pslot + W;
  int* R_ctx = R_tn + W;
  if (!resume)
    for (long long i = tid; i < HC; i += BEAM_THREADS) hk[i] = 0ull;
  const int Tu = STREAM ? it[1] : (out_len ? min(max(out_len[u], 0), T) : T);
  const float* prow = STREAM ? probs + (size_t)it[0] * C : probs + (size_t)u * T * C;
  if (tid == 0) t_base = resume ? reinterpret_cast<const int*>(rec)[2] : 0;
  if (resume) {
    if (tid == 0) {
      n_list = reinterpret_cast<const int*>(rec)[0];
      pool_next = reinterpret_cast<const int*>(rec)[1];
    }
    if (tid < W) {
      lb[tid] = R_lb[tid]; lnb[tid] = R_lnb[tid]; sc[tid] = R_sc[tid]; kids[tid] = R_kids[tid];
      lab[tid] = R_lab[tid]; node[tid] = R_node[tid]; pnode[tid] = R_pnode[tid]; pslot[tid] = R_pslot[tid];
      if constexpr (LM) {
        lmv[tid] = R_lmv[tid]; amask[tid] = R_amask[tid]; tn[tid] = R_tn[tid];
        for (int k = 0; k < LM_CTX; ++k) ctx[tid * LM_CTX + k] = R_ctx[tid * LM_CTX + k];
      }
    }
  } else if (tid == 0) {
    P_par[0] = -1; P_lab[0] = -1; P_ts[0] = 0; P_depth[0] = 0; P_best[0] = -CUDART_INF;
    lb[0] = 0.0; lnb[0] = -CUDART_INF; sc[0] = 0.0;
    lab[0] = -1; node[0] = 0; pnode[0] = -1; pslot[0] = -1; kids[0] = 0ull;
    n_list = 1; pool_next = 1;
  }
  LmView lmt;
  const int order = LM ? lmp.order : 1, space = LM ? lmp.space : -1;
  if constexpr (LM) {
    lmt = lm_view(lmp.tables);
    if (tid == 0 && !resume) {
      tn[0] = 0;                                     // the root: the empty partial word, not a word itself
      amask[0] = lmt.mask[0];
      lmv[0] = 0.0;
      for (int k = 0; k < LM_CTX; ++k) ctx[k] = lmt.bos;
    }
  }
  __syncthreads();

  const bool prune = cutoff_prob < 1.f || top_n < C;
  const int t0 = STREAM ? t_base : 0;                 // stream frame of this call's first row
  for (int t = 0; t < Tu; ++t) {
    const int tg = t0 + t;
    // ---- A. probabilities, logs, the kept set K (rule 3)
    if (warp == 0) {
      const float* p = prow + (size_t)t * C;
      for (int c = lane; c < C; c += 32) {
        const float v = p[c];
        pf[c] = v;
        lp[c] = log((double)v);
      }
      __syncwarp();
      bool keep0 = true, keep1 = true;
      if (prune) {
        int r0 = 0, r1 = 0;
        const int c0 = lane, c1 = lane + 32;
        const float v0 = c0 < C ? pf[c0] : 0.f, v1 = c1 < C ? pf[c1] : 0.f;
        for (int k = 0; k < C; ++k) {
          const float w = pf[k];
          r0 += (w > v0 || (w == v0 && k < c0));
          r1 += (w > v1 || (w == v1 && k < c1));
        }
        if (c0 < C) ordc[r0] = c0;
        if (c1 < C) ordc[r1] = c1;
        __syncwarp();
        int nkeep = min(top_n, C);
        if (cutoff_prob < 1.f) {
          if (lane == 0) {
            const double thr = (double)cutoff_prob;
            double cum = 0.0;
            int m = 0;
            while (m < C) {
              cum += (double)pf[ordc[m]];
              ++m;
              if (cum >= thr || m >= top_n) break;
            }
            nkeep = m;
          }
          nkeep = __shfl_sync(0xffffffffu, nkeep, 0);
        }
        keep0 = r0 < nkeep;
        keep1 = r1 < nkeep;
      }
      const unsigned m0 = __ballot_sync(0xffffffffu, lane < C && keep0);
      const unsigned m1 = __ballot_sync(0xffffffffu, lane + 32 < C && keep1);
      const unsigned long long km = ((unsigned long long)m1 << 32) | m0;
      const unsigned long long nbm = km & ~(1ull << blank);
      const unsigned long long lt = (1ull << lane) - 1ull;
      if ((nbm >> lane) & 1ull) knb[__popcll(nbm & lt)] = lane;
      if ((nbm >> (lane + 32)) & 1ull) knb[__popcll(nbm & ((lt << 32) | 0xffffffffull))] = lane + 32;
      if (lane == 0) {
        kmask = km;
        nK = __popcll(nbm);
        n_valid = 0;
        n_sel = 0;
      }
    }
    if (tid < W) rnk[tid] = 0;
    __syncthreads();

    // ---- B. candidate keys (rule 4); the timestep move of rule 7
    const int n = n_list, S = 1 + nK, N = n * S;
    const unsigned long long km = kmask;
    const bool blank_in = (km >> blank) & 1ull;
    // L4: contributions with lp[c] + score_x < m are dropped; m = -inf (nothing dropped) unless the list is full
    double m = -CUDART_INF;
    if constexpr (LM) {
      if (n == W) m = sc[n - 1] + lp[blank] - fmax(0.0, lmp.beta);
    }
    int valid = 0;
    for (int e = tid; e < N; e += BEAM_THREADS) {
      const int i = e / S, s = e - i * S;
      double v;
      if (s == 0) {
        double bb = blank_in ? lp[blank] + sc[i] : -CUDART_INF;
        if constexpr (LM) {
          if (bb < m) bb = -CUDART_INF;
        }
        double nn = -CUDART_INF;
        const int l = lab[i];
        if (l >= 0 && ((km >> l) & 1ull)) {
          const double lpl = lp[l];
          nn = lpl + lnb[i];
          const int pi = pslot[i];
          if constexpr (LM) {
            if (lpl + sc[i] < m) nn = -CUDART_INF;
            if (pi >= 0 && !(lpl + sc[pi] < m)) {
              double v2 = lpl + (lab[pi] == l ? lb[pi] : sc[pi]);
              if (l == space) v2 = __dadd_rn(v2, lm_term(lmp, lmv[pi]));            // L3
              nn = lse(nn, v2);
              const int nd = node[i];
              if (lpl > P_best[nd]) { P_best[nd] = lpl; P_ts[nd] = tg; }
            }
          } else if (pi >= 0) {
            nn = lse(nn, lpl + (lab[pi] == l ? lb[pi] : sc[pi]));
            const int nd = node[i];
            if (lpl > P_best[nd]) { P_best[nd] = lpl; P_ts[nd] = tg; }
          }
        }
        sb[i] = bb;
        snb[i] = nn;
        v = lse(bb, nn);
      } else {
        const int c = knb[s - 1];
        if constexpr (LM) {
          // L1 (allowed extensions), L4, then the L3 term of a space candidate
          if (((kids[i] >> c) & 1ull) || !((amask[i] >> c) & 1ull) || lp[c] + sc[i] < m) {
            v = -CUDART_INF;
          } else {
            v = lp[c] + (c == lab[i] ? lb[i] : sc[i]);
            if (c == space) v = __dadd_rn(v, lm_term(lmp, lmv[i]));
          }
        } else {
          v = ((kids[i] >> c) & 1ull) ? -CUDART_INF : lp[c] + (c == lab[i] ? lb[i] : sc[i]);
        }
      }
      const unsigned long long k = score_key(v);
      key[e] = k;
      valid += (k != KEY_DROPPED);
    }
    valid = __reduce_add_sync(0xffffffffu, valid);
    if (lane == 0 && valid) atomicAdd(&n_valid, valid);
    __syncthreads();

    // ---- C. the W smallest (key, e), in order (rule 5)
    const int nv = n_valid, Wsel = min(W, nv);
    bool all_valid = nv <= W;
    if (!all_valid) {
      if (tid == 0) { need = Wsel; pre_hi = 0ull; pre_e = 0; done = 0; passes = 0; }
      for (int p = 0; p < 10; ++p) {
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        const unsigned long long ph = pre_hi;
        const int pe = pre_e;
        for (int e = tid; e < N; e += BEAM_THREADS) {
          const unsigned long long k = key[e];
          bool in;
          int d;
          if (p < 8) {
            in = p == 0 || (k >> (64 - 8 * p)) == (ph >> (64 - 8 * p));
            d = (int)((k >> (56 - 8 * p)) & 255ull);
          } else if (p == 8) {
            in = k == ph;
            d = e >> 7;
          } else {
            in = k == ph && (e >> 7) == pe;
            d = e & 127;
          }
          if (in) atomicAdd(&hist[d], 1);
        }
        __syncthreads();
        if (warp == 0) {
          int h[8], sum = 0;
#pragma unroll
          for (int q = 0; q < 8; ++q) { h[q] = hist[lane * 8 + q]; sum += h[q]; }
          int incl = sum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
          }
          const int nd = need, excl = incl - sum;
          const unsigned hit = __ballot_sync(0xffffffffu, excl < nd && nd <= incl);
          if (lane == __ffs(hit) - 1) {
            int before = excl, bsel = lane * 8;
            while (before + hist[bsel] < nd) before += hist[bsel++];
            const int rem = nd - before;
            if (p < 8) pre_hi = ph | ((unsigned long long)bsel << (56 - 8 * p));
            else if (p == 8) pre_e = bsel;
            else pre_e = (pe << 7) | bsel;
            need = rem;
            done = rem == hist[bsel];
            passes = p + 1;
          }
        }
        __syncthreads();
        if (done) break;
      }
    }
    {
      const int ps = all_valid ? 0 : passes;
      const unsigned long long ph = pre_hi;
      const int pe = pre_e;
      for (int e = tid; e < N; e += BEAM_THREADS) {
        const unsigned long long k = key[e];
        bool s;
        if (all_valid) s = k != KEY_DROPPED;
        else if (ps <= 8) s = (k >> (64 - 8 * ps)) <= (ph >> (64 - 8 * ps));
        else if (ps == 9) s = k < ph || (k == ph && (e >> 7) <= pe);
        else s = k < ph || (k == ph && e <= pe);
        if (s) {
          const int at = atomicAdd(&n_sel, 1);   // at < Wsel: the select takes exactly Wsel candidates
          if (at < W) sel[at] = e;
        }
      }
    }
    __syncthreads();
    for (int x = tid; x < Wsel * Wsel; x += BEAM_THREADS) {
      const int a = x / Wsel, o = x - a * Wsel;
      const int ea = sel[a], eo = sel[o];
      const unsigned long long ka = key[ea], ko = key[eo];
      if (ko < ka || (ko == ka && eo < ea)) atomicAdd(&rnk[a], 1);
    }
    __syncthreads();
    if (tid < Wsel) ord[rnk[tid]] = sel[tid];
    __syncthreads();

    // ---- D. the new list; returning prefixes find their node (rule 2), new ones take the next pool nodes
    bool is_new = false;
    long long hs = 0;
    unsigned long long hkey_new = 0ull;
    int tn_new = 0, ctx_new[LM_CTX];   // LM: the new slot's trie node, context and lm value (written after the barrier)
    double lmv_new = 0.0;
    if (tid < Wsel) {
      const int e = ord[tid], i = e / S, s = e - i * S;
      if constexpr (LM) {
        tn_new = tn[i];
        lmv_new = lmv[i];
#pragma unroll
        for (int k = 0; k < LM_CTX; ++k) ctx_new[k] = ctx[i * LM_CTX + k];
      }
      if (s == 0) {
        b2[tid] = sb[i]; nb2[tid] = snb[i]; lab2[tid] = lab[i]; node2[tid] = node[i]; pnode2[tid] = pnode[i];
      } else {
        const int c = knb[s - 1];
        b2[tid] = -CUDART_INF;
        double nb = lp[c] + (c == lab[i] ? lb[i] : sc[i]);
        if constexpr (LM) {
          if (c == space) {                                 // "...w" -> "...w ": w joins the context
            nb = __dadd_rn(nb, lm_term(lmp, lmv[i]));
#pragma unroll
            for (int k = 0; k < LM_CTX - 1; ++k) ctx_new[k] = ctx_new[k + 1];
            ctx_new[LM_CTX - 1] = lmt.word[tn_new];
            tn_new = 0;
          } else {
            tn_new = lmt.first[tn_new] + __popcll(lmt.mask[tn_new] & ((1ull << c) - 1ull));
          }
        }
        nb2[tid] = nb;
        lab2[tid] = c;
        pnode2[tid] = node[i];
        hkey_new = hash_key(node[i], c);
        hs = hash_slot(hkey_new, HC);
        int found = -1;
        for (;;) {
          const unsigned long long x = hk[hs];
          if (x == hkey_new) { found = hv[hs]; break; }
          if (x == 0ull) break;
          hs = (hs + 1) & (HC - 1);
        }
        node2[tid] = found;
        is_new = found < 0;
        if constexpr (LM) {                                 // a returning prefix (rule 2) keeps its lm value;
          lmv_new = is_new ? 0.0 : pool.lm[(size_t)slot * NP + found];   // a new one is looked up below
        }
      }
    }
    if (tid < BEAM_MAX_W) {
      const unsigned m = __ballot_sync(0xffffffffu, is_new);
      if (lane == 0) warp_new[warp] = m;
    }
    // pool_next is read here, one barrier before thread 0 advances it below: no thread may see the advanced value
    const int first_new = pool_next;
    __syncthreads();
    if (tid < Wsel) {
      if constexpr (LM) {
        // the slot's own context, written and then read by this thread only
#pragma unroll
        for (int k = 0; k < LM_CTX; ++k) ctx[tid * LM_CTX + k] = ctx_new[k];
        if (is_new && lmt.word[tn_new] >= 0)
          lmv_new = lm_logp(lmt, order, ctx + tid * LM_CTX + LM_CTX - (order - 1), lmt.word[tn_new]);
      }
      if (is_new) {
        int id = first_new + __popc(warp_new[warp] & ((1u << lane) - 1u));
        for (int w = 0; w < warp; ++w) id += __popc(warp_new[w]);
        const int pn = pnode2[tid], c = lab2[tid];
        P_par[id] = pn; P_lab[id] = c; P_ts[id] = tg; P_best[id] = lp[c]; P_depth[id] = P_depth[pn] + 1;
        for (;;) {                                       // hs: the empty slot the lookup stopped at, or later
          const unsigned long long prev = atomicCAS(&hk[hs], 0ull, hkey_new);
          if (prev == 0ull) { hv[hs] = id; break; }
          hs = (hs + 1) & (HC - 1);
        }
        node2[tid] = id;
        if constexpr (LM) pool.lm[(size_t)slot * NP + id] = lmv_new;
      }
      lb[tid] = b2[tid]; lnb[tid] = nb2[tid]; sc[tid] = lse(b2[tid], nb2[tid]);
      lab[tid] = lab2[tid]; node[tid] = node2[tid]; pnode[tid] = pnode2[tid];
      pslot[tid] = -1; kids[tid] = 0ull;
      if constexpr (LM) {
        tn[tid] = tn_new;
        lmv[tid] = lmv_new;
        amask[tid] = lmt.mask[tn_new] | (lmt.word[tn_new] >= 0 ? 1ull << space : 0ull);
      }
    }
    if (tid == 0) {
      int added = 0;
      for (int w = 0; w < BEAM_MAX_W / 32; ++w) added += __popc(warp_new[w]);
      pool_next = first_new + added;
      n_list = Wsel;
    }
    __syncthreads();
    for (int x = tid; x < Wsel * Wsel; x += BEAM_THREADS) {
      const int j = x / Wsel, k = x - j * Wsel;
      if (node[k] == pnode[j]) {
        pslot[j] = k;
        atomicOr(&kids[k], 1ull << lab[j]);
      }
    }
    __syncthreads();
  }

  // ---- streaming: save the list for the session's next call (the end term below does not change it)
  if constexpr (STREAM) {
    if (tid < W) {
      R_lb[tid] = lb[tid]; R_lnb[tid] = lnb[tid]; R_sc[tid] = sc[tid]; R_kids[tid] = kids[tid];
      R_lab[tid] = lab[tid]; R_node[tid] = node[tid]; R_pnode[tid] = pnode[tid]; R_pslot[tid] = pslot[tid];
      if constexpr (LM) {
        R_lmv[tid] = lmv[tid]; R_amask[tid] = amask[tid]; R_tn[tid] = tn[tid];
        for (int k = 0; k < LM_CTX; ++k) R_ctx[tid * LM_CTX + k] = ctx[tid * LM_CTX + k];
      }
    }
    if (tid == 0) {
      int* h = reinterpret_cast<int*>(rec);
      h[0] = n_list; h[1] = pool_next; h[2] = t0 + Tu; h[3] = 0;
    }
  }

  // ---- LM: the end-of-utterance term and the reorder (rule L5); the final score goes to sb, the position to rnk
  if constexpr (LM) {
    const int n = n_list;
    if (tid < n) {
      double f = sc[tid];
      const int l = lab[tid];
      if (l >= 0 && l != space) f = __dadd_rn(f, lm_term(lmp, lmt.word[tn[tid]] >= 0 ? lmv[tid] : LM_OOV));
      sb[tid] = f;
      rnk[tid] = 0;
    }
    __syncthreads();
    for (int x = tid; x < n * n; x += BEAM_THREADS) {
      const int a = x / n, o = x - a * n;
      if (sb[o] > sb[a] || (sb[o] == sb[a] && o < a)) atomicAdd(&rnk[a], 1);
    }
    __syncthreads();
  }

  // ---- output (rule 6): zero the rows, then walk each beam's parent chain
  if constexpr (STREAM) {   // final: all W beams in rows out_row.., else the best one in row out_row
    const int rows = (it[3] & 2) ? W : 1, Tout = sa.Tout;
    const size_t r0 = (size_t)it[4];
    for (size_t x = tid; x < (size_t)rows * Tout; x += BEAM_THREADS) {
      labels[r0 * Tout + x] = 0;
      timesteps[r0 * Tout + x] = 0;
    }
    __syncthreads();
    if (tid < W) {
      const int r = LM && tid < n_list ? rnk[tid] : tid;
      if (r < rows) {
        if (tid < n_list) {
          int nd = node[tid];
          const int len = P_depth[nd];
          lengths[r0 + r] = len;
          scores[r0 + r] = -(LM ? sb[tid] : sc[tid]) + 0.0;
          int32_t* L = labels + (r0 + r) * Tout;
          int32_t* S = timesteps + (r0 + r) * Tout;
          for (int pos = len - 1; pos >= 0; --pos) {
            L[pos] = P_lab[nd];
            S[pos] = P_ts[nd];
            nd = P_par[nd];
          }
        } else {
          lengths[r0 + r] = 0;
          scores[r0 + r] = CUDART_INF;
        }
      }
    }
    if (tid == 0) n_beams[u] = n_list;
    return;
  }
  if constexpr (TOP) {
    int32_t* L = labels + (size_t)out * T;
    for (int x = tid; x < T; x += BEAM_THREADS) L[x] = 0;
    __syncthreads();
    const int n = n_list;
    if (n == 0) {
      if (tid == 0) lengths[out] = 0;
    } else if (tid < n && (LM ? rnk[tid] : tid) == 0) {
      int nd = node[tid];
      const int len = P_depth[nd];
      lengths[out] = len;
      for (int pos = len - 1; pos >= 0; --pos) {
        L[pos] = P_lab[nd];
        nd = P_par[nd];
      }
    }
    return;
  }
  const size_t row0 = (size_t)out * W * T;
  for (size_t x = tid; x < (size_t)W * T; x += BEAM_THREADS) {
    labels[row0 + x] = 0;
    timesteps[row0 + x] = 0;
  }
  __syncthreads();
  if (tid < W) {
    const int r = LM && tid < n_list ? rnk[tid] : tid;
    const size_t o = (size_t)out * W + r;
    if (tid < n_list) {
      int nd = node[tid];
      const int len = P_depth[nd];
      lengths[o] = len;
      scores[o] = -(LM ? sb[tid] : sc[tid]) + 0.0;
      int32_t* L = labels + row0 + (size_t)r * T;
      int32_t* S = timesteps + row0 + (size_t)r * T;
      for (int pos = len - 1; pos >= 0; --pos) {
        L[pos] = P_lab[nd];
        S[pos] = P_ts[nd];
        nd = P_par[nd];
      }
    } else {
      lengths[o] = 0;
      scores[o] = CUDART_INF;
    }
  }
  if (tid == 0) n_beams[out] = n_list;
}

// ds2_beam_decode / ds2_beam_decode_lm: one CTA per utterance, pool slot = utterance
template <bool LM>
__global__ void __launch_bounds__(BEAM_THREADS)
beam_decode_kernel(int T, int C, const float* __restrict__ probs, const int32_t* __restrict__ out_len, int blank,
                   int W, int top_n, float cutoff_prob, int32_t* __restrict__ labels, int32_t* __restrict__ timesteps,
                   int32_t* __restrict__ lengths, double* __restrict__ scores, int32_t* __restrict__ n_beams,
                   BeamPool pool, BeamLm lmp) {
  const int u = blockIdx.x;
  beam_search_item<LM, false>(u, u, u, T, C, probs, out_len, blank, W, top_n, cutoff_prob, labels, timesteps,
                              lengths, scores, n_beams, pool, lmp);
}

// ds2_beam_decode_lm_grid: item i = u * K + k is utterance u with pair k (utterance-major, so the caller's length
// order is the start order).  CTA b runs items b, b + gridDim.x, ... in its own pool slot b; each item starts from a
// cleared hash and node 0, so which slot runs an item does not change its result.
__global__ void __launch_bounds__(BEAM_THREADS)
beam_decode_grid_kernel(int B, int K, int T, int C, const float* __restrict__ probs,
                        const int32_t* __restrict__ out_len, int blank, int W, int top_n, float cutoff_prob,
                        const double* __restrict__ pairs, int32_t* __restrict__ labels,
                        int32_t* __restrict__ lengths, BeamPool pool, BeamLm lmp) {
  const int n_items = B * K;
  for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
    const int u = it / K, k = it - u * K;
    BeamLm L = lmp;
    L.alpha = pairs[2 * k];
    L.beta = pairs[2 * k + 1];
    beam_search_item<true, true>(u, blockIdx.x, k * B + u, T, C, probs, out_len, blank, W, top_n, cutoff_prob,
                                 labels, nullptr, lengths, nullptr, nullptr, pool, L);
    __syncthreads();   // the next item's set-up overwrites the list this one's output read
  }
}

// ds2_beam_decode_stream / ds2_beam_decode_lm_stream: one CTA per session of the call, in its own pool slot
template <bool LM>
__global__ void __launch_bounds__(BEAM_THREADS)
beam_decode_stream_kernel(int C, const float* __restrict__ probs, int blank, int W, int top_n, float cutoff_prob,
                          int32_t* __restrict__ labels, int32_t* __restrict__ timesteps, int32_t* __restrict__ lengths,
                          double* __restrict__ scores, int32_t* __restrict__ n_beams, BeamPool pool, BeamLm lmp,
                          StreamArgs sa) {
  const int s = blockIdx.x;
  beam_search_item<LM, false, true>(s, sa.items[5 * s + 2], s, 0, C, probs, nullptr, blank, W, top_n, cutoff_prob,
                                    labels, timesteps, lengths, scores, n_beams, pool, lmp, sa);
}

// The pools of `slots` CTAs at offset `off` of a workspace, each array 256-byte aligned:
//   parent | label | ts | depth (slots*NP ints) | best (slots*NP doubles) | hkey | hval (slots*HC) | LM: lm (slots*NP)
// With a null base only `off` advances.
BeamPool carve_pool(void* base, size_t& off, int slots, int T, int W, bool lm) {
  BeamPool pool;
  pool_sizes(T, W, &pool.NP, &pool.HC);
  const size_t n = (size_t)slots * pool.NP, h = (size_t)slots * pool.HC;
  pool.parent = carve<int>(base, off, n * 4);
  pool.label = carve<int>(base, off, n * 4);
  pool.ts = carve<int>(base, off, n * 4);
  pool.depth = carve<int>(base, off, n * 4);
  pool.best = carve<double>(base, off, n * 8);
  pool.hkey = carve<unsigned long long>(base, off, h * 8);
  pool.hval = carve<int>(base, off, h * 4);
  pool.lm = lm ? carve<double>(base, off, n * 8) : nullptr;
  return pool;
}

size_t beam_workspace_bytes(int B, int T, int beam_width, bool lm) {
  if (B <= 0 || T <= 0 || beam_width <= 0) return 0;
  size_t off = 0;
  carve_pool(nullptr, off, B, T, beam_width, lm);
  return off;
}

// the checks every beam entry makes (DS2_REQUIRE returns from the caller's frame through this function's result)
int beam_check_args(const char* fn, int B, int T, int C, int blank, int beam_width, int cutoff_top_n,
                    float cutoff_prob) {
  DS2_REQUIRE(B > 0 && T > 0, "%s: bad shape B=%d T=%d", fn, B, T);
  DS2_REQUIRE(C >= 2 && C <= BEAM_MAX_C, "%s: C=%d outside [2, %d]", fn, C, BEAM_MAX_C);
  DS2_REQUIRE(blank >= 0 && blank < C, "%s: blank=%d outside [0, C=%d)", fn, blank, C);
  DS2_REQUIRE(beam_width >= 1 && beam_width <= BEAM_MAX_W, "%s: beam_width=%d outside [1, %d]", fn, beam_width,
              BEAM_MAX_W);
  DS2_REQUIRE(cutoff_top_n >= 1, "%s: cutoff_top_n=%d < 1", fn, cutoff_top_n);
  DS2_REQUIRE(cutoff_prob > 0.f && cutoff_prob <= 1.f, "%s: cutoff_prob=%g outside (0, 1]", fn, (double)cutoff_prob);
  DS2_REQUIRE((long long)T * beam_width < (1ll << 31) - 1, "%s: T*beam_width too large for the node pool", fn);
  return DS2_OK;
}

int lm_check_args(const char* fn, int C, int blank, const void* lm, int lm_order, int space) {
  DS2_REQUIRE(lm, "%s: null language model", fn);
  DS2_REQUIRE(lm_order >= 1 && lm_order <= LM_MAX_ORDER, "%s: order=%d outside [1, %d]", fn, lm_order,
              LM_MAX_ORDER);
  DS2_REQUIRE(space >= 0 && space < C && space != blank && C <= BEAM_MAX_C,
              "%s: space=%d outside [0, C=%d) or equal to blank=%d", fn, space, C, blank);
  return DS2_OK;
}

template <bool LM>
int beam_decode_launch(const char* fn, int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                       int beam_width, int cutoff_top_n, float cutoff_prob, BeamLm lm, int32_t* labels,
                       int32_t* timesteps, int32_t* lengths, double* scores, int32_t* n_beams, void* workspace,
                       size_t workspace_bytes, void* stream) {
  const int rc = beam_check_args(fn, B, T, C, blank, beam_width, cutoff_top_n, cutoff_prob);
  if (rc != DS2_OK) return rc;
  DS2_REQUIRE(probs && labels && timesteps && lengths && scores && n_beams, "%s: null pointer", fn);
  size_t need = 0;
  const BeamPool pool = carve_pool(workspace, need, B, T, beam_width, LM);
  DS2_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu bytes)", fn, workspace_bytes,
              need);
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    DS2_CHECK_CUDA(cudaFuncSetAttribute(beam_decode_kernel<LM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)dyn_smem_bytes(BEAM_MAX_W, BEAM_MAX_C, LM)));
    attr_once.done();
  }
  cudaStream_t st = as_stream(stream);
  DS2_PROF(LM ? "beam_decode_lm" : "beam_decode", st);
  DS2_LAUNCH(beam_decode_kernel<LM>, B, BEAM_THREADS, dyn_smem_bytes(beam_width, C, LM), st, T, C, probs, out_len,
             blank, beam_width, cutoff_top_n, cutoff_prob, labels, timesteps, lengths, scores, n_beams, pool, lm);
  return DS2_OK;
}

// CTAs of the grid kernel: as many as can be resident on the current device (occupancy x SMs), at most `items`;
// 0 if the device cannot be queried
long long grid_slots(long long items, int W, int C) {
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    if (cudaFuncSetAttribute(beam_decode_grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)dyn_smem_bytes(BEAM_MAX_W, BEAM_MAX_C, true)) != cudaSuccess)
      return 0;
    attr_once.done();
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, beam_decode_grid_kernel, BEAM_THREADS,
                                                    dyn_smem_bytes(W, C, true)) != cudaSuccess || per_sm < 1)
    return 0;
  const long long resident = (long long)per_sm * device_sm_count();
  return resident < items ? resident : items;
}

// Workspace of the grid decode (bytes; with a base, also the addresses): the K (alpha, beta) pairs, 256-byte aligned,
// then the pools of `slots` CTAs
struct GridWs { double* pairs; BeamPool pool; };
size_t grid_ws_carve(int K, int slots, int T, int W, void* base, GridWs& w) {
  size_t off = 0;
  w.pairs = carve<double>(base, off, (size_t)K * 2 * sizeof(double));
  w.pool = carve_pool(base, off, slots, T, W, true);
  return off;
}

// Streaming state of max_sessions slots: the pools (sized for max_frames), then one list record per slot
struct StreamState { BeamPool pool; unsigned char* recs; size_t rec_bytes; };
size_t stream_state_carve(int S, int max_frames, int W, bool lm, void* base, StreamState& st) {
  size_t off = 0;
  st.pool = carve_pool(base, off, S, max_frames, W, lm);
  st.rec_bytes = stream_rec_bytes(W);
  st.recs = carve<unsigned char>(base, off, (size_t)S * st.rec_bytes);
  return off;
}

template <bool LM>
int beam_stream_launch(const char* fn, int n_sess, int C, const float* probs, const int32_t* items, int blank,
                       int beam_width, int cutoff_top_n, float cutoff_prob, BeamLm lm, int max_sessions,
                       int max_frames, int Tout, int32_t* labels, int32_t* timesteps, int32_t* lengths,
                       double* scores, int32_t* n_beams, void* state, size_t state_bytes, void* stream) {
  const int rc = beam_check_args(fn, max_sessions, max_frames, C, blank, beam_width, cutoff_top_n, cutoff_prob);
  if (rc != DS2_OK) return rc;
  DS2_REQUIRE(n_sess > 0 && n_sess <= max_sessions && Tout > 0, "%s: bad shape n_sess=%d Tout=%d", fn, n_sess, Tout);
  DS2_REQUIRE(probs && items && labels && timesteps && lengths && scores && n_beams, "%s: null pointer", fn);
  StreamState S;
  const size_t need = stream_state_carve(max_sessions, max_frames, beam_width, LM, state, S);
  DS2_REQUIRE(state && state_bytes >= need, "%s: state too small (%zu < %zu bytes)", fn, state_bytes, need);
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    DS2_CHECK_CUDA(cudaFuncSetAttribute(beam_decode_stream_kernel<LM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)dyn_smem_bytes(BEAM_MAX_W, BEAM_MAX_C, LM)));
    attr_once.done();
  }
  StreamArgs sa{items, S.recs, S.rec_bytes, Tout};
  cudaStream_t st = as_stream(stream);
  DS2_PROF(LM ? "beam_decode_lm_stream" : "beam_decode_stream", st);
  DS2_LAUNCH(beam_decode_stream_kernel<LM>, n_sess, BEAM_THREADS, dyn_smem_bytes(beam_width, C, LM), st, C, probs,
             blank, beam_width, cutoff_top_n, cutoff_prob, labels, timesteps, lengths, scores, n_beams, S.pool, lm, sa);
  return DS2_OK;
}

}  // namespace
}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_beam_decode_workspace_bytes(int B, int T, int C, int beam_width) {
  return beam_workspace_bytes(B, T, beam_width, false);
}

size_t ds2_beam_decode_lm_workspace_bytes(int B, int T, int C, int beam_width) {
  return beam_workspace_bytes(B, T, beam_width, true);
}

int ds2_beam_decode(int B, int T, int C, const float* probs, const int32_t* out_len, int blank, int beam_width,
                    int cutoff_top_n, float cutoff_prob, int32_t* labels, int32_t* timesteps, int32_t* lengths,
                    double* scores, int32_t* n_beams, void* workspace, size_t workspace_bytes, void* stream) {
  return beam_decode_launch<false>("ds2_beam_decode", B, T, C, probs, out_len, blank, beam_width, cutoff_top_n,
                                   cutoff_prob, BeamLm{}, labels, timesteps, lengths, scores, n_beams, workspace,
                                   workspace_bytes, stream);
}

int ds2_beam_decode_lm(int B, int T, int C, const float* probs, const int32_t* out_len, int blank, int beam_width,
                       int cutoff_top_n, float cutoff_prob, const void* lm, int lm_order, double alpha, double beta,
                       int space, int32_t* labels, int32_t* timesteps, int32_t* lengths, double* scores,
                       int32_t* n_beams, void* workspace, size_t workspace_bytes, void* stream) {
  const int rc = lm_check_args("ds2_beam_decode_lm", C, blank, lm, lm_order, space);
  if (rc != DS2_OK) return rc;
  DS2_REQUIRE(std::isfinite(alpha) && std::isfinite(beta), "ds2_beam_decode_lm: alpha=%g, beta=%g not finite", alpha,
              beta);
  BeamLm L;
  L.tables = lm;
  L.order = lm_order;
  L.space = space;
  L.alpha = alpha;
  L.beta = beta;
  return beam_decode_launch<true>("ds2_beam_decode_lm", B, T, C, probs, out_len, blank, beam_width, cutoff_top_n,
                                  cutoff_prob, L, labels, timesteps, lengths, scores, n_beams, workspace,
                                  workspace_bytes, stream);
}

size_t ds2_beam_decode_lm_grid_workspace_bytes(int B, int T, int C, int beam_width, int K) {
  if (B <= 0 || T <= 0 || beam_width <= 0 || C <= 0 || K <= 0) return 0;
  const long long slots = grid_slots((long long)B * K, beam_width, C);
  if (slots <= 0) return 0;
  GridWs w;
  return grid_ws_carve(K, (int)slots, T, beam_width, nullptr, w);
}

int ds2_beam_decode_lm_grid(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                            int beam_width, int cutoff_top_n, float cutoff_prob, const void* lm, int lm_order, int K,
                            const double* pairs, int space, int32_t* labels, int32_t* lengths, void* workspace,
                            size_t workspace_bytes, void* stream) {
  const char* fn = "ds2_beam_decode_lm_grid";
  int rc = lm_check_args(fn, C, blank, lm, lm_order, space);
  if (rc != DS2_OK) return rc;
  rc = beam_check_args(fn, B, T, C, blank, beam_width, cutoff_top_n, cutoff_prob);
  if (rc != DS2_OK) return rc;
  DS2_REQUIRE(K >= 1, "%s: K=%d pairs, need at least 1", fn, K);
  DS2_REQUIRE((long long)B * K < (1ll << 31) - 1, "%s: B*K too large", fn);
  DS2_REQUIRE(probs && labels && lengths && pairs, "%s: null pointer", fn);
  for (int k = 0; k < K; ++k)       // on the host: the kernel never sees a NaN or an infinity
    DS2_REQUIRE(std::isfinite(pairs[2 * k]) && std::isfinite(pairs[2 * k + 1]),
                "%s: pair %d: alpha=%g, beta=%g not finite", fn, k, pairs[2 * k], pairs[2 * k + 1]);
  const long long slots = grid_slots((long long)B * K, beam_width, C);
  DS2_REQUIRE(slots > 0, "%s: occupancy query failed", fn);
  GridWs G;
  const size_t need = grid_ws_carve(K, (int)slots, T, beam_width, workspace, G);
  DS2_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu bytes)", fn, workspace_bytes,
              need);
  BeamLm L;
  L.tables = lm;
  L.order = lm_order;
  L.space = space;
  L.alpha = 0.0;
  L.beta = 0.0;
  cudaStream_t st = as_stream(stream);
  DS2_CHECK_CUDA(cudaMemcpyAsync(G.pairs, pairs, (size_t)K * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
  DS2_PROF("beam_decode_lm_grid", st);
  DS2_LAUNCH(beam_decode_grid_kernel, (int)slots, BEAM_THREADS, dyn_smem_bytes(beam_width, C, true), st, B, K, T, C,
             probs, out_len, blank, beam_width, cutoff_top_n, cutoff_prob, G.pairs, labels, lengths, G.pool, L);
  return DS2_OK;
}

size_t ds2_beam_decode_stream_state_bytes(int max_sessions, int max_frames, int beam_width) {
  if (max_sessions <= 0 || max_frames <= 0 || beam_width <= 0) return 0;
  StreamState S;
  return stream_state_carve(max_sessions, max_frames, beam_width, false, nullptr, S);
}

size_t ds2_beam_decode_lm_stream_state_bytes(int max_sessions, int max_frames, int beam_width) {
  if (max_sessions <= 0 || max_frames <= 0 || beam_width <= 0) return 0;
  StreamState S;
  return stream_state_carve(max_sessions, max_frames, beam_width, true, nullptr, S);
}

int ds2_beam_decode_stream(int n_sess, int C, const float* probs, const int32_t* items, int blank, int beam_width,
                           int cutoff_top_n, float cutoff_prob, int max_sessions, int max_frames, int Tout,
                           int32_t* labels, int32_t* timesteps, int32_t* lengths, double* scores, int32_t* n_beams,
                           void* state, size_t state_bytes, void* stream) {
  return beam_stream_launch<false>("ds2_beam_decode_stream", n_sess, C, probs, items, blank, beam_width, cutoff_top_n,
                                   cutoff_prob, BeamLm{}, max_sessions, max_frames, Tout, labels, timesteps, lengths,
                                   scores, n_beams, state, state_bytes, stream);
}

int ds2_beam_decode_lm_stream(int n_sess, int C, const float* probs, const int32_t* items, int blank, int beam_width,
                              int cutoff_top_n, float cutoff_prob, const void* lm, int lm_order, double alpha,
                              double beta, int space, int max_sessions, int max_frames, int Tout, int32_t* labels,
                              int32_t* timesteps, int32_t* lengths, double* scores, int32_t* n_beams, void* state,
                              size_t state_bytes, void* stream) {
  const int rc = lm_check_args("ds2_beam_decode_lm_stream", C, blank, lm, lm_order, space);
  if (rc != DS2_OK) return rc;
  DS2_REQUIRE(std::isfinite(alpha) && std::isfinite(beta), "ds2_beam_decode_lm_stream: alpha=%g, beta=%g not finite",
              alpha, beta);
  BeamLm L;
  L.tables = lm;
  L.order = lm_order;
  L.space = space;
  L.alpha = alpha;
  L.beta = beta;
  return beam_stream_launch<true>("ds2_beam_decode_lm_stream", n_sess, C, probs, items, blank, beam_width,
                                  cutoff_top_n, cutoff_prob, L, max_sessions, max_frames, Tout, labels, timesteps,
                                  lengths, scores, n_beams, state, state_bytes, stream);
}

}  // extern "C"
