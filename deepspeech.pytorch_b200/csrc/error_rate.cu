// WER / CER edit counts on the device (ds2_error_counts): the numbers validation.py:48-126 (CharErrorRate,
// WordErrorRate; metrics.py here) computes from strings, for K x B hypotheses at once, without moving any label row
// to the host.
//
// Definitions (LABELS-level restatement of `s.replace(' ', '')` and `s.split()`, ' ' being the only whitespace label):
//  - reference b = targets[off_b, off_b + size_b) with the blank labels dropped (GreedyDecoder.convert_to_strings);
//    the hypothesis = its first length labels, as given (the decoders never emit the blank);
//  - characters = the labels other than `space`; words = maximal runs of non-space labels (space = C when the labels
//    have no space: then a non-empty row is one word);
//  - char_edits / word_edits = Levenshtein distance (unit costs) between the character / word sequences; two words are
//    equal only if their label sequences are (a 64-bit hash only filters the comparisons).
//
// Algorithm: Myers' bit-vector edit distance in Hyyroe's block form (the column of the DP over the reference, 64 cells
// per word; vertical deltas Pv / Mv per block; the horizontal delta of the last row of a block carries into the next
// block; the top row grows by one per hypothesis symbol, so block 0 gets hin = +1).  The score is the bottom cell,
// D[m][j] = D[m][j-1] + the horizontal delta at bit (m-1) mod 64 of the last block.  Bits above m in the last block
// only influence higher bits (carries and shifts go upward), so no padding is needed.  One warp per row: the equality
// masks of a block are two ballots over its 64 reference symbols; the block recurrence is warp-uniform.  Pv / Mv live
// in shared memory for references of up to 64 x SH_BLOCKS symbols and in the workspace beyond, so there is no length
// cap.  tests/test_evaluation_host.py restates this recurrence in numpy.
//
// Per utterance, a prep kernel (one warp) finds the target offset, drops blanks and writes the reference's
// characters and its word table (start, length, hash) into the workspace.  Counts are int64; the per-pair sums are
// integer atomics, so their order does not matter.

#include "common.cuh"

namespace ds2 {

namespace {

constexpr int ER_THREADS = 256, ER_WARPS = ER_THREADS / 32;
constexpr int SH_BLOCKS = 64;          // 64-bit blocks of Pv / Mv per warp in shared memory (4096 symbols)

struct RefTables {
  long long* meta;          // per utterance: offset, non-blank length, characters, words
  int* nb;                  // blank-dropped reference labels (at the utterance's target offset)
  int* chars;               // its non-space labels
  int* wstart;              // per word: start in nb, length, hash (at the utterance's target offset)
  int* wlen;
  unsigned long long* whash;
};

__device__ __forceinline__ unsigned long long word_hash_step(unsigned long long h, int label) {
  return (h ^ (unsigned long long)(label + 1)) * 0x100000001b3ull;
}
constexpr unsigned long long HASH0 = 0xcbf29ce484222325ull;

__global__ void __launch_bounds__(ER_THREADS)
ref_prep_kernel(int B, const int64_t* __restrict__ targets, long long n_targets, const int32_t* __restrict__ sizes,
                int blank, int space, RefTables R) {
  const int u = (blockIdx.x * ER_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (u >= B) return;
  long long off = 0;
  for (int v = lane; v < u; v += 32) off += max(sizes[v], 0);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) off += __shfl_xor_sync(0xffffffffu, off, o);
  if (lane != 0) return;
  long long n = max(sizes[u], 0);
  if (off > n_targets) off = n_targets;
  if (off + n > n_targets) n = n_targets - off;       // sizes that overrun the buffer are cut at its end
  int* nb = R.nb + off;
  int* ch = R.chars + off;
  int* ws = R.wstart + off;
  int* wl = R.wlen + off;
  unsigned long long* wh = R.whash + off;
  int j = 0, nc = 0, nw = 0;
  bool in_word = false;
  unsigned long long h = HASH0;
  for (long long i = 0; i < n; ++i) {
    const int x = (int)targets[off + i];
    if (x == blank) continue;
    nb[j] = x;
    if (x == space) {
      if (in_word) { wl[nw] = j - ws[nw]; wh[nw] = h; ++nw; in_word = false; }
    } else {
      ch[nc++] = x;
      if (!in_word) { ws[nw] = j; h = HASH0; in_word = true; }
      h = word_hash_step(h, x);
    }
    ++j;
  }
  if (in_word) { wl[nw] = j - ws[nw]; wh[nw] = h; ++nw; }
  R.meta[4 * u + 0] = off;
  R.meta[4 * u + 1] = j;
  R.meta[4 * u + 2] = nc;
  R.meta[4 * u + 3] = nw;
}

// Myers / Hyyroe over m pattern symbols in nb = ceil(m / 64) blocks; Pv / Mv at P / M (shared or global), the
// whole warp computing the same values and lane 0 storing them
struct BitLev {
  unsigned long long* P;
  unsigned long long* M;
  int m, nb, lane;
  long long score;

  __device__ void init(unsigned long long* P_, unsigned long long* M_, int m_) {
    P = P_; M = M_; m = m_; nb = (m_ + 63) >> 6; lane = threadIdx.x & 31; score = m_;
    for (int w = lane; w < nb; w += 32) { P[w] = ~0ull; M[w] = 0ull; }
    __syncwarp();
  }

  // one hypothesis symbol; eq(w) gives the 64-bit equality mask of block w
  template <class Eq>
  __device__ void step(const Eq& eq) {
    int hin = 1;
    for (int w = 0; w < nb; ++w) {
      unsigned long long Eqm = eq(w);
      const unsigned long long Pv = P[w], Mv = M[w];
      const unsigned long long neg = hin < 0 ? 1ull : 0ull;
      const unsigned long long Xv = Eqm | Mv;
      Eqm |= neg;
      const unsigned long long Xh = (((Eqm & Pv) + Pv) ^ Pv) | Eqm;
      unsigned long long Ph = Mv | ~(Xh | Pv);
      unsigned long long Mh = Pv & Xh;
      const int hb = w == nb - 1 ? ((m - 1) & 63) : 63;
      const int hout = (int)((Ph >> hb) & 1ull) - (int)((Mh >> hb) & 1ull);
      Ph <<= 1;
      Mh <<= 1;
      Mh |= neg;
      Ph |= hin > 0 ? 1ull : 0ull;
      if (lane == 0) {
        P[w] = Mh | ~(Xv | Ph);
        M[w] = Ph & Xv;
      }
      hin = hout;
    }
    score += nb ? hin : 1;     // no pattern: every symbol is an insertion
    __syncwarp();
  }
};

__global__ void __launch_bounds__(ER_THREADS)
error_counts_kernel(int K, int B, int T, const int32_t* __restrict__ labels, const int32_t* __restrict__ lengths,
                    int space, RefTables R, unsigned long long* __restrict__ pm_global, int pm_blocks,
                    long long* __restrict__ row_counts, unsigned long long* __restrict__ pair_counts) {
  __shared__ unsigned long long pm_sh[ER_WARPS][2][SH_BLOCKS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * ER_WARPS + warp;
  if (r >= (long long)K * B) return;
  const int u = (int)(r % B), k = (int)(r / B);
  const long long off = R.meta[4 * u + 0];
  const int mc = (int)R.meta[4 * u + 2], mw = (int)R.meta[4 * u + 3];
  const int* __restrict__ nbv = R.nb + off;
  const int* __restrict__ chars = R.chars + off;
  const int* __restrict__ wstart = R.wstart + off;
  const int* __restrict__ wlen = R.wlen + off;
  const unsigned long long* __restrict__ whash = R.whash + off;
  const int32_t* __restrict__ hyp = labels + r * T;
  const int n = min(max(lengths[r], 0), T);

  unsigned long long *P, *M;
  const int need = (max(mc, mw) + 63) >> 6;
  if (need <= SH_BLOCKS) {
    P = pm_sh[warp][0];
    M = pm_sh[warp][1];
  } else if (need > pm_blocks) {        // a reference longer than max_target_size: no room; marked, not counted
    if (lane == 0 && row_counts)
      for (int q = 0; q < 4; ++q) row_counts[4 * r + q] = -1;
    return;
  } else {
    P = pm_global + (size_t)r * 2 * pm_blocks;
    M = P + pm_blocks;
  }

  // characters: the hypothesis' non-space labels against the reference's
  BitLev lev;
  lev.init(P, M, mc);
  for (int i = 0; i < n; ++i) {
    const int x = hyp[i];
    if (x == space) continue;
    lev.step([&](int w) {
      const int j0 = 64 * w + lane, j1 = j0 + 32;
      const unsigned lo = __ballot_sync(0xffffffffu, j0 < mc && chars[j0] == x);
      const unsigned hi = __ballot_sync(0xffffffffu, j1 < mc && chars[j1] == x);
      return ((unsigned long long)hi << 32) | lo;
    });
  }
  const long long char_edits = lev.score;

  // words
  lev.init(P, M, mw);
  int pos = 0;
  for (;;) {
    while (pos < n && hyp[pos] == space) ++pos;
    if (pos >= n) break;
    const int s = pos;
    unsigned long long h = HASH0;
    while (pos < n && hyp[pos] != space) h = word_hash_step(h, hyp[pos++]);
    const int len = pos - s;
    auto same = [&](int j) {
      if (j >= mw || wlen[j] != len || whash[j] != h) return false;
      const int* a = nbv + wstart[j];
      for (int t = 0; t < len; ++t)
        if (a[t] != hyp[s + t]) return false;
      return true;
    };
    lev.step([&](int w) {
      const int j0 = 64 * w + lane;
      const unsigned lo = __ballot_sync(0xffffffffu, same(j0));
      const unsigned hi = __ballot_sync(0xffffffffu, same(j0 + 32));
      return ((unsigned long long)hi << 32) | lo;
    });
  }
  const long long word_edits = lev.score;

  if (lane == 0) {
    const long long c[4] = {char_edits, mc, word_edits, mw};
    if (row_counts)
      for (int q = 0; q < 4; ++q) row_counts[4 * r + q] = c[q];
    if (pair_counts)
      for (int q = 0; q < 4; ++q) atomicAdd(pair_counts + 4 * k + q, (unsigned long long)c[q]);
  }
}

size_t pm_global_blocks(int max_target_size) {
  const int need = (max(max_target_size, 0) + 63) / 64;
  return need > SH_BLOCKS ? (size_t)need : 0;
}

// Workspace of ds2_error_counts (bytes; with a base, also the addresses), each buffer 256-byte aligned: the reference
// tables, meta (B,4) | nb | chars | wstart | wlen | whash (n_targets each, at least 1) | only when a reference is
// longer than the shared-memory blocks hold: the Myers bit vectors (K x B rows of 2 x pm_global_blocks)
struct CountsWs { RefTables R; unsigned long long* pm; };
size_t error_counts_carve(int K, int B, long long n_targets, int max_target_size, void* base, CountsWs& w) {
  const size_t n = (size_t)(n_targets > 0 ? n_targets : 1), pm_blocks = pm_global_blocks(max_target_size);
  size_t off = 0;
  w.R.meta = carve<long long>(base, off, (size_t)B * 4 * 8);
  w.R.nb = carve<int>(base, off, n * 4);
  w.R.chars = carve<int>(base, off, n * 4);
  w.R.wstart = carve<int>(base, off, n * 4);
  w.R.wlen = carve<int>(base, off, n * 4);
  w.R.whash = carve<unsigned long long>(base, off, n * 8);
  w.pm = pm_blocks ? carve<unsigned long long>(base, off, (size_t)K * B * 2 * pm_blocks * 8) : nullptr;
  return off;
}

}  // namespace
}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_error_counts_workspace_bytes(int K, int B, int64_t n_targets, int max_target_size) {
  if (K <= 0 || B <= 0 || n_targets < 0) return 0;
  CountsWs w;
  return error_counts_carve(K, B, n_targets, max_target_size, nullptr, w);
}

int ds2_error_counts(int K, int B, int T, const int32_t* labels, const int32_t* lengths, const int64_t* targets,
                     int64_t n_targets, const int32_t* target_sizes, int max_target_size, int blank, int space,
                     int64_t* row_counts, int64_t* pair_counts, void* workspace, size_t workspace_bytes,
                     void* stream) {
  const char* fn = "ds2_error_counts";
  DS2_REQUIRE(K >= 1 && B >= 1 && T >= 1, "%s: bad shape K=%d B=%d T=%d", fn, K, B, T);
  DS2_REQUIRE((long long)K * B * T < (1ll << 62), "%s: K*B*T too large", fn);
  DS2_REQUIRE(n_targets >= 0 && max_target_size >= 0, "%s: n_targets=%lld, max_target_size=%d", fn,
              (long long)n_targets, max_target_size);
  DS2_REQUIRE(labels && lengths && target_sizes && (targets || n_targets == 0), "%s: null pointer", fn);
  CountsWs W;
  const size_t need = error_counts_carve(K, B, n_targets, max_target_size, workspace, W);
  DS2_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu bytes)", fn, workspace_bytes,
              need);
  const int pm_blocks = (int)pm_global_blocks(max_target_size);
  cudaStream_t st = as_stream(stream);
  DS2_PROF("error_counts", st);
  DS2_LAUNCH(ref_prep_kernel, cdiv((long long)B, ER_WARPS), ER_THREADS, 0, st, B, targets, (long long)n_targets,
             target_sizes, blank, space, W.R);
  DS2_LAUNCH(error_counts_kernel, cdiv((long long)K * B, ER_WARPS), ER_THREADS, 0, st, K, B, T, labels, lengths,
             space, W.R, W.pm, pm_blocks, reinterpret_cast<long long*>(row_counts),
             reinterpret_cast<unsigned long long*>(pair_counts));
  return DS2_OK;
}

}  // extern "C"
