// CTC forced alignment: the Viterbi path of each utterance's target through the extended-label lattice the CTC loss
// sums over (ctc.cu), i.e. the max-plus twin of the alpha recursion plus backpointers and a backtrack.
//   (log-softmax rows: ctc.cu's kernel, when the input are logits)
//   ctc_align_kernel  one CTA per utterance, states across threads, the two DP rows in shared memory (fp64), one
//                     __syncthreads per time step; 2-bit backpointers to global memory; then thread 0 walks the path
//                     back and writes the spans (and, on request, the per-frame labels and log-probs).
// Recursion (fp64, fixed order: bit-repeatable, no atomics):
//   score_t(s) = max(score_{t-1}(s), score_{t-1}(s-1), [score_{t-1}(s-2) if ext[s] != blank && ext[s] != ext[s-2]])
//                + (double)lp[t][ext[s]],   ties prefer s, then s-1, then s-2;  at t = 0 only states 0 and 1 are live;
//   the path ends in S-1 if score(S-1) >= score(S-2), else in S-2.
#include <cuda_pipeline.h>
#include <math_constants.h>

#include "common.cuh"

namespace ds2 {

constexpr int ALIGN_MAX_THREADS = 1024;
constexpr int ALIGN_LP_BUDGET = 8192;   // bytes of shared memory for the two staged blocks of log-prob rows

// Rows t of one utterance's log-probs staged per block: as many as fit the budget, at most 32
inline int align_rows_per_block(int C) {
  int r = ALIGN_LP_BUDGET / (2 * 4 * C);
  return r < 1 ? 1 : (r > 32 ? 32 : r);
}

// Dynamic shared memory: double rows[2][Smax + 2] | float lp_blk[2][TCH * C] | uint16 ext[Smax]
inline size_t align_smem_bytes(int Smax, int C) {
  return 2 * ((size_t)Smax + 2) * 8 + 2 * (size_t)align_rows_per_block(C) * C * 4 + align_up((size_t)Smax * 2, 16);
}

// Backpointer words: per (utterance, frame), one uint2 per group of 32 states; bit (s % 32) of .x / .y is bit 0 / 1
// of the step taken into state s (0: stay, 1: from s-1, 2: from s-2)
__host__ __device__ inline size_t align_groups(int Smax) { return ((size_t)Smax + 31) / 32; }

__global__ void __launch_bounds__(ALIGN_MAX_THREADS)
ctc_align_kernel(int T, int B, int C, int Smax, int TCH, const float* __restrict__ lp,
                 const int64_t* __restrict__ targets, const long long* __restrict__ tgt_off,
                 const int32_t* __restrict__ in_len, const int32_t* __restrict__ tgt_len, int max_tgt_len, int blank,
                 uint2* __restrict__ bp, int32_t* __restrict__ frame_labels, float* __restrict__ frame_lp,
                 int32_t* __restrict__ spans, double* __restrict__ path_score) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int W = Smax + 2;  // row: [0,1] = -inf guards, states at [2, 2+S)
  double* rows = reinterpret_cast<double*>(smem_raw);
  float* lp_blk = reinterpret_cast<float*>(rows + 2 * W);
  unsigned short* ext = reinterpret_cast<unsigned short*>(lp_blk + 2 * TCH * C);
  __shared__ int end_state;
  const int b = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
  const int Tb = min(max(in_len[b], 0), T), Lb = tgt_len[b];
  const size_t G = align_groups(Smax);
  const size_t row_stride = (size_t)B * C;
  const float* lpb = lp + (size_t)b * C;

  // A target length outside [0, max_tgt_len] or a label outside [0, C) leaves the utterance unaligned.
  bool ok = Lb >= 0 && Lb <= max_tgt_len;
  const int S = ok ? 2 * Lb + 1 : 1;
  const int64_t* tg = targets + (ok && Lb > 0 ? tgt_off[b] : 0);
  for (int r = tid; r < S; r += nthr) {
    long long l = (r & 1) ? tg[r >> 1] : blank;
    if (l < 0 || l >= C) ok = false;
    ext[r] = (unsigned short)l;
  }
  for (int i = tid; i < 2 * W; i += nthr) rows[i] = -CUDART_INF;
  ok = __syncthreads_and(ok);

  int cur = 0;
  if (ok && Tb > 0) {
    // Log-prob rows are staged in blocks of TCH frames through cp.async, one block ahead of the recursion.
    auto stage = [&](int blk) {
      float* dst = lp_blk + (blk & 1) * TCH * C;
      const int t0 = blk * TCH;
      for (int i = tid; i < TCH * C; i += nthr) {
        const int t = t0 + i / C;
        if (t < Tb) __pipeline_memcpy_async(dst + i, lpb + (size_t)t * row_stride + i % C, 4);
      }
      __pipeline_commit();
    };
    stage(0);
    stage(1);
    const int nk = (S + nthr - 1) / nthr;
    const int warp = tid / 32, lane = tid % 32, nwarps = nthr / 32;
    for (int blk = 0; blk * TCH < Tb; ++blk) {
      __pipeline_wait_prior(1);
      __syncthreads();
      const float* lpc = lp_blk + (blk & 1) * TCH * C;
      for (int i = 0; i < TCH; ++i) {
        const int t = blk * TCH + i;
        if (t >= Tb) break;  // block-uniform
        const double* prev = rows + cur * W + 2;
        double* next = rows + (cur ^ 1) * W + 2;
        uint2* bpt = bp + ((size_t)b * T + t) * G;
        for (int k = 0; k < nk; ++k) {  // uniform trip count: every lane takes part in the ballots
          const int r = tid + k * nthr;
          unsigned d = 0;
          if (r < S) {
            const int l = ext[r];
            double best;
            if (t == 0) {
              best = (r < 2) ? 0.0 : -CUDART_INF;
            } else {
              best = prev[r];
              const double a1 = prev[r - 1];  // prev[-1], prev[-2] are the -inf guards
              if (a1 > best) { best = a1; d = 1; }
              if (r >= 2 && l != blank && l != ext[r - 2]) {
                const double a2 = prev[r - 2];
                if (a2 > best) { best = a2; d = 2; }
              }
            }
            next[r] = best + (double)lpc[i * C + l];
          }
          const unsigned lo = __ballot_sync(0xffffffffu, d & 1), hi = __ballot_sync(0xffffffffu, d >> 1);
          const int g = warp + k * nwarps;
          if (lane == 0 && t > 0 && g * 32 < S) bpt[g] = make_uint2(lo, hi);
        }
        __syncthreads();
        cur ^= 1;
      }
      stage(blk + 2);  // into the block just consumed: every thread is past the step's barrier
    }
  }

  // ---- end state and score
  if (tid == 0) {
    double score;
    int s_end = -1;
    if (!ok) {
      score = -CUDART_INF;
    } else if (Tb == 0) {
      score = (Lb == 0) ? 0.0 : -CUDART_INF;
    } else {
      const double* last = rows + cur * W + 2;
      s_end = S - 1;
      if (S > 1 && !(last[S - 1] >= last[S - 2])) s_end = S - 2;
      score = last[s_end];
      if (!(score > -CUDART_INF)) s_end = -1;
    }
    path_score[b] = score;
    end_state = s_end;
  }
  __syncthreads();
  const int s_end = end_state;
  const bool aligned = ok && (s_end >= 0 || (Tb == 0 && Lb == 0));
  const int t_from = aligned ? Tb : 0;           // frames written as -1 / 0 by all threads
  const int k_from = aligned ? Lb : 0;           // spans written as -1
  if (frame_labels)
    for (int t = t_from + tid; t < T; t += nthr) frame_labels[(size_t)b * T + t] = -1;
  if (frame_lp)
    for (int t = t_from + tid; t < T; t += nthr) frame_lp[(size_t)b * T + t] = 0.f;
  for (int k = k_from + tid; k < max_tgt_len; k += nthr)
    reinterpret_cast<int2*>(spans)[(size_t)b * max_tgt_len + k] = make_int2(-1, -1);
  if (!aligned || s_end < 0 || tid != 0) return;

  // ---- backtrack (thread 0): state s at frame t; a run of one state [t, end) closes where the step leaves it
  int s = s_end, end = Tb;
  for (int t = Tb - 1; t >= 0; --t) {
    int sp = -1;
    if (t > 0) {
      const uint2 w = bp[((size_t)b * T + t) * G + (s >> 5)];
      const int bit = s & 31;
      sp = s - (int)(((w.x >> bit) & 1u) | (((w.y >> bit) & 1u) << 1));
    }
    const int l = ext[s];
    if (frame_labels) frame_labels[(size_t)b * T + t] = l;
    if (frame_lp) frame_lp[(size_t)b * T + t] = lpb[(size_t)t * row_stride + l];
    if (sp != s) {
      if (s & 1) reinterpret_cast<int2*>(spans)[(size_t)b * max_tgt_len + (s >> 1)] = make_int2(t, end);
      end = t;
    }
    s = sp;
  }
}

// Workspace of ds2_ctc_align (bytes; with a base, also the addresses), each buffer 256-byte aligned:
//   log-softmax lp (T,B,C) fp32 | backpointers (B,T,ceil(Smax/32)) uint2 | target offsets (B) int64
struct AlignWs {
  float* lp;
  uint2* bp;
  long long* off;
};
static size_t align_ws_carve(int T, int B, int C, int max_tgt_len, void* base, AlignWs& w) {
  const size_t TB = (size_t)T * B;
  size_t off = 0;
  w.lp = carve<float>(base, off, TB * C * 4);
  w.bp = carve<uint2>(base, off, TB * align_groups(2 * max_tgt_len + 1) * 8);
  w.off = carve<long long>(base, off, (size_t)B * 8);
  return off;
}

}  // namespace ds2

extern "C" {

size_t ds2_ctc_align_workspace_bytes(int T, int B, int C, int max_tgt_len) {
  if (T <= 0 || B <= 0 || C <= 0 || max_tgt_len < 0) return 0;
  ds2::AlignWs w;
  return ds2::align_ws_carve(T, B, C, max_tgt_len, nullptr, w);
}

int ds2_ctc_align(int T, int B, int C, const float* x, int apply_log_softmax, const int64_t* targets,
                  const int32_t* in_len, const int32_t* tgt_len, int max_tgt_len, int blank, int32_t* frame_labels,
                  float* frame_log_probs, int32_t* token_spans, double* path_score, void* workspace,
                  size_t workspace_bytes, void* stream) {
  using namespace ds2;
  DS2_REQUIRE(T > 0 && B > 0 && C > 0 && max_tgt_len >= 0 && blank >= 0 && blank < C,
              "ds2_ctc_align: bad shape (T=%d B=%d C=%d max_tgt_len=%d blank=%d)", T, B, C, max_tgt_len, blank);
  DS2_REQUIRE(max_tgt_len <= DS2_CTC_ALIGN_MAX_TGT_LEN,
              "ds2_ctc_align: max_tgt_len %d exceeds the supported maximum DS2_CTC_ALIGN_MAX_TGT_LEN = %d (the two "
              "fp64 DP rows of 2L+1 states live in shared memory)", max_tgt_len, DS2_CTC_ALIGN_MAX_TGT_LEN);
  DS2_REQUIRE(C <= DS2_CTC_ALIGN_MAX_CLASSES, "ds2_ctc_align: C = %d exceeds the supported maximum "
              "DS2_CTC_ALIGN_MAX_CLASSES = %d", C, DS2_CTC_ALIGN_MAX_CLASSES);
  DS2_REQUIRE(x && in_len && tgt_len && path_score && (max_tgt_len == 0 || (targets && token_spans)),
              "ds2_ctc_align: null input or output pointer");
  DS2_REQUIRE(apply_log_softmax == 0 || apply_log_softmax == 1, "ds2_ctc_align: apply_log_softmax must be 0 or 1");
  AlignWs Wk;
  const size_t need = align_ws_carve(T, B, C, max_tgt_len, workspace, Wk);
  DS2_REQUIRE(workspace && workspace_bytes >= need, "ds2_ctc_align: workspace null or too small (%zu < %zu bytes)",
              workspace_bytes, need);
  cudaStream_t st = as_stream(stream);
  const int Smax = 2 * max_tgt_len + 1;
  int threads = (Smax + 31) / 32 * 32;
  if (threads > ALIGN_MAX_THREADS) threads = ALIGN_MAX_THREADS;
  if (threads < 64) threads = 64;
  const size_t smem = align_smem_bytes(Smax, C);
  static DeviceOnce smem_set;
  if (smem_set.first()) {
    DS2_CHECK_CUDA(cudaFuncSetAttribute(ctc_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)align_smem_bytes(2 * DS2_CTC_ALIGN_MAX_TGT_LEN + 1,
                                                              DS2_CTC_ALIGN_MAX_CLASSES)));
    smem_set.done();
  }
  DS2_PROF("ctc_align", st);
  const float* lp = x;
  if (apply_log_softmax) {
    if (int rc = ctc_log_softmax(T * B, C, x, Wk.lp, st)) return rc;
    lp = Wk.lp;
  }
  if (int rc = ctc_target_offsets(B, tgt_len, Wk.off, st)) return rc;
  DS2_LAUNCH(ctc_align_kernel, B, threads, smem, st, T, B, C, Smax, align_rows_per_block(C), lp, targets, Wk.off,
             in_len, tgt_len, max_tgt_len, blank, Wk.bp, frame_labels, frame_log_probs, token_spans, path_score);
  return DS2_OK;
}

}  // extern "C"
