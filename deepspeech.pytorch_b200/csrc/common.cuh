// Shared host/device helpers for libds2_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/ds2_b200.h"

namespace ds2 {

void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
int precision();
inline bool tensor_core_mode() { return precision() != DS2_PREC_FP32; }   // TF32 or precision-16: wgmma kernels
inline bool f16_gemm_mode() { return precision() == DS2_PREC_F16; }       // fp16 operands for the dense RNN GEMMs

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Host-side "once per device" latch: cudaFuncSetAttribute and the device attributes are per device, so a plain
// function-local static would leave the second GPU of a process without its shared-memory opt-in.
inline int current_device() {
  int d = 0;
  (void)cudaGetDevice(&d);
  return d & 63;
}
struct DeviceOnce {
  std::atomic<unsigned long long> mask{0};
  bool first() const { return !((mask.load(std::memory_order_acquire) >> current_device()) & 1ull); }
  void done() { mask.fetch_or(1ull << current_device(), std::memory_order_release); }
};
int device_sm_count();   // SM count of the current device (cached per device)

// A row class of the tensor-core 32->32 convolution (conv_tc_run in conv_tc.cu): its output rows d in [0, R_out) read
// the vertical taps j in [0, J), input row row_mul * d + row_off + j * row_step with tap matrix w_off + j * w_step, and
// land in output row out_row_mul * d + out_row_off.  The forward is one class; the data gradient two (even / odd rows).
struct ConvRows {
  int R_out, J, row_off, w_off, out_row_off;
};

// A tensor-core-mode call that had to take the one-launch-per-time-step FFMA kernels (shape not eligible for the
// persistent sweeps): counted and reported once per shape on stderr, never silent.
void note_fallback(const char* what, int rnn, int T, int B, int H, int D);

// Optional side stream (ds2_set_side_stream): deferred work whose results nobody on the main stream needs before
// ds2_join_side_stream.  Workspaces read by side work are protected by per-workspace events.
extern std::atomic<void*> g_side_stream;
int side_wait_for_workspace(const void* ws, cudaStream_t main);
int side_fork(cudaStream_t main, cudaStream_t side);
int side_mark_workspace(const void* ws, cudaStream_t side);

#define DS2_CHECK_CUDA(expr)                                                             \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ds2::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return DS2_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)

#define DS2_REQUIRE(cond, ...)                      \
  do {                                              \
    if (!(cond)) {                                  \
      ds2::set_error(__VA_ARGS__);                  \
      return DS2_ERR_INVALID;                       \
    }                                               \
  } while (0)

// Launch bookkeeping: every kernel launch of the library goes through this.
#define DS2_LAUNCH(kernel, grid, block, smem, stream, ...)                \
  do {                                                                    \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);           \
    ds2::g_launches.fetch_add(1, std::memory_order_relaxed);              \
    DS2_CHECK_CUDA(cudaGetLastError());                                   \
  } while (0)

// Device-time ranges (cudaEvent pairs on the launching stream), off unless ds2_prof_enable(1).
void prof_begin(const char* tag, cudaStream_t st);
void prof_end(cudaStream_t st);
struct ProfRange {
  cudaStream_t st;
  ProfRange(const char* tag, cudaStream_t s) : st(s) { prof_begin(tag, s); }
  ~ProfRange() { prof_end(st); }
};
#define DS2_PROF(tag, st) ds2::ProfRange _prof_range_##__LINE__(tag, st)

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
#ifdef __CUDACC__
__device__ __forceinline__ int cdiv_dev(int a, int b) { return (a + b - 1) / b; }
#endif
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// The next `bytes` (256-aligned) of a workspace layout at offset `off`, or null when the base is null (sizing only)
template <typename T>
inline T* carve(void* base, size_t& off, size_t bytes) {
  T* at = base ? reinterpret_cast<T*>(static_cast<char*>(base) + off) : nullptr;
  off += align_up(bytes, 256);
  return at;
}

#ifdef __CUDACC__
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

// ---- internal cross-file entry points -------------------------------------------------------
// C[M,N] = alpha*op(A)op(B) + beta*C (row-major, fp32 FFMA kernel; any shape/stride)
// (ws: room for the split-K partial slabs, gemm_simt_workspace_bytes; without it the kernel makes one pass over K)
int gemm_simt(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
              int ldb, float beta, float* C, int ldc, cudaStream_t st, void* ws = nullptr, size_t ws_bytes = 0);
size_t gemm_simt_workspace_bytes(int M, int N, int K);
// wgmma TF32 kernel.  Returns 1 if the shape is not eligible (caller falls back to gemm_simt).
int gemm_tc(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
            int ldb, float beta, float* C, int ldc, void* ws, size_t ws_bytes, cudaStream_t st);
size_t gemm_tc_workspace_bytes(int transA, int transB, int M, int N, int K);
// precision-16 GEMM: fp16 K-major operands, fp32 accumulation / output (gemm_tc.cu); 1 = not eligible
int gemm_tc_f16(int M, int N, int K, float alpha, const void* A16, int lda, const void* B16, int ldb, float beta,
                float* C, int ldc, const float* alpha_dev, cudaStream_t st);
// fp32 -> fp16 operand copies (convert.cu)
int f32_to_f16_rows(int rows, int cols, const float* in, size_t ld_in, void* out, size_t ld_out, const float* scale_dev,
                    cudaStream_t st);
int f32_to_f16_transpose(int rows, int cols, const float* in, size_t ld_in, void* out, size_t ld_out, void* outT,
                         size_t ld_outT, const float* scale_dev, cudaStream_t st);
int pow2_scale_for(int rows, int cols, const float* x, size_t ld, unsigned int* absmax_ws, float* scale, int top,
                   cudaStream_t st);

// BatchNorm over rows of a (rows, F) matrix (BatchNorm1d under SequenceWise, model.py:18-33,86,196)
// training: batch stats (biased var) -> mean/invstd, running stats updated; else running stats.
// y = (x-mean)*invstd*gamma+beta ; xhat optionally stored.
int bn_rows_fwd(int rows, int F, const float* x, const float* gamma, const float* beta, float* rmean, float* rvar,
                int training, float momentum, float eps, float* y, float* xhat, float* mean_invstd /*2F*/,
                double* ws_sums /*4F doubles*/, cudaStream_t st);
// y / xhat again from saved statistics (backward recomputation)
int bn_rows_reapply(int rows, int F, const float* x, const float* gamma, const float* beta,
                    const float* mean_invstd, float* y, float* xhat, cudaStream_t st);
int transpose(int R, int C, const float* in, float* out, cudaStream_t st);
int transpose_strided(int R, int C, const float* in, size_t ldi, float* out, size_t ldo, cudaStream_t st);
// dx = gamma*invstd*(dy - mean(dy) - xhat*mean(dy*xhat)); dgamma, dbeta written.
int bn_rows_bwd(int rows, int F, const float* xhat, const float* gamma, const float* mean_invstd, const float* dy,
                float* dx, float* dgamma, float* dbeta, double* ws_sums /*2F doubles*/, cudaStream_t st);
// The BatchNorm steps the conv front-end's BatchNorm2d shares with bn_rows_fwd / bn_rows_bwd.
// mean_invstd (2F) of F features over `count` values each; training: from the raw sums (sum x, sum x^2) or, where
// E[x^2] > max_cancel * var, from the pivoted ones (sum (x - K), sum (x - K)^2, K = pivot[f]), running stats updated;
// else from the running stats.  The cancellation thresholds of the two BatchNorms: bn.cu's header says why each.
constexpr double RAW_MAX_CANCEL = 256.0, BN2D_RAW_MAX_CANCEL = 16.0;
int bn_finalize(int F, double count, const double* sums, const double* piv_sums, const float* pivot,
                double max_cancel, float* rmean, float* rvar, int training, float momentum, float eps,
                float* mean_invstd, cudaStream_t st);
// dbeta = sums[0..F), dgamma = sums[F..2F) (the backward's sum dy, sum dy*xhat)
int bn_bwd_params(int F, const double* sums, float* dgamma, float* dbeta, cudaStream_t st);
// CTC helpers (ctc.cu), shared by the loss and the forced alignment (ctc_align.cu):
// fp32 log-softmax of `rows` rows of C values; the exclusive prefix sum of the target lengths (offsets into the flat
// targets)
int ctc_log_softmax(int rows, int C, const float* logits, float* lp, cudaStream_t st);
int ctc_target_offsets(int B, const int32_t* tgt_len, long long* off, cudaStream_t st);

}  // namespace ds2
