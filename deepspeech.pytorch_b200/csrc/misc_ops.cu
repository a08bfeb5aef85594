// Small blocks of the path: Lookahead (+Hardtanh), fc head (BN1d + Linear [+softmax]), greedy
// decode, and the fused clip + AdamW / SGD-Nesterov step on flat buffers.
#include <math_constants.h>

#include "common.cuh"

namespace ds2 {

// ------------------------------------------------------------------ Lookahead  (model.py:105-130,189-193)
// x,y (T, R) with R = B*H rows flattened; channel c = r % H;  y = clamp(sum_k w[c,k] x[t+k], 0, 20)
__global__ void lookahead_fwd_kernel(int T, int R, int H, int ctx, const float* __restrict__ x,
                                     const float* __restrict__ w, float* __restrict__ y) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)T * R) return;
  int t = (int)(i / R), r = (int)(i % R), c = r % H;
  float acc = 0.f;
  for (int k = 0; k < ctx && t + k < T; ++k) acc = fmaf(w[c * ctx + k], x[(size_t)(t + k) * R + r], acc);
  y[i] = fminf(fmaxf(acc, 0.f), 20.f);
}

// dz = dy * 1[0 < pre < 20] (torch hardtanh_backward is strict); dx[t] = sum_k w[c,k] dz[t-k]
__global__ void lookahead_dz_kernel(int T, int R, int H, int ctx, const float* __restrict__ x,
                                    const float* __restrict__ w, const float* __restrict__ dy,
                                    float* __restrict__ dz) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)T * R) return;
  int t = (int)(i / R), r = (int)(i % R), c = r % H;
  float acc = 0.f;
  for (int k = 0; k < ctx && t + k < T; ++k) acc = fmaf(w[c * ctx + k], x[(size_t)(t + k) * R + r], acc);
  dz[i] = (acc > 0.f && acc < 20.f) ? dy[i] : 0.f;
}

__global__ void lookahead_dx_kernel(int T, int R, int H, int ctx, const float* __restrict__ w,
                                    const float* __restrict__ dz, float* __restrict__ dx) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)T * R) return;
  int t = (int)(i / R), r = (int)(i % R), c = r % H;
  float acc = 0.f;
  for (int k = 0; k < ctx && t - k >= 0; ++k) acc = fmaf(w[c * ctx + k], dz[(size_t)(t - k) * R + r], acc);
  dx[i] = acc;
}

// dw[c,k] = sum_{t,b} dz[t,b,c] x[t+k,b,c]; grid (ceil(H/32), ctx, chunks), block (32, 8)
__global__ void lookahead_dw_kernel(int T, int B, int H, int ctx, const float* __restrict__ x,
                                    const float* __restrict__ dz, float* __restrict__ dw) {
  __shared__ float red[8][33];
  int c = blockIdx.x * 32 + threadIdx.x, k = blockIdx.y;
  int rows = (T - k) * B;  // (t,b) pairs with t+k < T
  int per = cdiv_dev(rows, gridDim.z);
  int r0 = blockIdx.z * per, r1 = min(rows, r0 + per);
  float acc = 0.f;
  if (c < H)
    for (int r = r0 + threadIdx.y; r < r1; r += 8)
      acc = fmaf(dz[(size_t)r * H + c], x[((size_t)r + (size_t)k * B) * H + c], acc);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < H) {
    for (int i = 1; i < 8; ++i) acc += red[i][threadIdx.x];
    atomicAdd(&dw[c * ctx + k], acc);
  }
}

// ------------------------------------------------------------------ softmax rows (InferenceBatchSoftmax)
__global__ void softmax_rows_kernel(int rows, int C, float* __restrict__ x) {
  int row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= rows) return;
  float* p = x + (size_t)row * C;
  float m = -CUDART_INF_F;
  for (int c = lane; c < C; c += 32) m = fmaxf(m, p[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += expf(p[c] - m);
  s = warp_sum(s);
  for (int c = lane; c < C; c += 32) p[c] = expf(p[c] - m) / s;
}

__global__ void affine_rows_kernel(size_t total, int F, const float* __restrict__ xhat, const float* __restrict__ g,
                                   const float* __restrict__ b, float* __restrict__ y) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    int f = (int)(i % F);
    y[i] = fmaf(xhat[i], g[f], b[f]);
  }
}

// ------------------------------------------------------------------ greedy decode (decoder.py:144-181)
// one thread per utterance (sequential collapse); argmax ties -> lowest index like torch.max
__global__ void greedy_decode_kernel(int B, int T, int C, const float* __restrict__ probs,
                                     const int32_t* __restrict__ out_len, int blank, int32_t* __restrict__ labels,
                                     int32_t* __restrict__ offsets, int32_t* __restrict__ counts) {
  int b = blockIdx.x;
  extern __shared__ int am[];  // argmax per frame
  int n = out_len ? min(out_len[b], T) : T;
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const float* p = probs + ((size_t)b * T + t) * C;
    int best = 0;
    float bv = p[0];
    for (int c = 1; c < C; ++c)
      if (p[c] > bv) { bv = p[c]; best = c; }
    am[t] = best;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int cnt = 0;
    for (int t = 0; t < n; ++t) {
      int c = am[t];
      if (c != blank && !(t != 0 && c == am[t - 1])) {
        labels[(size_t)b * T + cnt] = c;
        offsets[(size_t)b * T + cnt] = t;
        ++cnt;
      }
    }
    counts[b] = cnt;
  }
}

// ------------------------------------------------------------------ optimizer (model.py:273-297 + clip 400)
// Squared gradient norm, bit-repeatable: a fixed grid of NORM_PARTS blocks (every block's share of the vector and its
// summation order depend on n only) writes one double partial each to ws[1 + block]; sumsq_final_kernel adds them in
// order into ws[0].  (The 256-byte optimizer workspace holds the 31 partials.)
constexpr int NORM_PARTS = 31, NORM_THREADS = 1024;
__global__ void __launch_bounds__(NORM_THREADS) sumsq_kernel(int64_t n, const float* __restrict__ g,
                                                             double* __restrict__ ws) {
  __shared__ double red[NORM_THREADS / 32];
  double acc = 0.0;
  const int64_t stride = (int64_t)NORM_PARTS * NORM_THREADS, tid = (int64_t)blockIdx.x * NORM_THREADS + threadIdx.x;
  const bool vec = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const int64_t n4 = vec ? n / 4 : 0;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  int64_t i = tid;
  for (; i + 3 * stride < n4; i += 4 * stride) {      // four independent 16-byte loads in flight per thread
    const float4 a = g4[i], b = g4[i + stride], c = g4[i + 2 * stride], d = g4[i + 3 * stride];
    float part = a.x * a.x;
    part = fmaf(a.y, a.y, part); part = fmaf(a.z, a.z, part); part = fmaf(a.w, a.w, part);
    part = fmaf(b.x, b.x, part); part = fmaf(b.y, b.y, part); part = fmaf(b.z, b.z, part); part = fmaf(b.w, b.w, part);
    part = fmaf(c.x, c.x, part); part = fmaf(c.y, c.y, part); part = fmaf(c.z, c.z, part); part = fmaf(c.w, c.w, part);
    part = fmaf(d.x, d.x, part); part = fmaf(d.y, d.y, part); part = fmaf(d.z, d.z, part); part = fmaf(d.w, d.w, part);
    acc += part;
  }
  for (; i < n4; i += stride) {
    const float4 a = g4[i];
    acc += (double)fmaf(a.w, a.w, fmaf(a.z, a.z, fmaf(a.y, a.y, a.x * a.x)));
  }
  for (int64_t j = 4 * n4 + tid; j < n; j += stride) acc += (double)g[j] * g[j];
  acc = warp_sum_d(acc);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = warp_sum_d(red[threadIdx.x]);
    if (threadIdx.x == 0) ws[1 + blockIdx.x] = v;
  }
}
__global__ void sumsq_final_kernel(double* __restrict__ ws) {
  double s = 0.0;
  for (int i = 0; i < NORM_PARTS; ++i) s += ws[1 + i];
  ws[0] = s;
}
static int launch_sumsq(int64_t n, const float* g, double* ws, cudaStream_t st) {
  DS2_LAUNCH(sumsq_kernel, NORM_PARTS, NORM_THREADS, 0, st, n, g, ws);
  DS2_LAUNCH(sumsq_final_kernel, 1, 1, 0, st, ws);
  return DS2_OK;
}

__device__ __forceinline__ float clip_coef(const double* sumsq, float grad_scale, float max_norm, float* norm_out) {
  float total = sqrtf((float)(*sumsq)) * grad_scale;
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) *norm_out = total;
  float coef = 1.f;
  if (max_norm > 0.f) {
    coef = max_norm / (total + 1e-6f);   // torch clip_grad_norm_
    coef = coef > 1.f ? 1.f : coef;
  }
  return coef * grad_scale;
}

__device__ __forceinline__ void adamw_one(float& pi, float gi, float& mi, float& vi, float s, float lr, float b1,
                                          float b2, float eps, float wd, float bc1, float bc2_sqrt) {
  gi *= s;
  pi *= (1.f - lr * wd);                               // decoupled weight decay
  mi = b1 * mi + (1.f - b1) * gi;
  vi = b2 * vi + (1.f - b2) * gi * gi;
  const float denom = sqrtf(vi) / bc2_sqrt + eps;
  pi -= (lr / bc1) * (mi / denom);
}

// 7 streams of 4 bytes per parameter (read p, g, m, v; write p, m, v): 16-byte accesses, the flat buffers are
// 16-byte aligned (checked by the caller), the n % 4 tail is done element-wise by the last threads.
__global__ void adamw_kernel(int64_t n, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, float lr, float b1, float b2, float eps, float wd, float bc1,
                             float bc2_sqrt, float grad_scale, float max_norm, const double* __restrict__ sumsq,
                             float* __restrict__ norm_out, int vec) {
  const float s = clip_coef(sumsq, grad_scale, max_norm, norm_out);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (int64_t)gridDim.x * blockDim.x;
  const int64_t n4 = vec ? n / 4 : 0;
  for (int64_t i = tid; i < n4; i += nthr) {
    float4 pv = reinterpret_cast<float4*>(p)[i], mv = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    adamw_one(pv.x, gv.x, mv.x, vv.x, s, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    adamw_one(pv.y, gv.y, mv.y, vv.y, s, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    adamw_one(pv.z, gv.z, mv.z, vv.z, s, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    adamw_one(pv.w, gv.w, mv.w, vv.w, s, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  for (int64_t i = 4 * n4 + tid; i < n; i += nthr) {
    float pi = p[i], mi = m[i], vi = v[i];
    adamw_one(pi, g[i], mi, vi, s, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
}

__global__ void sgd_nesterov_kernel(int64_t n, float* __restrict__ p, const float* __restrict__ g,
                                    float* __restrict__ buf, float lr, float mom, float wd, int first,
                                    float grad_scale, float max_norm, const double* __restrict__ sumsq,
                                    float* __restrict__ norm_out) {
  const float s = clip_coef(sumsq, grad_scale, max_norm, norm_out);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i] * s + wd * p[i];
    float bi = first ? gi : mom * buf[i] + gi;
    buf[i] = bi;
    p[i] -= lr * (gi + mom * bi);
  }
}

}  // namespace ds2

extern "C" {
using namespace ds2;

int ds2_lookahead_fwd(int T, int B, int H, int ctx, const float* x, const float* w, float* y, void* stream) {
  DS2_REQUIRE(T > 0 && B > 0 && H > 0 && ctx > 0, "ds2_lookahead_fwd: bad shape");
  size_t total = (size_t)T * B * H;
  DS2_LAUNCH(lookahead_fwd_kernel, cdiv(total, 256), 256, 0, as_stream(stream), T, B * H, H, ctx, x, w, y);
  return DS2_OK;
}

int ds2_lookahead_bwd(int T, int B, int H, int ctx, const float* x, const float* w, const float* dy, float* dz,
                      float* dx, float* dw, void* stream) {
  DS2_REQUIRE(T > 0 && B > 0 && H > 0 && ctx > 0 && dz && dz != dx, "ds2_lookahead_bwd: bad arguments");
  cudaStream_t st = as_stream(stream);
  size_t total = (size_t)T * B * H;
  DS2_LAUNCH(lookahead_dz_kernel, cdiv(total, 256), 256, 0, st, T, B * H, H, ctx, x, w, dy, dz);
  DS2_CHECK_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)H * ctx, st));
  int chunks = (T * B) / 512;
  chunks = chunks < 1 ? 1 : (chunks > 32 ? 32 : chunks);
  DS2_LAUNCH(lookahead_dw_kernel, dim3(cdiv(H, 32), ctx, chunks), dim3(32, 8), 0, st, T, B, H, ctx, x, dz, dw);
  DS2_LAUNCH(lookahead_dx_kernel, cdiv(total, 256), 256, 0, st, T, B * H, H, ctx, w, dz, dx);
  return DS2_OK;
}

size_t ds2_fc_head_workspace_bytes(int rows, int H, int C) {
  return align_up((size_t)rows * H * 4, 256) + align_up((size_t)2 * H * 8, 256) +
         ds2_gemm_workspace_bytes(1, 0, C, H, rows) + 4096;
}

int ds2_fc_head_fwd(int rows, int H, int C, const float* x, const float* g, const float* b, float* rmean,
                    float* rvar, const float* w, int training, float momentum, float eps, int softmax,
                    float* logits, float* xhat, float* stats, void* ws, size_t ws_bytes, void* stream) {
  DS2_REQUIRE(rows > 0 && H > 0 && C > 0, "ds2_fc_head_fwd: bad shape");
  DS2_REQUIRE(ws_bytes >= ds2_fc_head_workspace_bytes(rows, H, C), "ds2_fc_head_fwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  Arena ar(ws, ws_bytes);
  DS2_PROF("fc_fwd", st);
  float* xbn = ar.take<float>((size_t)rows * H);
  double* sums = ar.take<double>(2 * (size_t)H);
  int r = bn_rows_fwd(rows, H, x, g, b, rmean, rvar, training, momentum, eps, xbn, xhat, stats, sums, st);
  if (r) return r;
  r = ds2_gemm(0, 1, rows, C, H, 1.f, xbn, H, w, H, 0.f, logits, C, ar.base + ar.off, ar.cap - ar.off, stream);
  if (r) return r;
  if (softmax) DS2_LAUNCH(softmax_rows_kernel, cdiv(rows, 8), 256, 0, st, rows, C, logits);
  return DS2_OK;
}

int ds2_fc_head_bwd(int rows, int H, int C, const float* g, const float* b, const float* w, const float* xhat,
                    const float* stats, const float* dlogits, float* dx, float* dg, float* db, float* dw, void* ws,
                    size_t ws_bytes, void* stream) {
  DS2_REQUIRE(rows > 0 && H > 0 && C > 0, "ds2_fc_head_bwd: bad shape");
  DS2_REQUIRE(ws_bytes >= ds2_fc_head_workspace_bytes(rows, H, C), "ds2_fc_head_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  Arena ar(ws, ws_bytes);
  DS2_PROF("fc_bwd", st);
  float* tmp = ar.take<float>((size_t)rows * H);
  double* sums = ar.take<double>(2 * (size_t)H);
  void* gws = ar.base + ar.off;
  size_t gws_bytes = ar.cap - ar.off;
  size_t total = (size_t)rows * H;
  int blocks = (int)((total + 1023) / 1024);
  blocks = blocks > 132 * 16 ? 132 * 16 : blocks;
  // dW = dlogits^T (C x rows) . xbn (rows x H)
  DS2_LAUNCH(affine_rows_kernel, blocks, 256, 0, st, total, H, xhat, g, b, tmp);
  int r = ds2_gemm(1, 0, C, H, rows, 1.f, dlogits, C, tmp, H, 0.f, dw, H, gws, gws_bytes, stream);
  if (r) return r;
  // dxbn = dlogits (rows x C) . W (C x H)
  r = ds2_gemm(0, 0, rows, H, C, 1.f, dlogits, C, w, H, 0.f, tmp, H, gws, gws_bytes, stream);
  if (r) return r;
  return bn_rows_bwd(rows, H, xhat, g, stats, tmp, dx, dg, db, sums, st);
}

int ds2_greedy_decode(int B, int T, int C, const float* probs, const int32_t* out_len, int blank, int32_t* labels,
                      int32_t* offsets, int32_t* counts, void* stream) {
  DS2_REQUIRE(B > 0 && T > 0 && C > 0, "ds2_greedy_decode: bad shape");
  size_t smem = (size_t)T * 4;
  if (smem > 48 * 1024)
    DS2_CHECK_CUDA(cudaFuncSetAttribute(greedy_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DS2_LAUNCH(greedy_decode_kernel, B, 256, smem, as_stream(stream), B, T, C, probs, out_len, blank, labels, offsets,
             counts);
  return DS2_OK;
}

size_t ds2_optim_workspace_bytes(void) { return (1 + NORM_PARTS) * sizeof(double); }   // 256

int ds2_adamw_step(int64_t n, float* p, const float* g, float* m, float* v, float lr, float beta1, float beta2,
                   float eps, float wd, int step, float grad_scale, float max_norm, float* grad_norm_out,
                   void* norm_ws, void* stream) {
  DS2_REQUIRE(n >= 0 && step >= 1 && norm_ws, "ds2_adamw_step: bad arguments");
  cudaStream_t st = as_stream(stream);
  double* sumsq = static_cast<double*>(norm_ws);
  DS2_PROF("optim", st);
  int blocks = (int)((n + 4095) / 4096);
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  int rc = launch_sumsq(n, g, sumsq, st);
  if (rc) return rc;
  float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  const int vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                    reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  DS2_LAUNCH(adamw_kernel, blocks, 256, 0, st, n, p, g, m, v, lr, beta1, beta2, eps, wd, bc1, sqrtf(bc2),
             grad_scale, max_norm, sumsq, grad_norm_out, vec);
  return DS2_OK;
}

int ds2_sgd_nesterov_step(int64_t n, float* p, const float* g, float* buf, float lr, float momentum, float wd,
                          int first_step, float grad_scale, float max_norm, float* grad_norm_out, void* norm_ws,
                          void* stream) {
  DS2_REQUIRE(n >= 0 && norm_ws, "ds2_sgd_nesterov_step: bad arguments");
  cudaStream_t st = as_stream(stream);
  double* sumsq = static_cast<double*>(norm_ws);
  int blocks = (int)((n + 4095) / 4096);
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  int rc = launch_sumsq(n, g, sumsq, st);
  if (rc) return rc;
  DS2_LAUNCH(sgd_nesterov_kernel, blocks, 256, 0, st, n, p, g, buf, lr, momentum, wd, first_step, grad_scale,
             max_norm, sumsq, grad_norm_out);
  return DS2_OK;
}

}  // extern "C"
