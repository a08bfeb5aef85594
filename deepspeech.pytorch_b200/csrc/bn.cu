// BatchNorm over the rows of a (rows, F) matrix: the SequenceWise(BatchNorm1d) of the reference
// (model.py:18-33, :86 per RNN layer, :196 in the fc head).  Statistics are over ALL T*B rows,
// padded rows included (SURVEY.md §8c quirks).  bn_finalize also finalizes the conv front-end's BatchNorm2d, whose
// sums the conv epilogues accumulate (conv_frontend.cu).
//
// Forward statistics: E[x^2] - E[x]^2 from raw sums (fp32 partials, flushed into double) cancels when a feature's mean
// is large against its spread.  Saturated LSTM units feed the next layer such features (the sum of the two directions
// of h sits near +-2 with a tiny spread: for mean 10 and std 0.001 the variance is 1e-8 of E[x^2], below fp32
// rounding); in the front-end the conv bias moves a channel's mean.  So the statistics pass also sums (x - K) and
// (x - K)^2 with a pivot K per feature: here the feature's first row (summed in double per element, the FP64 adds
// hidden under the loads), in the front-end the channel's conv bias (known before the convolution runs).  From those,
// mean = K + S1/n and var = S2/n - (S1/n)^2, where S2/n stays within a small factor of (S1/n)^2.  bn_finalize_kernel
// takes them for a feature whose E[x^2] exceeds max_cancel * var and keeps the raw result everywhere else, so a
// well-conditioned feature gets exactly the bits it always had: a last-bit change in the statistics, carried through
// fp16 operand copies and AdamW, moves the loss of the benchmark step by 0.1 % after 11 steps.  The thresholds
// (common.cuh): RAW_MAX_CANCEL = 256 for the rows, where the raw variance error below it is about 1e-6 relative,
// typical, and every feature of the benchmark's model is below it (E[x^2] / var <= 18); BN2D_RAW_MAX_CANCEL = 16 for
// the front-end, where the raw variance below it is within a few 1e-7 of float64.
#include "common.cuh"

namespace ds2 {

// blockDim = (32, 8): 32 consecutive features x 8 row lanes; grid = (ceil(F/32), row_chunks)
__global__ void bn_colsum_kernel(int rows, int F, const float* __restrict__ a, const float* __restrict__ b,
                                 const float* __restrict__ pivot, double* __restrict__ sums) {
  // sums[0..F) += sum_r a ; sums[F..2F) += sum_r a*b   (b == a for the forward statistics)
  // with a pivot (forward statistics): sums[2F..3F) += sum_r (a - K), sums[3F..4F) += sum_r (a - K)^2, K = pivot[f]
  __shared__ double s[4][8][33];
  int f = blockIdx.x * 32 + threadIdx.x;
  int rows_per = cdiv_dev(rows, gridDim.y);
  int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float p1 = 0.f, p2 = 0.f;
  double d1 = 0.0, d2 = 0.0, e1 = 0.0, e2 = 0.0;
  int cnt = 0;
  if (f < F) {
    const double k = pivot ? (double)pivot[f] : 0.0;
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      float va = a[(size_t)r * F + f], vb = b[(size_t)r * F + f];
      p1 += va;
      p2 = fmaf(va, vb, p2);
      if (pivot) {
        const double d = (double)va - k;
        e1 += d;
        e2 = fma(d, d, e2);
      }
      if (++cnt == 64) {  // flush the fp32 partials into double every 64 rows
        d1 += p1; d2 += p2; p1 = p2 = 0.f; cnt = 0;
      }
    }
    d1 += p1; d2 += p2;
  }
  s[0][threadIdx.y][threadIdx.x] = d1;
  s[1][threadIdx.y][threadIdx.x] = d2;
  s[2][threadIdx.y][threadIdx.x] = e1;
  s[3][threadIdx.y][threadIdx.x] = e2;
  __syncthreads();
  if (threadIdx.y == 0 && f < F) {
    for (int i = 1; i < 8; ++i) { d1 += s[0][i][threadIdx.x]; d2 += s[1][i][threadIdx.x]; }
    atomicAdd(&sums[f], d1);
    atomicAdd(&sums[F + f], d2);
    if (pivot) {
      for (int i = 1; i < 8; ++i) { e1 += s[2][i][threadIdx.x]; e2 += s[3][i][threadIdx.x]; }
      atomicAdd(&sums[2 * F + f], e1);
      atomicAdd(&sums[3 * F + f], e2);
    }
  }
}

// sums: sum x [F], sum x^2 [F]; piv_sums: sum (x - K) [F], sum (x - K)^2 [F], K = pivot[f]
__global__ void bn_finalize_kernel(int F, double count, const double* __restrict__ sums,
                                   const double* __restrict__ piv_sums, const float* __restrict__ pivot,
                                   double max_cancel, float* __restrict__ rmean, float* __restrict__ rvar,
                                   int training, float momentum, float eps, float* __restrict__ mean_invstd) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float mean, var;
  if (training) {
    double m = sums[f] / count;
    double v = sums[F + f] / count - m * m;
    if (v < 0.0) v = 0.0;
    const double ms = piv_sums[f] / count;  // mean - K
    double vs = piv_sums[F + f] / count - ms * ms;
    if (vs < 0.0) vs = 0.0;
    if (!(sums[F + f] / count <= max_cancel * vs)) {  // the raw sums cancel: take the pivoted ones
      m = (double)pivot[f] + ms;
      v = vs;
    }
    mean = (float)m;
    var = (float)v;
    double unbiased = count > 1.0 ? v * count / (count - 1.0) : v;
    rmean[f] = (1.f - momentum) * rmean[f] + momentum * mean;
    rvar[f] = (1.f - momentum) * rvar[f] + momentum * (float)unbiased;
  } else {
    mean = rmean[f];
    var = rvar[f];
  }
  mean_invstd[f] = mean;
  mean_invstd[F + f] = rsqrtf(var + eps);
}

__global__ void bn_apply_kernel(size_t total, int F, const float* __restrict__ x, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ mean_invstd,
                                float* __restrict__ y, float* __restrict__ xhat) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    int f = (int)(i % F);
    float h = (x[i] - mean_invstd[f]) * mean_invstd[F + f];
    if (xhat) xhat[i] = h;
    if (y) y[i] = fmaf(h, gamma[f], beta[f]);
  }
}

__global__ void bn_bwd_apply_kernel(size_t total, int F, double inv_count, const float* __restrict__ xhat,
                                    const float* __restrict__ gamma, const float* __restrict__ mean_invstd,
                                    const float* __restrict__ dy, const double* __restrict__ sums,
                                    float* __restrict__ dx) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    int f = (int)(i % F);
    float mdy = (float)(sums[f] * inv_count), mdyx = (float)(sums[F + f] * inv_count);
    dx[i] = gamma[f] * mean_invstd[F + f] * (dy[i] - mdy - xhat[i] * mdyx);
  }
}

__global__ void bn_bwd_params_kernel(int F, const double* __restrict__ sums, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  dbeta[f] = (float)sums[f];
  dgamma[f] = (float)sums[F + f];
}

static int colsum_grid_y(int rows) {
  int g = rows / 256;
  return g < 1 ? 1 : (g > 64 ? 64 : g);
}

// blocks of 256 threads for the grid-stride elementwise kernels: about 4 entries per thread, at most 16 blocks per SM
static int elementwise_blocks(size_t total) {
  const size_t blocks = (total + 1023) / 1024;
  return blocks < 1 ? 1 : (blocks > 132 * 16 ? 132 * 16 : (int)blocks);
}

int bn_finalize(int F, double count, const double* sums, const double* piv_sums, const float* pivot,
                double max_cancel, float* rmean, float* rvar, int training, float momentum, float eps,
                float* mean_invstd, cudaStream_t st) {
  DS2_LAUNCH(bn_finalize_kernel, cdiv(F, 128), 128, 0, st, F, count, sums, piv_sums, pivot, max_cancel, rmean, rvar,
             training, momentum, eps, mean_invstd);
  return DS2_OK;
}

int bn_bwd_params(int F, const double* sums, float* dgamma, float* dbeta, cudaStream_t st) {
  DS2_LAUNCH(bn_bwd_params_kernel, cdiv(F, 128), 128, 0, st, F, sums, dgamma, dbeta);
  return DS2_OK;
}

int bn_rows_fwd(int rows, int F, const float* x, const float* gamma, const float* beta, float* rmean, float* rvar,
                int training, float momentum, float eps, float* y, float* xhat, float* mean_invstd,
                double* ws_sums, cudaStream_t st) {
  if (training) {
    DS2_CHECK_CUDA(cudaMemsetAsync(ws_sums, 0, sizeof(double) * 4 * F, st));
    dim3 grid(cdiv(F, 32), colsum_grid_y(rows)), block(32, 8);
    DS2_LAUNCH(bn_colsum_kernel, grid, block, 0, st, rows, F, x, x, x /* pivot: row 0 */, ws_sums);
  }
  int rc = bn_finalize(F, (double)rows, ws_sums, ws_sums + 2 * F, x, RAW_MAX_CANCEL, rmean, rvar, training, momentum,
                       eps, mean_invstd, st);
  if (rc) return rc;
  return bn_rows_reapply(rows, F, x, gamma, beta, mean_invstd, y, xhat, st);
}

int bn_rows_reapply(int rows, int F, const float* x, const float* gamma, const float* beta,
                    const float* mean_invstd, float* y, float* xhat, cudaStream_t st) {
  const size_t total = (size_t)rows * F;
  DS2_LAUNCH(bn_apply_kernel, elementwise_blocks(total), 256, 0, st, total, F, x, gamma, beta, mean_invstd, y, xhat);
  return DS2_OK;
}

int bn_rows_bwd(int rows, int F, const float* xhat, const float* gamma, const float* mean_invstd, const float* dy,
                float* dx, float* dgamma, float* dbeta, double* ws_sums, cudaStream_t st) {
  DS2_CHECK_CUDA(cudaMemsetAsync(ws_sums, 0, sizeof(double) * 2 * F, st));
  dim3 grid(cdiv(F, 32), colsum_grid_y(rows)), block(32, 8);
  DS2_LAUNCH(bn_colsum_kernel, grid, block, 0, st, rows, F, dy, xhat, nullptr, ws_sums);
  int rc = bn_bwd_params(F, ws_sums, dgamma, dbeta, st);
  if (rc) return rc;
  const size_t total = (size_t)rows * F;
  DS2_LAUNCH(bn_bwd_apply_kernel, elementwise_blocks(total), 256, 0, st, total, F, 1.0 / (double)rows, xhat, gamma,
             mean_invstd, dy, ws_sums, dx);
  return DS2_OK;
}

}  // namespace ds2
