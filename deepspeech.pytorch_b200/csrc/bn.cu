// BatchNorm over the rows of a (rows, F) matrix: the SequenceWise(BatchNorm1d) of the reference
// (model.py:18-33, :86 per RNN layer, :196 in the fc head).  Statistics are over ALL T*B rows,
// padded rows included (SURVEY.md §8c quirks).  Column sums are accumulated in double to avoid
// E[x^2]-E[x]^2 cancellation.
#include "common.cuh"

namespace ds2 {

// blockDim = (32, 8): 32 consecutive features x 8 row lanes; grid = (ceil(F/32), row_chunks)
__global__ void bn_colsum_kernel(int rows, int F, const float* __restrict__ a, const float* __restrict__ b,
                                 double* __restrict__ sums) {
  // sums[0..F) += sum_r a ; sums[F..2F) += sum_r a*b   (b == a for the forward statistics)
  __shared__ double s1[8][33], s2[8][33];
  int f = blockIdx.x * 32 + threadIdx.x;
  int rows_per = cdiv_dev(rows, gridDim.y);
  int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float p1 = 0.f, p2 = 0.f;
  double d1 = 0.0, d2 = 0.0;
  int cnt = 0;
  if (f < F) {
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      float va = a[(size_t)r * F + f], vb = b[(size_t)r * F + f];
      p1 += va;
      p2 = fmaf(va, vb, p2);
      if (++cnt == 64) {  // flush the fp32 partials into double every 64 rows
        d1 += p1; d2 += p2; p1 = p2 = 0.f; cnt = 0;
      }
    }
    d1 += p1; d2 += p2;
  }
  s1[threadIdx.y][threadIdx.x] = d1;
  s2[threadIdx.y][threadIdx.x] = d2;
  __syncthreads();
  if (threadIdx.y == 0 && f < F) {
    for (int i = 1; i < 8; ++i) { d1 += s1[i][threadIdx.x]; d2 += s2[i][threadIdx.x]; }
    atomicAdd(&sums[f], d1);
    atomicAdd(&sums[F + f], d2);
  }
}

__global__ void bn_finalize_kernel(int F, double count, const double* __restrict__ sums, float* __restrict__ rmean,
                                   float* __restrict__ rvar, int training, float momentum, float eps,
                                   float* __restrict__ mean_invstd) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float mean, var;
  if (training) {
    double m = sums[f] / count;
    double v = sums[F + f] / count - m * m;
    if (v < 0.0) v = 0.0;
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

int bn_rows_fwd(int rows, int F, const float* x, const float* gamma, const float* beta, float* rmean, float* rvar,
                int training, float momentum, float eps, float* y, float* xhat, float* mean_invstd,
                double* ws_sums, cudaStream_t st) {
  if (training) {
    DS2_CHECK_CUDA(cudaMemsetAsync(ws_sums, 0, sizeof(double) * 2 * F, st));
    dim3 grid(cdiv(F, 32), colsum_grid_y(rows)), block(32, 8);
    DS2_LAUNCH(bn_colsum_kernel, grid, block, 0, st, rows, F, x, x, ws_sums);
  }
  DS2_LAUNCH(bn_finalize_kernel, cdiv(F, 128), 128, 0, st, F, (double)rows, ws_sums, rmean, rvar, training, momentum,
             eps, mean_invstd);
  size_t total = (size_t)rows * F;
  int blocks = (int)((total + 1023) / 1024);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  DS2_LAUNCH(bn_apply_kernel, blocks, 256, 0, st, total, F, x, gamma, beta, mean_invstd, y, xhat);
  return DS2_OK;
}

int bn_rows_reapply(int rows, int F, const float* x, const float* gamma, const float* beta,
                    const float* mean_invstd, float* y, float* xhat, cudaStream_t st) {
  size_t total = (size_t)rows * F;
  int blocks = (int)((total + 1023) / 1024);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  DS2_LAUNCH(bn_apply_kernel, blocks, 256, 0, st, total, F, x, gamma, beta, mean_invstd, y, xhat);
  return DS2_OK;
}

int bn_rows_bwd(int rows, int F, const float* xhat, const float* gamma, const float* mean_invstd, const float* dy,
                float* dx, float* dgamma, float* dbeta, double* ws_sums, cudaStream_t st) {
  DS2_CHECK_CUDA(cudaMemsetAsync(ws_sums, 0, sizeof(double) * 2 * F, st));
  dim3 grid(cdiv(F, 32), colsum_grid_y(rows)), block(32, 8);
  DS2_LAUNCH(bn_colsum_kernel, grid, block, 0, st, rows, F, dy, xhat, ws_sums);
  DS2_LAUNCH(bn_bwd_params_kernel, cdiv(F, 128), 128, 0, st, F, ws_sums, dgamma, dbeta);
  size_t total = (size_t)rows * F;
  int blocks = (int)((total + 1023) / 1024);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  DS2_LAUNCH(bn_bwd_apply_kernel, blocks, 256, 0, st, total, F, 1.0 / (double)rows, xhat, gamma, mean_invstd, dy,
             ws_sums, dx);
  return DS2_OK;
}

}  // namespace ds2
