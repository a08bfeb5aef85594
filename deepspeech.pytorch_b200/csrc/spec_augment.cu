// Input pipeline: SpecAugment on the padded spectrogram batch, draw for draw the reference's `spec_augment`
// (deepspeech_pytorch/loader/spec_augment.py:48-115, sparse_image_warp.py:88-410, its defaults: W = 5, one frequency
// mask of up to 26 rows, one time mask of up to 69 frames).  The random numbers come from the caller
// (Ds2SpecAugDraws); the arithmetic that depends on the data runs here, per utterance of its own width T.
//
// Kernel 1 (spec_augment_setup_kernel), one thread per utterance: reads the control point's time coordinate
// p = in[u, F/2, idx] (the reference uses the spectrogram's VALUE there), forms c = (F/2, fp32(p + d)) and
// fx = fp32(c1 - p) in fp32 as the reference does, and solves the order-2 polyharmonic system
//     [[A, b^T], [b, Z]] [w; v] = [fx; 0],   b = (c0, c1, 1),   A = phi(|c - c|^2) = 0
// in double with partial pivoting.  Only the x column is solved: the y-flow's right-hand side is zero, so the
// reference's y-flow is exactly 0 and every output row reads its own input row (the last row: rows F-2, F-1).  It
// stores w, v (rounded to fp32, the reference's solve is fp32), |c|^2 and the grid sum of
// cross_squared_distance_matrix (sparse_image_warp.py:197 sums x^2 over ALL query points, not per point): exact in
// int64, rounded to fp32.
//
// Kernel 2 (spec_augment_warp_kernel), one output element per thread, consecutive threads on consecutive frames:
// the dense x-flow in fp32 in the reference's operation order (explicit __f*_rn so that no contraction reorders it),
// the clamped bilinear sample, both masks and the zero padding.  No atomics: results are bit-repeatable.
#include <math_constants.h>

#include "common.cuh"

namespace ds2 {

namespace sa {
constexpr int THREADS = 256;   // warp kernel: frames per CTA
constexpr int MIN_T = 11;      // random.randrange(5, T - 5) needs T > 10
struct Params {                // per utterance, in the workspace
  float w, v0, v1, v2;         // spline weight and linear terms of the x-flow
  float grid_sum, c_norm2;     // fp32(sum over the (F, T) grid of j^2 + i^2), fp32(c0^2 + c1^2)
  float c0, c1;                // control point (row, frame)
  int ok;                      // 0: frames / draws out of range -> the utterance's frames are written as NaN
  int pad[3];
};
}  // namespace sa

__global__ void spec_augment_setup_kernel(int n_utts, int F, int Tmax, const float* __restrict__ in,
                                          const int32_t* __restrict__ frames,
                                          const Ds2SpecAugDraws* __restrict__ draws, sa::Params* __restrict__ prm) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_utts) return;
  const int T = frames[u];
  const Ds2SpecAugDraws dr = draws[u];
  sa::Params P = {};
  P.ok = T >= sa::MIN_T && T <= Tmax && dr.idx >= 0 && dr.idx < T;
  if (!P.ok) {
    prm[u] = P;
    return;
  }
  // spec_augment.py:52-62: y = F // 2, point_to_warp = spec[0][y][idx], dest = (y, point + dist)
  const float p = in[((size_t)u * F + F / 2) * Tmax + dr.idx];
  const float c0 = (float)(F / 2);
  const float c1 = __fadd_rn(p, (float)dr.d);
  const float fx = __fsub_rn(c1, p);                  // dest - src: not exactly d
  // sparse_image_warp.py:150-180: lhs = [[A, c0, c1, 1], [c0, Z], [c1, Z], [1, Z]], rhs = (fx, 0, 0, 0)
  double M[4][5] = {{0.0, c0, c1, 1.0, fx},
                    {c0, dr.Z[0], dr.Z[1], dr.Z[2], 0.0},
                    {c1, dr.Z[3], dr.Z[4], dr.Z[5], 0.0},
                    {1.0, dr.Z[6], dr.Z[7], dr.Z[8], 0.0}};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    // partial pivoting with compile-time row indices (keeps M in registers): row k ends up holding the largest
    // |M[r][k]|, r >= k
#pragma unroll
    for (int r = k + 1; r < 4; ++r) {
      const bool sw = fabs(M[r][k]) > fabs(M[k][k]);
#pragma unroll
      for (int c = 0; c < 5; ++c) {
        const double a = M[k][c], b = M[r][c];
        M[k][c] = sw ? b : a;
        M[r][c] = sw ? a : b;
      }
    }
#pragma unroll
    for (int r = k + 1; r < 4; ++r) {
      const double m = M[r][k] / M[k][k];
#pragma unroll
      for (int c = k; c < 5; ++c) M[r][c] -= m * M[k][c];
    }
  }
  double x[4];
#pragma unroll
  for (int k = 3; k >= 0; --k) {
    double s = M[k][4];
#pragma unroll
    for (int c = k + 1; c < 4; ++c) s -= M[k][c] * x[c];
    x[k] = s / M[k][k];
  }
  P.w = (float)x[0];
  P.v0 = (float)x[1];
  P.v1 = (float)x[2];
  P.v2 = (float)x[3];
  // sum_{j<F, i<T} (j^2 + i^2) = T sum j^2 + F sum i^2, exact in int64 (5.5e10 at F = 161, T = 1000)
  const long long sj = (long long)(F - 1) * F * (2 * F - 1) / 6, si = (long long)(T - 1) * T * (2 * T - 1) / 6;
  P.grid_sum = (float)(T * sj + F * si);
  P.c_norm2 = __fadd_rn(__fmul_rn(c0, c0), __fmul_rn(c1, c1));
  P.c0 = c0;
  P.c1 = c1;
  prm[u] = P;
}

__global__ void __launch_bounds__(sa::THREADS) spec_augment_warp_kernel(
    int F, int Tmax, const float* __restrict__ in, const int32_t* __restrict__ frames,
    const Ds2SpecAugDraws* __restrict__ draws, const sa::Params* __restrict__ prm, float* __restrict__ out) {
  const int u = blockIdx.z, j = blockIdx.y, i = blockIdx.x * sa::THREADS + threadIdx.x;
  if (i >= Tmax) return;
  const int T = frames[u];
  float* dst = out + ((size_t)u * F + j) * Tmax + i;
  const Ds2SpecAugDraws& dr = draws[u];
  if (i >= T || (j >= dr.f0 && j < dr.f0 + dr.f) || (i >= dr.t0 && i < dr.t0 + dr.t)) {   // padding, masks
    *dst = 0.f;
    return;
  }
  const sa::Params P = prm[u];
  if (!P.ok) {
    *dst = CUDART_NAN_F;
    return;
  }
  const float fj = (float)j, fi = (float)i;
  // cross_squared_distance_matrix (:197-203): (sum x^2 - 2 x.c) + |c|^2; phi (:225): 0.5 * r * log(max(r, 1e-10))
  const float xc = __fadd_rn(__fmul_rn(fj, P.c0), __fmul_rn(fi, P.c1));
  const float r = __fadd_rn(__fsub_rn(P.grid_sum, __fmul_rn(2.f, xc)), P.c_norm2);
  const float phi = __fmul_rn(__fmul_rn(0.5f, r), logf(fmaxf(r, 1e-10f)));
  // apply_interpolation (:255-266): rbf_term + linear_term
  const float lin = __fadd_rn(__fadd_rn(__fmul_rn(fj, P.v0), __fmul_rn(fi, P.v1)), P.v2);
  const float flow = __fadd_rn(__fmul_rn(phi, P.w), lin);
  // dense_image_warp (:306) + interpolate_bilinear (:357-410) on the utterance's own width T
  const float q = __fsub_rn(fi, flow);
  const float fl = fminf(fmaxf(0.f, floorf(q)), (float)(T - 2));
  const float ax = fminf(fmaxf(0.f, __fsub_rn(q, fl)), 1.f);
  const int ix = (int)fl;
  const int fy = j < F - 2 ? j : F - 2;
  const float ay = j > F - 2 ? 1.f : 0.f;             // j - floor(j): 1 only on the last row
  const float* r0 = in + ((size_t)u * F + fy) * Tmax + ix;
  const float* r1 = r0 + Tmax;
  const float tl = __ldg(r0), tr = __ldg(r0 + 1), bl = __ldg(r1), br = __ldg(r1 + 1);
  const float top = __fadd_rn(__fmul_rn(ax, __fsub_rn(tr, tl)), tl);
  const float bot = __fadd_rn(__fmul_rn(ax, __fsub_rn(br, bl)), bl);
  *dst = __fadd_rn(__fmul_rn(ay, __fsub_rn(bot, top)), top);
}

}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_spec_augment_workspace_bytes(int n_utts) {
  return align_up((size_t)(n_utts > 0 ? n_utts : 0) * sizeof(sa::Params), 256);
}

int ds2_spec_augment(int n_utts, int F, int Tmax, const float* in, const int32_t* frames,
                     const Ds2SpecAugDraws* draws, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  DS2_REQUIRE(n_utts > 0 && n_utts <= 65535, "spec_augment: n_utts %d out of range [1, 65535]", n_utts);
  DS2_REQUIRE(F >= 2 && F <= 65535, "spec_augment: F %d out of range [2, 65535]", F);
  DS2_REQUIRE(Tmax >= sa::MIN_T, "spec_augment: Tmax %d < %d (random.randrange(5, T - 5) needs T > 10)", Tmax,
              sa::MIN_T);
  DS2_REQUIRE(in && frames && draws && out && workspace, "spec_augment: null argument");
  const size_t n = (size_t)n_utts * F * Tmax;
  DS2_REQUIRE(out + n <= in || in + n <= out, "spec_augment: in and out overlap");
  DS2_REQUIRE(workspace_bytes >= ds2_spec_augment_workspace_bytes(n_utts), "spec_augment: workspace too small");
  cudaStream_t st = as_stream(stream);
  sa::Params* prm = static_cast<sa::Params*>(workspace);
  DS2_LAUNCH(spec_augment_setup_kernel, cdiv(n_utts, 32), 32, 0, st, n_utts, F, Tmax, in, frames, draws, prm);
  DS2_LAUNCH(spec_augment_warp_kernel, dim3(cdiv(Tmax, sa::THREADS), F, n_utts), sa::THREADS, 0, st, F, Tmax, in,
             frames, draws, prm, out);
  return DS2_OK;
}

}  // extern "C"
