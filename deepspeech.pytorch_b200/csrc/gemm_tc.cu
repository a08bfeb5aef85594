// wgmma TF32 / fp16 GEMM:  C[M,N] = alpha * A[M,K] . B[N,K]^T + beta * C   (both operands K-major).
//
//   warp 0       TMA producer: cp.async.bulk.tensor 2-D tiles (128B swizzle) of A (128 x 32 fp32) and
//                B (BN x 32 fp32) into a 6-stage (BN = 128) or 4-stage (BN = 256) shared-memory ring, mbarrier
//                complete_tx signalling
//   warps 4..11  two MMA warpgroups: wgmma.mma_async m64nBNk8 (tf32) x4 per stage on their 64-row half of
//                the A tile, fp32 accumulators in registers; the epilogue stores them (alpha / beta) to global
//
// Operands that are not K-major in memory (transA / !transB) are first transposed into the workspace.
// Shapes the kernel does not take (tiny or unaligned) return 1 and the caller uses the FFMA GEMM.
#include <stdio.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace ds2 {

// ---- tensor maps ----------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
// TFLOAT32 makes the TMA unit round fp32 -> tf32 (nearest) while copying into shared memory: measured
// bit-identical error statistics to cuBLAS TF32; plain FLOAT32 would let the MMA truncate (2.6x the
// rms error and a -7e-4 relative bias on same-sign data).
static constexpr CUtensorMapDataType g_tmap_dtype = CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;

static int load_encode() {
  if (g_encode) return DS2_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  DS2_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return DS2_ERR_CUDA;
  }
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return DS2_OK;
}

static int make_tmap_2d_sw(CUtensorMap* out, const float* base, int rows, int cols, int ld, int box_rows, int box_cols,
                           CUtensorMapSwizzle sw);
int make_tmap_2d(CUtensorMap* out, const float* base, int rows, int cols, int ld, int box_rows, int box_cols) {
  return make_tmap_2d_sw(out, base, rows, cols, ld, box_rows, box_cols, CU_TENSOR_MAP_SWIZZLE_128B);
}
static int make_tmap_2d_sw(CUtensorMap* out, const float* base, int rows, int cols, int ld, int box_rows, int box_cols,
                           CUtensorMapSwizzle sw) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, g_tmap_dtype, 2, const_cast<float*>(base), gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(2d rows=%d cols=%d ld=%d box=%dx%d base=%p) failed: %d", rows, cols, ld,
              box_rows, box_cols, (const void*)base, (int)r);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

static int make_tmap_3d_sw(CUtensorMap* out, const float* base, int d0, int d1, int d2, size_t stride1, size_t stride2,
                           int box0, int box1, int box2, CUtensorMapSwizzle sw);
int make_tmap_3d(CUtensorMap* out, const float* base, int d0, int d1, int d2, size_t stride1, size_t stride2,
                 int box0, int box1, int box2) {
  return make_tmap_3d_sw(out, base, d0, d1, d2, stride1, stride2, box0, box1, box2, CU_TENSOR_MAP_SWIZZLE_128B);
}
static int make_tmap_3d_sw(CUtensorMap* out, const float* base, int d0, int d1, int d2, size_t stride1, size_t stride2,
                           int box0, int box1, int box2, CUtensorMapSwizzle sw) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
  cuuint64_t gstr[2] = {(cuuint64_t)stride1 * sizeof(float), (cuuint64_t)stride2 * sizeof(float)};
  cuuint32_t box[3] = {(cuuint32_t)box0, (cuuint32_t)box1, (cuuint32_t)box2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(out, g_tmap_dtype, 3, const_cast<float*>(base), gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(3d %d,%d,%d box %d,%d,%d) failed: %d", d0, d1, d2, box0, box1, box2, (int)r);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

int make_tmap_nd_f32(CUtensorMap* out, const float* base, int rank, const unsigned long long* dims,
                     const unsigned long long* strides_bytes, const unsigned int* box) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = g_encode(out, g_tmap_dtype, (cuuint32_t)rank, const_cast<float*>(base), gdim, gstr, bx, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(rank %d) failed: %d", rank, (int)r);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

int make_tmap_4d_f32(CUtensorMap* out, const float* base, const unsigned long long dims[4],
                     const unsigned long long strides_bytes[3], const unsigned int box[4]) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(out, g_tmap_dtype, 4, const_cast<float*>(base), gdim, gstr, bx, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d %llu,%llu,%llu,%llu) failed: %d", dims[0], dims[1], dims[2], dims[3], (int)r);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

// fp16 tensor of rank 2 or 3 (d0 innermost), strides in ELEMENTS, 128B swizzle (box0 * 2 bytes <= 128)
int make_tmap_f16(CUtensorMap* out, const void* base, int rank, int d0, int d1, int d2, size_t stride1,
                  size_t stride2, int box0, int box1, int box2) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
  cuuint64_t gstr[2] = {(cuuint64_t)stride1 * 2, (cuuint64_t)stride2 * 2};
  cuuint32_t box[3] = {(cuuint32_t)box0, (cuuint32_t)box1, (cuuint32_t)box2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(f16 rank %d dims %d,%d,%d box %d,%d,%d) failed: %d", rank, d0, d1, d2, box0, box1,
              box2, (int)r);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

// ---- kernel ----------------------------------------------------------------------------------------
// 128 x BN output tile per CTA; a 128-byte swizzle row holds 32 fp32 (or 64 fp16) of K, one stage = one row of K
// for both operand tiles.  Two configurations, chosen on the host from N (`tile_n`):
//   BN = 128: six 32 KB stages, wgmma m64n128 per warpgroup (N <= 128: the fc head, small shapes)
//   BN = 256: four 48 KB stages (A 16 KB + B 32 KB), wgmma m64n256 per warpgroup (the recurrent stack's GEMMs):
//             half the shared-memory operand reads per MMA of the 128 x 128 tile
namespace gtc {
constexpr int BM = 128, BK = 32, THREADS = 384;
// registers per thread after the producer warpgroup hands its surplus to the two MMA warpgroups: 128 x 40 + 256 x 232
// = 384 x 168, the whole allotment of one CTA of 384 threads
constexpr int PRODUCER_REGS = 40, MMA_REGS = 232;
template <int BN>
struct Cfg {
  static constexpr int STAGES = BN == 256 ? 4 : 6;
  static constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128, STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};
static_assert(Cfg<256>::SMEM_BYTES <= 227 * 1024 && Cfg<128>::SMEM_BYTES <= 227 * 1024, "shared memory");
}  // namespace gtc

// F16 (precision-16 mode): fp16 operands, the same 128-byte rows hold 64 halfs, wgmma k16 instead of tf32 k8;
// accumulation and C stay fp32.  `alpha_dev` (optional) multiplies alpha by a device-resident factor (the inverse of
// the power-of-two scale of a scaled fp16 operand).
// The MMA warpgroups keep one wgmma group in flight: stage s is released once stage s + 1's group is issued and
// stage s's has completed, so the tensor pipe does not drain between stages.  The products still reach every
// accumulator in ascending K, one k-step after the other.
template <bool F16, int BN>
__global__ void __launch_bounds__(gtc::THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
               float alpha, float beta, float* __restrict__ C, int ldc, const float* __restrict__ alpha_dev) {
  using namespace gtc;
  using namespace tc;
  constexpr int STAGES = Cfg<BN>::STAGES, A_BYTES = Cfg<BN>::A_BYTES, STAGE_BYTES = Cfg<BN>::STAGE_BYTES;
  constexpr int BK = F16 ? 2 * gtc::BK : gtc::BK;         // K elements per stage (shadows gtc::BK)
  if (alpha_dev) alpha *= __ldg(alpha_dev);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int nk = (K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // two MMA warpgroups
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // TMA producer (one thread of warpgroup 0)
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      for (int it = 0; it < nk; ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
        uint8_t* sa = smem + s * STAGE_BYTES;
        tma_load_2d(sa, &tmA, &full[s], it * BK, m0);
        tma_load_2d(sa + A_BYTES, &tmB, &full[s], it * BK, n0);
      }
    }
  } else {
    // two MMA warpgroups, 64 rows of the tile each; the accumulators stay in registers for the epilogue
    setmaxnreg_inc<MMA_REGS>();
    const int wg = warp / 4 - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int it = 0; it < nk; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full[s], (it / STAGES) & 1);
      const uint64_t adesc = smem_desc_sw128(smem_u32(smem + s * STAGE_BYTES)) + (uint64_t)(512 * wg);
      const uint64_t bdesc = smem_desc_sw128(smem_u32(smem + s * STAGE_BYTES + A_BYTES));
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)          // four 32-byte k-steps per 128-byte row (K = 8 tf32 / 16 fp16)
        Wgmma<BN, F16>::mma(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
      wg_commit();
      wg_wait<1>();                        // the previous stage's group has read its operands
      if (it > 0 && leader) mbar_arrive(&empty[(it - 1) % STAGES]);
    }
    wg_wait<0>();
    if (leader) mbar_arrive(&empty[(nk - 1) % STAGES]);
    // fragment: rows 16 w + l/4 (+8), column pairs 8 i + 2 (l%4)
    const int w = warp % 4;
    const bool vec_ok = ((ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(C) & 7) == 0);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = m0 + 64 * wg + 16 * w + (lane >> 2) + 8 * hh;
      if (row >= M) continue;
      float* crow = C + (size_t)row * ldc;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = n0 + 8 * i + 2 * (lane & 3);
        float2 o = make_float2(alpha * acc[4 * i + 2 * hh], alpha * acc[4 * i + 2 * hh + 1]);
        if (vec_ok && col + 1 < N) {
          float2* cp2 = reinterpret_cast<float2*>(crow + col);
          if (beta != 0.f) {
            const float2 old = *cp2;
            o.x = fmaf(beta, old.x, o.x);
            o.y = fmaf(beta, old.y, o.y);
          }
          *cp2 = o;
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (col + j >= N) break;
            float v = j ? o.y : o.x;
            if (beta != 0.f) v = fmaf(beta, crow[col + j], v);
            crow[col + j] = v;
          }
        }
      }
    }
  }
}

// out (C x R, pitch ldo) = in (R x C, pitch ldi)^T
__global__ void transpose_strided_kernel(int R, int C, const float* __restrict__ in, size_t ldi,
                                         float* __restrict__ out, size_t ldo) {
  __shared__ float tile[32][33];
  int c = blockIdx.x * 32 + threadIdx.x, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (r0 + j < R && c < C) tile[j][threadIdx.x] = in[(size_t)(r0 + j) * ldi + c];
  __syncthreads();
  int r = r0 + threadIdx.x, c0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (c0 + j < C && r < R) out[(size_t)(c0 + j) * ldo + r] = tile[threadIdx.x][j];
}

int transpose_strided(int R, int C, const float* in, size_t ldi, float* out, size_t ldo, cudaStream_t st) {
  DS2_LAUNCH(transpose_strided_kernel, dim3(cdiv(C, 32), cdiv(R, 32)), dim3(32, 8), 0, st, R, C, in, ldi, out, ldo);
  return DS2_OK;
}
int transpose(int R, int C, const float* in, float* out, cudaStream_t st) {
  return transpose_strided(R, C, in, (size_t)C, out, (size_t)R, st);
}

static inline size_t k4(int K) { return (size_t)((K + 3) / 4 * 4); }

// Workspace of gemm_tc (bytes; with a base, also the addresses), each buffer 256-byte aligned: the K-major copy of an
// operand stored the other way round, A^T (M,k4(K)) if transA | B^T (N,k4(K)) if !transB; null for the others.
struct GemmTcWs { float *At, *Bt; };
static size_t gemm_tc_ws_carve(int transA, int transB, int M, int N, int K, void* base, GemmTcWs& w) {
  size_t off = 0;
  w.At = transA ? carve<float>(base, off, (size_t)M * k4(K) * 4) : nullptr;
  w.Bt = transB ? nullptr : carve<float>(base, off, (size_t)N * k4(K) * 4);
  return off;
}

size_t gemm_tc_workspace_bytes(int transA, int transB, int M, int N, int K) {
  GemmTcWs w;
  return gemm_tc_ws_carve(transA, transB, M, N, K, nullptr, w);
}

static bool tc_eligible(int M, int N, int K) { return K >= 32 && M >= 32 && N >= 16 && (long long)M * N * K >= (1 << 18); }

// columns of the output tile: 256 wherever N needs more than one 128-column tile
static int tile_n(int N) { return N > 128 ? 256 : 128; }

template <bool F16, int BN>
static int launch_gemm_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, float alpha, float beta,
                          float* C, int ldc, cudaStream_t st, const float* alpha_dev) {
  auto kern = gemm_tc_kernel<F16, BN>;
  constexpr int smem = gtc::Cfg<BN>::SMEM_BYTES;
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    DS2_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_once.done();
  }
  dim3 grid(cdiv(N, BN), cdiv(M, gtc::BM));
  DS2_LAUNCH(kern, grid, gtc::THREADS, smem, st, tmA, tmB, M, N, K, alpha, beta, C, ldc, alpha_dev);
  return DS2_OK;
}

template <bool F16>
static int launch_gemm_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, float alpha, float beta,
                          float* C, int ldc, cudaStream_t st, const float* alpha_dev = nullptr) {
  if (tile_n(N) == 256) return launch_gemm_tc<F16, 256>(tmA, tmB, M, N, K, alpha, beta, C, ldc, st, alpha_dev);
  return launch_gemm_tc<F16, 128>(tmA, tmB, M, N, K, alpha, beta, C, ldc, st, alpha_dev);
}

// TF32 wgmma reads both operands K-major: an operand stored the other way round (transA / !transB) is first
// transposed into the workspace.  Without room for those copies the kernel declines.
int gemm_tc(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
            int ldb, float beta, float* C, int ldc, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (!tc_eligible(M, N, K)) return 1;
  GemmTcWs W;
  if (gemm_tc_ws_carve(transA, transB, M, N, K, ws, W) > (ws ? ws_bytes : 0)) return 1;
  const float* Ak = A;
  int ldak = lda;
  if (transA) {  // stored (K, M)
    int rc = transpose_strided(K, M, A, (size_t)lda, W.At, k4(K), st);
    if (rc) return rc;
    Ak = W.At;
    ldak = (int)k4(K);
  }
  const float* Bk = B;
  int ldbk = ldb;
  if (!transB) {  // stored (K, N)
    int rc = transpose_strided(K, N, B, (size_t)ldb, W.Bt, k4(K), st);
    if (rc) return rc;
    Bk = W.Bt;
    ldbk = (int)k4(K);
  }
  if ((ldak & 3) || (ldbk & 3) || (reinterpret_cast<uintptr_t>(Ak) & 15) || (reinterpret_cast<uintptr_t>(Bk) & 15))
    return 1;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_2d(&tmA, Ak, M, K, ldak, gtc::BM, gtc::BK);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, Bk, N, K, ldbk, tile_n(N), gtc::BK);
  if (rc) return rc;
  return launch_gemm_tc<false>(tmA, tmB, M, N, K, alpha, beta, C, ldc, st);
}

// C[M,N] (fp32) = alpha * [*alpha_dev] * A[M,K] . B[N,K]^T + beta * C with fp16 K-major operands (precision-16 mode).
// Returns 1 when the shape / alignment is not eligible (the caller then runs the TF32 path on the fp32 tensors).
int gemm_tc_f16(int M, int N, int K, float alpha, const void* A16, int lda, const void* B16, int ldb, float beta,
                float* C, int ldc, const float* alpha_dev, cudaStream_t st) {
  if (!tc_eligible(M, N, K) || M < 128) return 1;
  if ((lda & 7) || (ldb & 7) || (reinterpret_cast<uintptr_t>(A16) & 15) || (reinterpret_cast<uintptr_t>(B16) & 15)) return 1;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_f16(&tmA, A16, 2, K, M, 1, (size_t)lda, 0, 64, gtc::BM, 1);
  if (rc) return rc;
  rc = make_tmap_f16(&tmB, B16, 2, K, N, 1, (size_t)ldb, 0, 64, tile_n(N), 1);
  if (rc) return rc;
  return launch_gemm_tc<true>(tmA, tmB, M, N, K, alpha, beta, C, ldc, st, alpha_dev);
}

}  // namespace ds2
