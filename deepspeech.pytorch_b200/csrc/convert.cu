// fp32 -> fp16 operand copies for the precision-16 GEMMs (SURVEY.md §8f row N4; the reference trains with
// `precision: 16`, configs/librispeech.yaml:12, i.e. autocast casts the GEMM operands to half and accumulates in fp32).
// The fp16 wgmma GEMM takes K-major operands only, so operands whose reduction index is the row index in memory
// (dG^T, x^T, h^T for the weight gradients; W_ih^T for the data gradient) are transposed while they are converted.
// Gradients are multiplied by a power of two first (a device-resident scale, like AMP's loss scale but per tensor and
// exact to undo): fp16 has 5 exponent bits, the gate gradients of a T' = 500 recurrence span more.
#include <cuda_fp16.h>

#include "common.cuh"

namespace ds2 {

// out[r, c] = half(scale * in[r, c]); rows x cols, row pitches ld_in / ld_out (elements); cols % 4 == 0, 16-byte aligned rows
__global__ void f32_to_f16_rows_kernel(int rows, int cols, const float* __restrict__ in, size_t ld_in,
                                       __half* __restrict__ out, size_t ld_out, const float* __restrict__ scale_dev) {
  const float s = scale_dev ? __ldg(scale_dev) : 1.f;
  const int c4 = cols / 4;
  const size_t total = (size_t)rows * c4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / c4, c = (i % c4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(in + r * ld_in + c);
    const __half2 lo = __floats2half2_rn(v.x * s, v.y * s), hi = __floats2half2_rn(v.z * s, v.w * s);
    uint2 pk;
    pk.x = *reinterpret_cast<const unsigned int*>(&lo);
    pk.y = *reinterpret_cast<const unsigned int*>(&hi);
    *reinterpret_cast<uint2*>(out + r * ld_out + c) = pk;
  }
}

// 64 x 64 tiles: outT[c, r] = half(scale * in[r, c]) and, when out != nullptr, out[r, c] = the same value row-major.
// grid (ceil(cols/64), ceil(rows/64)), block 256.  Vector path (cols % 4 == 0, rows % 8 == 0, pitches / bases
// 16-byte aligned): float4 loads, 8-byte row-major stores, 16-byte transposed stores (8 consecutive rows of one
// column gathered from the shared-memory tile); anything else takes the element-wise path.
__global__ void __launch_bounds__(256) f32_to_f16_transpose_kernel(int rows, int cols, const float* __restrict__ in,
                                                                   size_t ld_in, __half* __restrict__ out, size_t ld_out,
                                                                   __half* __restrict__ outT, size_t ld_outT,
                                                                   const float* __restrict__ scale_dev, int vec) {
  __shared__ __align__(16) __half tile[64][72];
  const float s = scale_dev ? __ldg(scale_dev) : 1.f;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  if (vec) {
    const int cq = threadIdx.x % 16, rq = threadIdx.x / 16;           // 16 float4 per row, 16 rows per pass
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = rq + 16 * i, r = r0 + rr, c = c0 + 4 * cq;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < rows && c < cols) v = *reinterpret_cast<const float4*>(in + (size_t)r * ld_in + c);
      const __half2 lo = __floats2half2_rn(v.x * s, v.y * s), hi = __floats2half2_rn(v.z * s, v.w * s);
      uint2 pk;
      pk.x = *reinterpret_cast<const unsigned int*>(&lo);
      pk.y = *reinterpret_cast<const unsigned int*>(&hi);
      *reinterpret_cast<uint2*>(&tile[rr][4 * cq]) = pk;
      if (out && r < rows && c < cols) *reinterpret_cast<uint2*>(out + (size_t)r * ld_out + c) = pk;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int pce = threadIdx.x + 256 * i, tc = pce / 8, seg = pce % 8;   // column tc, rows 8*seg .. 8*seg+7
      const int c = c0 + tc, r = r0 + 8 * seg;
      if (c < cols && r < rows) {
        __align__(16) __half h[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) h[k] = tile[8 * seg + k][tc];
        *reinterpret_cast<uint4*>(outT + (size_t)c * ld_outT + r) = *reinterpret_cast<const uint4*>(h);
      }
    }
    return;
  }
  const int tx = threadIdx.x % 64, ty = threadIdx.x / 64;   // 64 x 4
  for (int rr = ty; rr < 64; rr += 4) {
    const int r = r0 + rr, c = c0 + tx;
    const float v = (r < rows && c < cols) ? in[(size_t)r * ld_in + c] * s : 0.f;
    const __half h = __float2half_rn(v);
    tile[rr][tx] = h;
    if (out && r < rows && c < cols) out[(size_t)r * ld_out + c] = h;
  }
  __syncthreads();
  for (int cc = ty; cc < 64; cc += 4) {
    const int c = c0 + cc, r = r0 + tx;
    if (c < cols && r < rows) outT[(size_t)c * ld_outT + r] = tile[tx][cc];
  }
}

// scale[0] = 2^k such that max|x| * 2^k lies in [2^(top-1), 2^top), scale[1] = 2^-k.  top = 10 when x is the tensor
// that gets converted (64x below the fp16 maximum), top = 5 when x only bounds it from below (dY for the gate
// gradients: 2^11 of headroom for what the recurrence adds).  absmax_bits: float bits of max|x|.
__global__ void pow2_scale_kernel(const unsigned int* __restrict__ absmax_bits, float* __restrict__ scale, int top) {
  const unsigned int m = *absmax_bits;
  int k = 0;
  if (m != 0u && m < 0x7f800000u) {
    const int E = (int)((m >> 23) & 0xffu);       // m = f * 2^(E-126), f in [0.5, 1)
    k = top + 126 - E;                            // m * 2^k in [2^(top-1), 2^top)
    k = k < -100 ? -100 : (k > 100 ? 100 : k);
  }
  scale[0] = __int_as_float((k + 127) << 23);
  scale[1] = __int_as_float((-k + 127) << 23);
}

__global__ void absmax_strided_kernel(int rows, int cols, const float* __restrict__ x, size_t ld,
                                      unsigned int* __restrict__ out) {
  float m = 0.f;
  const int c4 = cols / 4;
  const size_t total = (size_t)rows * c4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / c4, c = (i % c4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + r * ld + c);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x % 32 == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

int f32_to_f16_rows(int rows, int cols, const float* in, size_t ld_in, void* out, size_t ld_out, const float* scale_dev,
                    cudaStream_t st) {
  DS2_REQUIRE(cols % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0, "f32_to_f16_rows: cols / pitches must be multiples of 4");
  const size_t total = (size_t)rows * (cols / 4);
  int blocks = (int)((total + 255) / 256);
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  DS2_LAUNCH(f32_to_f16_rows_kernel, blocks, 256, 0, st, rows, cols, in, ld_in, static_cast<__half*>(out), ld_out, scale_dev);
  return DS2_OK;
}

int f32_to_f16_transpose(int rows, int cols, const float* in, size_t ld_in, void* out, size_t ld_out, void* outT,
                         size_t ld_outT, const float* scale_dev, cudaStream_t st) {
  const int vec = cols % 4 == 0 && rows % 8 == 0 && ld_in % 4 == 0 && ld_outT % 8 == 0 && (!out || ld_out % 4 == 0) &&
                  (reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(outT) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(out) & 7) == 0;
  DS2_LAUNCH(f32_to_f16_transpose_kernel, dim3(cdiv(cols, 64), cdiv(rows, 64)), 256, 0, st, rows, cols, in, ld_in,
             static_cast<__half*>(out), ld_out, static_cast<__half*>(outT), ld_outT, scale_dev, vec);
  return DS2_OK;
}

// scale[0..1] <- power-of-two scale / inverse for the (rows x cols, pitch ld) fp32 matrix x; absmax_ws: 1 uint scratch
int pow2_scale_for(int rows, int cols, const float* x, size_t ld, unsigned int* absmax_ws, float* scale, int top,
                   cudaStream_t st) {
  DS2_REQUIRE(cols % 4 == 0 && ld % 4 == 0, "pow2_scale_for: cols / pitch must be multiples of 4");
  DS2_CHECK_CUDA(cudaMemsetAsync(absmax_ws, 0, sizeof(unsigned int), st));
  DS2_LAUNCH(absmax_strided_kernel, 132 * 4, 256, 0, st, rows, cols, x, ld, absmax_ws);
  DS2_LAUNCH(pow2_scale_kernel, 1, 1, 0, st, absmax_ws, scale, top);
  return DS2_OK;
}

}  // namespace ds2
