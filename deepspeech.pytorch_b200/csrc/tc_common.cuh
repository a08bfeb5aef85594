// sm_90a building blocks shared by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA
// (wgmma) shared-memory descriptors, issue / commit / wait, and the shared-memory accumulator image the recurrent
// sweeps hand from the MMA warpgroup to their epilogue warps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "wgmma.cuh"

namespace ds2 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (mbarrier.try_wait may suspend the thread for a system-dependent time when the
// phase is not complete; test_wait returns immediately)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- TMA --------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates (c0 = innermost element index, c1 = row)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// Warp-converged issue: every lane executes the instruction stream, one elected lane issues (a lone divergent
// lane pays a uniform-register round trip per descriptor / address operand).
__device__ __forceinline__ void mbar_arrive_expect_tx_w(uint64_t* bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\telect.sync _|pe, 0xffffffff;\n\t"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_w(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\telect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_w(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                              int c2) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\telect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---- warpgroup MMA (wgmma) --------------------------------------------------------------------
// K-major operand tile stored as rows of 128 bytes (32 fp32 / 64 fp16) with the 128-byte swizzle (what TMA writes
// with CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups are 1024 bytes apart (stride byte offset), the leading byte offset
// is unused for swizzled K-major tiles.  A k-step (32 bytes) advances the start address field by 2, 64 rows by 512.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                        // layout type SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Move registers between the warpgroups of a CTA: a warpgroup gives up registers (dec) or waits until it can take
// that many (inc).  Every warp of the warpgroup executes it.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// tell the compiler a value is warp-uniform (lane 0's copy): arithmetic on it then runs in the uniform datapath
__device__ __forceinline__ uint64_t warp_uniform(uint64_t v) {
  const uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)v, 0), hi = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), 0);
  return ((uint64_t)hi << 32) | lo;
}
// Release a pipeline stage once the MMAs issued so far have read it: every thread of the warpgroup waits for its
// wgmma groups, one thread arrives on the stage's (count 1) mbarrier.
__device__ __forceinline__ void wg_release(uint64_t* bar) {
  wg_commit();
  wg_wait<0>();
  if ((threadIdx.x & 127) == 0) mbar_arrive(bar);
}

// floats of the accumulator image for a batch width NB (a multiple of 32: the epilogues read 32 columns at a time; odd
// pitch: the 32 lanes of a warp read 32 different rows without bank conflicts)
__host__ __device__ constexpr int acc_pitch(int NB) { return (NB + 31) / 32 * 32 + 1; }
__host__ __device__ constexpr int acc_image_bytes(int NB) { return 128 * acc_pitch(NB) * 4; }

// The same for a stage barrier initialised with count 128: every thread arrives, so no wgmma of the loop sits behind a
// divergent branch (which makes ptxas serialise them).
__device__ __forceinline__ void wg_release_all(uint64_t* bar) {
  wg_commit();
  wg_wait<0>();
  mbar_arrive(bar);
}

// Accumulator of the recurrent sweeps: MH blocks of 64 rows x 32*NCH columns (the batch, padded to a multiple of 32),
// issued as wgmma m64n32 per (row block, column chunk).  Shapes are compile-time, so no wgmma sits on a divergent path.
template <int MH, int NCH>
struct WgAcc {
  float r[MH][NCH][16];
};
// D (+)= A . B^T for a K step: A = MH x 64 rows at adesc (+512 per 64 rows), B = 32*NCH rows at bdesc (+256 per 32 rows)
template <bool F16, int MH, int NCH>
__device__ __forceinline__ void wg_mma_nb(WgAcc<MH, NCH>& acc, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
#pragma unroll
  for (int h = 0; h < MH; ++h) {
#pragma unroll
    for (int c = 0; c < NCH; ++c)
      Wgmma<32, F16>::mma(acc.r[h][c], adesc + (uint64_t)(512 * h), bdesc + (uint64_t)(256 * c), accumulate);
  }
}
// the four k-steps of one 128-byte K chunk (K = 32 tf32 / 64 fp16); `accumulate` = 0 starts a new sum
template <bool F16, int MH, int NCH>
__device__ __forceinline__ void wg_mma4(WgAcc<MH, NCH>& acc, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  wg_fence();
  wg_mma_nb<F16>(acc, adesc, bdesc, accumulate);
#pragma unroll
  for (int k = 1; k < 4; ++k) wg_mma_nb<F16>(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
}
// Call f(std::integral_constant<int, NB / 32>) for a batch width NB = 32, 64, .. 32 * MAXCH: the MMA loop of a sweep is
// instantiated once per accumulator width and chosen once per launch, outside the step loop.
template <int MAXCH, class F>
__device__ __forceinline__ void with_nch(int NB, F&& f) {
  if (NB == 32) f(std::integral_constant<int, 1>{});
  else if constexpr (MAXCH >= 2) {
    if (NB == 64) f(std::integral_constant<int, 2>{});
    else if constexpr (MAXCH >= 4) {
      if (NB == 96) f(std::integral_constant<int, 3>{});
      else if (NB == 128) f(std::integral_constant<int, 4>{});
    }
  }
}
// Shared-memory image of the accumulator, addressed like the accumulator rows the epilogues read: row `lane` of
// `pitch` floats.  M = 128 (MH = 2): lane = row; M = 64: row r sits in lane 32 (r / 16) + r % 16 (rows 16 q .. 16 q + 15
// in lanes 0..15 of quarter q).  Called by the whole warpgroup after wg_wait<0>().
template <int MH, int NCH>
__device__ __forceinline__ void wg_store_acc(const WgAcc<MH, NCH>& acc, float* tm, int pitch) {
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < MH; ++h) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int col = 32 * c + 8 * i + 2 * (l & 3);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = 16 * w + (l >> 2) + 8 * hh;
          const int lane = MH == 2 ? 64 * h + r : 32 * (r >> 4) + (r & 15);
          tm[lane * pitch + col] = acc.r[h][c][4 * i + 2 * hh];
          tm[lane * pitch + col + 1] = acc.r[h][c][4 * i + 2 * hh + 1];
        }
      }
    }
  }
}
// All MMAs of the step done: write the accumulator image, then one arrival on `bar` (count 1) once the whole
// warpgroup has written (named barrier 2 orders the other threads' stores before the arrival's release).
template <int MH, int NCH>
__device__ __forceinline__ void wg_publish(const WgAcc<MH, NCH>& acc, float* tm, uint64_t* bar) {
  wg_commit();
  wg_wait<0>();
  wg_store_acc(acc, tm, acc_pitch(32 * NCH));
  asm volatile("bar.sync 2, 128;" ::: "memory");
  if ((threadIdx.x & 127) == 0) mbar_arrive(bar);
}
// accumulator image -> registers: this thread's lane (taddr >> 16 plus the lane id), 32 consecutive columns
__device__ __forceinline__ void tmem_ld32(const float* tm, int pitch, uint32_t taddr, float* v) {
  const float* src = tm + (size_t)((taddr >> 16) + (threadIdx.x & 31)) * pitch + (taddr & 0xFFFFu);
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = src[i];
}
}  // namespace tc

// ---- host: tensor-map encoding through the driver entry point (no -lcuda link dependency) ------
// 2-D row-major fp32 matrix [rows, cols] with row pitch `ld` floats; box = box_rows x 32 floats,
// 128-byte swizzle, out-of-bounds elements read as zero.
int make_tmap_2d(CUtensorMap* out, const float* base, int rows, int cols, int ld, int box_rows, int box_cols);
int make_tmap_3d(CUtensorMap* out, const float* base, int d0, int d1, int d2, size_t stride1_floats,
                 size_t stride2_floats, int box0, int box1, int box2);
int make_tmap_f16(CUtensorMap* out, const void* base, int rank, int d0, int d1, int d2, size_t stride1_elems,
                  size_t stride2_elems, int box0, int box1, int box2);

}  // namespace ds2
