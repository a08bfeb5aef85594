// Persistent, warp-specialised recurrent sweeps on wgmma tensor cores.
//
// One launch per layer covers ALL time steps and, when the GPU holds both, both directions.  Per step a CTA computes
//     acc[(g,u), b] = sum_k W_hh[g*H+u, k] * h_{t-1}[b, k]        (wgmma, tf32 or f16, N = batch)
// for its hidden units with fp32 accumulators.  288 threads per CTA (rp::THREADS):
//   warp 8     TMA producer: weight chunks and h_{t-1} chunks (after the grid barrier) into 128B-swizzled shared
//              memory, either a ring of STAGES chunks (streaming variants) or, in the resident variants, the whole
//              fp16 weight slice once and the fp16 h_{t-1} per step
//   warps 4-7  MMA warpgroup: wgmma into registers, then the accumulator image in shared memory -> mbarrier
//   warps 0-3  epilogue: accumulator image -> registers, + input projection + biases, gate non-linearities,
//              cell update (c / h state stays in shared memory for the whole sweep), masked stores of h_t (and
//              the saved tensors for backward)
// (rnn_fwd_splitk_kernel differs: its MMA warpgroup finishes the step from its registers, see there.)
// Steps are separated by a per-direction grid barrier (monotonic counter in global memory, release / acquire,
// bounded spin so that a fault cannot hang the GPU).  All CTAs of a launch must be co-resident: launch_sweep checks
// occupancy and launches cooperatively; shapes that do not fit return 1 (FFMA step kernels).
//
// Kernels: rnn_fwd_persist_kernel (16 units per CTA), rnn_fwd_splitk_kernel (2-CTA clusters split K = H),
// rnn_bwd_persist_kernel (16 units per CTA on W_hh^T) and rnn_bwd_splitk_kernel (4- or 8-CTA groups split
// K = G*H; the partial sums travel through distributed shared memory or, with XG, through L2).
#include <cooperative_groups.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"
#include "rnn_cells.cuh"
#include "rnn_common.cuh"
#include "tc_common.cuh"

namespace cg = cooperative_groups;

namespace ds2 {

namespace rp {
constexpr int UT = 16;        // hidden units per CTA
constexpr int MM = 64;        // MMA M (G*UT rows, padded for GRU / tanh)
constexpr int BK = 32;        // fp32 elements per 128-byte swizzle row
constexpr int STAGES = 8;
constexpr int THREADS = 288;  // warps 0..3 epilogue, warps 4..7 MMA warpgroup, warp 8 producer
constexpr int A_BYTES = MM * 128;
constexpr long long SPIN_LIMIT = 4000000000LL;   // ~2 s of SM clocks
}  // namespace rp

struct PersistParams {
  CUtensorMap tmW[2];   // 3-D (k, unit, gate) over W_hh[d]
  CUtensorMap tmV[2];   // 2-D (k, row) over the per-direction vector sequence (hseq[d] as [T*B, H])
  CUtensorMap tmV2[2];  // bwd GRU: the n-gate part of dGh lives in the aux buffer
  CUtensorMap tmV3[2];  // resident: 3-D view (k in chunk, row, chunk) of the streamed fp16 operand, box = 4 chunks
  int box3;             // 1: tmV3 is valid (number of chunks divisible by 4): one TMA instruction per group
  int T, B, NB, H, D, NT, G, training;
  const float* dy;      // bwd: (T,B,H)
  __half* h16;          // resident fwd: fp16 copy of hseq (D,T,B,H), the MMA operand of the next step
  __half* dg16;         // resident bwd: scaled fp16 copy of dGh (T*B, D*G*H)
  unsigned int* gmax;   // resident bwd: [D][T+1] float bits of max|dGh| per processed step (slot 0: bound from dY)
  unsigned int* dymax;  // resident bwd: [T] float bits of max_b,u |dY[t]| (the scale of a step also covers its own dY)
  __half* dgn16;        // resident bwd, optional: fp16 copy of the gate gradients x nscale, (T*B, D*G*H) row-major
  __half* dgn16T;       //   ... transposed (D*G*H, T*B)
  __half* auxn16T;      //   ... GRU h-side n-gate gradient, transposed (D*H, T*B)
  const float* nscale;  //   device: power-of-two scale of those copies
  long long* trace;     // optional: clock64 stamps of CTA 0, 4 per step
  const int32_t* len;
  float* gates;
  float* hseq;
  float* aux;
  const float* b_ih[2];
  const float* b_hh[2];
  unsigned int* bar;    // [2][NT] per-CTA step flags (zeroed by the host): flag = number of finished steps
  int defer;            // 1: stores that only later kernels read are issued after the barrier arrival
  int d0;               // first direction handled by this launch (directions can be launched one at a time
                        // when both together would not be co-resident, e.g. H = 1536)
  float* dbias[2];      // split-K bwd: bias-gradient accumulators (G*H per direction, zeroed by the host) or null
  float* dbias_hn[2];   // split-K bwd, GRU: sum of dGh_n (H per direction)
  float* xbuf;          // split-K bwd, exchange through L2: [CTA][source rank][step parity] partial dh_rec tiles
  unsigned int* xcnt;   //   ... [CTA] number of partial tiles received (monotonic, zeroed by the host)
  int* err;             // set to 1 if a barrier wait timed out
  const float* h0;      // resident / split-K fwd with an initial state (ST): (D,B,H) or null (zeros)
  const float* c0;      //   ... LSTM cell state, (D,B,H) or null
};

__device__ __forceinline__ void red_release(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Cross-proxy ordering for data that one CTA writes with ordinary stores and another CTA reads with TMA.  The
// unqualified fence.proxy.async compiles to MEMBAR.ALL.GPU + FENCE.VIEW.ASYNC (measured ~950 cycles per call inside
// the sweeps, three of them on the per-step critical path); the .global form is the proxy fence alone, and the
// gpu-scope ordering comes from the release / acquire pair on the barrier counter, which is needed anyway.
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// The waits below only set *err on a timeout (sweep_check_kernel reports it after the launch): a device printf is
// a function call, and a call anywhere in a kernel makes ptxas serialise every wgmma of that kernel.
__device__ __forceinline__ unsigned int ld_relaxed(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Grid barrier of one direction: every CTA adds 1 per finished step to a monotonic arrival counter (red.release);
// one thread waits until it reaches target (relaxed polling loads, then one acquire fence: an acquire load would
// invalidate L1 on every poll).  Bounded spin: a fault cannot hang the GPU.
__device__ __forceinline__ void grid_wait_counter(const unsigned int* ctr, unsigned int target, int* err) {
  if (ld_relaxed(ctr) < target) {
    const long long t0 = clock64();
    unsigned int it = 0;
    while (ld_relaxed(ctr) < target) {
      if ((++it & 255u) == 0) {
        if (*(volatile int*)err) break;
        if (clock64() - t0 > rp::SPIN_LIMIT) {
          *(volatile int*)err = 1;
          break;
        }
      }
    }
  }
  asm volatile("fence.acquire.gpu;" ::: "memory");
}
// MUFU.EX2 / MUFU.RCP without the denormal-range fix-up code of the CUDA fast-math intrinsics (that code
// serialises independent chains through one predicate register); inputs are gate pre-activations.
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_ftz(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
constexpr float LOG2E = 1.4426950408889634f;
__device__ __forceinline__ float fast_sigmoid(float x) { return rcp_ftz(1.f + ex2_ftz(-LOG2E * x)); }
__device__ __forceinline__ float fast_tanh(float x) { return fmaf(2.f, rcp_ftz(1.f + ex2_ftz(-2.f * LOG2E * x)), -1.f); }

// debug trace: 16 clock64 slots per (CTA, step); slot 12 holds %globaltimer (ns) instead
constexpr int TRACE_SLOTS = 16;
__device__ __forceinline__ void trace_stamp(long long* trace, int T, int step, int slot) {
  if (trace) trace[((size_t)blockIdx.x * T + step) * TRACE_SLOTS + slot] = clock64();
}
__device__ __forceinline__ void trace_stamp_ns(long long* trace, int T, int step, int slot) {
  if (trace) {
    unsigned long long ns;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(ns));
    trace[((size_t)blockIdx.x * T + step) * TRACE_SLOTS + slot] = (long long)ns;
  }
}

// Resident variants: the streamed operand arrives in groups of 4 K chunks (256 k), one mbarrier per group.
// (A single-chunk first group was measured: the MMA chain starts ~250 cycles earlier but the extra
// producer instructions delay the later groups by as much; what limits the start of a step is the ~110
// cycles the single producer thread needs per TMA instruction, hence one 3-D box per group where possible.)
__device__ __forceinline__ int grp_begin(int g) { return 4 * g; }
__device__ __forceinline__ int grp_count(int nkr) { return (nkr + 3) / 4; }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}


// RES = true: "resident" variant.  W_hh is converted to fp16 once per call and this CTA's slice
// (G*16 rows x H, 128 KB at H=1024) stays in shared memory for the whole sweep; per step only the
// fp16 copy of h_{t-1} (B x H, 64 KB) is streamed by TMA, and the MMAs are kind::f16 (K=16, half the
// instruction count).  fp16 has the same 10-bit mantissa as TF32 and |h| < 1, |w| << 65504, so this
// is the same arithmetic class as the TF32 path (fp32 accumulation either way).
// ST (resident only): initial state p.h0 / p.c0.  Step 0 then runs the MMAs too, on fp16(h0) from the extra time step
// of h16 (f16_weight_maps), the carried cst starts from c0 (LSTM) / h0 (GRU), and the reverse direction writes
// fp16(h0) instead of 0 into the h16 rows of its padded steps: row len[b] is the operand of utterance b's first step.
template <int RNN, bool RES, bool ST = false>
__global__ void __launch_bounds__(rp::THREADS, 1) rnn_fwd_persist_kernel(const __grid_constant__ PersistParams p) {
  using namespace rp;
  using namespace tc;
  static_assert(RES || !ST, "the streaming variant reads h_{t-1} from hseq and cannot carry an initial state");
  constexpr int G = num_gates(RNN);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);   // 1 KB aligned, still __shared__
  const int NB = p.NB, B = p.B, T = p.T, H = p.H, D = p.D;
  const int B_BYTES = NB * 128, STAGE_BYTES = A_BYTES + B_BYTES;
  const int NBp = NB + 1;
  const int NKR = H / 64;                                  // resident: 64 fp16 (128 B) of K per chunk
  const int NG = grp_count(NKR);
  // streaming layout: STAGES x (A | B) ; resident layout: NKR x A (weights) then NKR x B (h chunks)
  const int ring_bytes = RES ? NKR * STAGE_BYTES : STAGES * STAGE_BYTES;
  float* ex = reinterpret_cast<float*>(smem + ring_bytes);            // [4][UT][NBp]
  float* cst = ex + 4 * UT * NBp;                                       // [UT][NBp] cell (LSTM) / hidden (GRU) state
  int* lens_s = reinterpret_cast<int*>(cst + UT * NBp);                 // [NB] (padded to even)
  uint64_t* full = reinterpret_cast<uint64_t*>(lens_s + ((NB + 1) & ~1));   // resident: one per h chunk (<= 32)
  uint64_t* empty = full + (RES ? 32 : STAGES);                             // resident: [0] = weights landed
  uint64_t* accum_bar = empty + STAGES;
  float* acc_img = reinterpret_cast<float*>(accum_bar + 1);   // accumulator image (tc::wg_store_acc)

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int d = p.d0 + blockIdx.x / p.NT, tile = blockIdx.x % p.NT, u0 = tile * UT;
  const int NK = H / BK;
  const int GH = G * H;
  unsigned int* ctr = p.bar + 32 * d;   // one 128-byte line per direction

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmW[d]);
    tma_prefetch_desc(&p.tmV[d]);
    for (int i = 0; i < (RES ? 32 : STAGES); ++i) mbar_init(&full[i], 1);
    for (int i = 0; i < STAGES; ++i) mbar_init(&empty[i], RES ? 1 : 128);   // streaming: every MMA-warpgroup thread arrives
    mbar_init(accum_bar, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < UT * NBp; i += THREADS) {
    float v = 0.f;
    if constexpr (ST) {
      const float* s0 = RNN == DS2_RNN_LSTM ? p.c0 : p.h0;
      const int b = i % NBp;
      if (RNN != DS2_RNN_TANH && s0 && b < B) v = s0[((size_t)d * B + b) * H + u0 + i / NBp];
    }
    cst[i] = v;
  }
  for (int i = threadIdx.x; i < NB; i += THREADS) lens_s[i] = i < B ? p.len[i] : 0;
  __syncthreads();
  const uint32_t tx_bytes = (uint32_t)(G * UT * 128 + B * 128);

  if (warp == 8) {                                        // TMA producer
    if (RES) {
      if (lane == 0) {
        // weights once: NKR chunks of (G*16 rows x 64 fp16) into the resident region
        mbar_arrive_expect_tx(&empty[0], (uint32_t)(NKR * G * UT * 128));
        for (int c = 0; c < NKR; ++c) tma_load_3d(smem + c * A_BYTES, &p.tmW[d], &empty[0], c * 64, u0, 0);
        uint8_t* hbuf = smem + NKR * A_BYTES;
        for (int step = ST ? 0 : 1; step < T; ++step) {
          const int t = d == 0 ? step : T - 1 - step;
          const int tp = d == 0 ? t - 1 : t + 1;
          const int row = (ST ? tp + 1 : tp) * B;         // ST: the maps start at time step -1
          // the previous step's MMAs have finished reading hbuf: this CTA's epilogue (which waited for them)
          // arrived at the barrier we are about to pass
          grid_wait_counter(ctr, (unsigned int)p.NT * (unsigned int)step, p.err);
          fence_proxy_async_global();
          trace_stamp(p.trace, p.T, step, 0);
          for (int g = 0; g < NG; ++g) {  // one mbarrier per group of chunks
            uint64_t* fb = full + g;
            const int c0 = grp_begin(g), c1 = min(NKR, grp_begin(g + 1));
            if (p.box3) {
              mbar_arrive_expect_tx(fb, (uint32_t)(4 * B_BYTES));
              tma_load_3d(hbuf + c0 * B_BYTES, &p.tmV3[d], fb, 0, row, c0);
            } else {
              mbar_arrive_expect_tx(fb, (uint32_t)((c1 - c0) * B * 128));
              for (int c = c0; c < c1; ++c) tma_load_2d(hbuf + c * B_BYTES, &p.tmV[d], fb, c * 64, row);
            }
          }
          trace_stamp(p.trace, p.T, step, 1);
        }
      }
    } else
    if (lane == 0) {
      // strict chunk order: slot free -> weight chunk -> (first chunk of a step: grid barrier) -> h chunk.
      // The weight chunk of the next step's first slot is therefore in flight while the barrier is awaited.
      int s = 0;
      uint32_t ph = 0;
      for (int step = 1; step < T; ++step) {
        const int t = d == 0 ? step : T - 1 - step;
        const int tp = d == 0 ? t - 1 : t + 1;
        for (int c = 0; c < NK; ++c) {
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], tx_bytes);
          tma_load_3d(smem + s * STAGE_BYTES, &p.tmW[d], &full[s], c * BK, u0, 0);
          if (c == 0) {
            grid_wait_counter(ctr, (unsigned int)p.NT * (unsigned int)step, p.err);
            fence_proxy_async_global();
            trace_stamp(p.trace, p.T, step, 0);
          }
          tma_load_2d(smem + s * STAGE_BYTES + A_BYTES, &p.tmV[d], &full[s], c * BK, tp * B);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // MMA warpgroup: accumulators in registers, handed to the epilogue warps as an image in shared memory; the
    // accumulator width (batch padded to 32 * NCH) is chosen once, outside the step loop
    with_nch<4>(NB, [&](auto nch) {
      WgAcc<1, decltype(nch)::value> acc;
      if (RES) {
        {
          const uint64_t a_base = warp_uniform(smem_desc_sw128(smem_u32(smem)));
          const uint64_t b_base = warp_uniform(smem_desc_sw128(smem_u32(smem + NKR * A_BYTES)));
          const uint64_t a_step = (uint64_t)(A_BYTES >> 4), b_step = (uint64_t)(B_BYTES >> 4);
          mbar_wait(&empty[0], 0);                 // weights resident
          uint32_t ph = 0;
          for (int step = ST ? 0 : 1; step < T; ++step) {
            for (int g = 0; g < NG; ++g) {
              mbar_wait(full + g, ph);
              if (g == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
              const int c0 = grp_begin(g), c1 = min(NKR, grp_begin(g + 1));
              if (c1 == NKR && lane == 0) trace_stamp(p.trace, p.T, step, 3);
              for (int c = c0; c < c1; ++c) {
                const uint64_t ad = a_base + (uint64_t)c * a_step, bd = b_base + (uint64_t)c * b_step;
                wg_mma4<true>(acc, ad, bd, c > 0);
              }
            }
            wg_publish(acc, acc_img, accum_bar);
            if (lane == 0) trace_stamp(p.trace, p.T, step, 4);
            ph ^= 1;
          }
        }
      } else
      {
        // The issue chain is the critical path of a step: the loop is free of div/mod and descriptor construction.
        const uint64_t a_base = smem_desc_sw128(smem_u32(smem));
        const uint64_t b_base = smem_desc_sw128(smem_u32(smem + A_BYTES));
        const uint64_t stage_step = (uint64_t)(STAGE_BYTES >> 4);
        int s = 0;
        uint32_t ph = 0;
        for (int step = 1; step < T; ++step) {
          for (int c = 0; c < NK; ++c) {
            mbar_wait(&full[s], ph);
            if (c == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 1);
            if (c == NK - 1 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
            const uint64_t ad = a_base + (uint64_t)s * stage_step, bd = b_base + (uint64_t)s * stage_step;
            wg_mma4<false>(acc, ad, bd, c > 0);
            wg_release_all(&empty[s]);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
          wg_publish(acc, acc_img, accum_bar);
        }
      }
    });
  } else {                                                // warps 0..3: epilogue
    // ---------------- epilogue warps: quarter q of accumulator-image == gate q (rows q*16 .. q*16+15 in lanes 0..15)
    // All 32 lanes work: lane L<16 owns row (q, L); its 32 batch columns are split with lane L+16
    // (columns 16..31 travel by shuffle), so every lane activates 16 values per 32-column chunk.
    const int q = warp % 4;
    const int e = threadIdx.x;          // 0..127
    const int ul = lane & 15, half = lane >> 4;
    const int u = u0 + ul;
    const bool has_row = (q < G) || (RNN == DS2_RNN_GRU && q == 3);
    const int gsel = (RNN == DS2_RNN_GRU && q == 3) ? 2 : q;   // GRU: warp 3 carries x_n + b_in
    float bias_x = 0.f, bias_h = 0.f;
    if (has_row) bias_x = p.b_ih[d][gsel * H + u];
    if (q < G) bias_h = p.b_hh[d][q * H + u];
    uint32_t acc_phase = 0;
    for (int step = 0; step < T; ++step) {
      const int t = d == 0 ? step : T - 1 - step;
      for (int cb = 0; cb < NB; cb += 32) {
        // input-projection values (independent of the recurrence: issued before waiting for the MMAs)
        float gx[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int b = cb + half * 16 + j;
          gx[j] = (has_row && b < B) ? p.gates[(((size_t)t * B + b) * D + d) * GH + (size_t)gsel * H + u] : 0.f;
        }
        float a16[16];
        if ((ST || step > 0) && q < G) {
          if (cb == 0) { mbar_wait(accum_bar, acc_phase); if (e == 0) trace_stamp(p.trace, p.T, step, 5); }
          float acc[32];
          tmem_ld32(acc_img, acc_pitch(NB), ((uint32_t)(q * 32) << 16) + (uint32_t)cb, acc);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float hi = __shfl_sync(0xffffffffu, acc[16 + j], ul);   // row owner's upper columns
            a16[j] = half ? hi : acc[j];
          }
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j) a16[j] = 0.f;
        }
        // The gate of a warp is uniform: v = sc * sigmoid(sc * pre) + (1 - sc) is the sigmoid for sc = 1 and tanh
        // for sc = 2, i.e. one EX2 + one RCP per value.  The 16 values of a lane are processed stage by stage so
        // that the special-function latencies overlap (the straightforward per-value form was compiled into two
        // serial chains and cost ~2200 cycles per step on the critical path).
        float v[16];
        const bool act = RNN == DS2_RNN_LSTM || (RNN == DS2_RNN_GRU && q < 2) || (RNN == DS2_RNN_TANH && q == 0);
        if (act) {
          const float sc = ((RNN == DS2_RNN_LSTM && q == 2) || RNN == DS2_RNN_TANH) ? 2.f : 1.f;
          const float bsum = bias_x + bias_h, nsc = -sc * LOG2E, off = 1.f - sc;
          float ev[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) ev[j] = ex2_ftz(nsc * ((gx[j] + a16[j]) + bsum));
#pragma unroll
          for (int j = 0; j < 16; ++j) ev[j] = rcp_ftz(1.f + ev[j]);
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = fmaf(sc, ev[j], off);
        } else if (RNN == DS2_RNN_GRU) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = q == 2 ? a16[j] + bias_h      // W_hn h + b_hn
                                                     : gx[j] + bias_x;      // x_n + b_in
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int b = cb + half * 16 + j;
          if (b < B) ex[(q * UT + ul) * NBp + b] = v[j];
        }
      }
      if (ST || step > 0) acc_phase ^= 1;
      if (e == 0) trace_stamp(p.trace, p.T, step, 6);
      named_bar_sync(1, 128);
      if (e == 0) trace_stamp(p.trace, p.T, step, 7);
      // ---------------- combine: thread e owns the 4 consecutive units 4*(e&3)..+3 of batch column (e>>2) [+32
      // per block], so every global access is one 8- or 16-byte vector, and the four cells are processed stage by
      // stage (independent special-function chains).  Only the fp16 copy of h_t (resident variant) is read by
      // the next step; the fp32 outputs (sequence output, saved activations / cell state for the backward) are
      // returned in o[] so that the caller can store them after the barrier arrival.
      constexpr int NDF = 4;
      const int uq = 4 * (e & 3);                  // first of this thread's units inside the CTA's 16
      auto combine4 = [&](int b, float (&o)[6][NDF]) {
        float e0[NDF], e1[NDF], e2[NDF], e3[NDF], cp[NDF], hval[NDF];
        const bool valid = t < lens_s[b];
#pragma unroll
        for (int j = 0; j < NDF; ++j) {
          const int ui = uq + j;
          e0[j] = ex[(0 * UT + ui) * NBp + b]; e1[j] = ex[(1 * UT + ui) * NBp + b];
          e2[j] = ex[(2 * UT + ui) * NBp + b]; e3[j] = ex[(3 * UT + ui) * NBp + b];
          cp[j] = cst[ui * NBp + b];
        }
        if (RNN == DS2_RNN_LSTM) {
          float cval[NDF], th[NDF];
#pragma unroll
          for (int j = 0; j < NDF; ++j) cval[j] = valid ? fmaf(e1[j], cp[j], e0[j] * e2[j]) : 0.f;
#pragma unroll
          for (int j = 0; j < NDF; ++j) th[j] = ex2_ftz(-2.f * LOG2E * cval[j]);
#pragma unroll
          for (int j = 0; j < NDF; ++j) th[j] = rcp_ftz(1.f + th[j]);
#pragma unroll
          for (int j = 0; j < NDF; ++j) {
            hval[j] = valid ? e3[j] * fmaf(2.f, th[j], -1.f) : 0.f;
            if (valid) cst[(uq + j) * NBp + b] = cval[j];
            o[0][j] = valid ? e0[j] : 0.f; o[1][j] = valid ? e1[j] : 0.f;
            o[2][j] = valid ? e2[j] : 0.f; o[3][j] = valid ? e3[j] : 0.f;
            o[4][j] = cval[j];
          }
        } else if (RNN == DS2_RNN_GRU) {
          float th[NDF];
#pragma unroll
          for (int j = 0; j < NDF; ++j) th[j] = ex2_ftz(-2.f * LOG2E * fmaf(e0[j], e2[j], e3[j]));
#pragma unroll
          for (int j = 0; j < NDF; ++j) th[j] = rcp_ftz(1.f + th[j]);
#pragma unroll
          for (int j = 0; j < NDF; ++j) {
            const float nval = valid ? fmaf(2.f, th[j], -1.f) : 0.f;
            hval[j] = valid ? fmaf(e1[j], cp[j] - nval, nval) : 0.f;
            if (valid) cst[(uq + j) * NBp + b] = hval[j];
            o[0][j] = valid ? e0[j] : 0.f; o[1][j] = valid ? e1[j] : 0.f; o[2][j] = nval; o[3][j] = 0.f;
            o[4][j] = valid ? e2[j] : 0.f;
          }
        } else {
#pragma unroll
          for (int j = 0; j < NDF; ++j) {
            hval[j] = valid ? e0[j] : 0.f;
            o[0][j] = hval[j]; o[1][j] = o[2][j] = o[3][j] = o[4][j] = 0.f;
          }
        }
#pragma unroll
        for (int j = 0; j < NDF; ++j) o[5][j] = hval[j];
        if constexpr (ST) {
          if (!valid && d == 1) {
#pragma unroll
            for (int j = 0; j < NDF; ++j) hval[j] = p.h0 ? p.h0[((size_t)B + b) * H + u0 + uq + j] : 0.f;
          }
        }
        if (RES) {
          const __half2 lo = __floats2half2_rn(hval[0], hval[1]), hi = __floats2half2_rn(hval[2], hval[3]);
          uint2 pk;
          pk.x = *reinterpret_cast<const unsigned int*>(&lo);
          pk.y = *reinterpret_cast<const unsigned int*>(&hi);
          *reinterpret_cast<uint2*>(p.h16 + (((size_t)d * T + t) * B + b) * H + u0 + uq) = pk;
        }
      };
      auto st4 = [](float* dst, const float (&v)[NDF]) {
        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      };
      auto store4 = [&](int b, const float (&o)[6][NDF]) {
        const size_t so = (((size_t)d * T + t) * B + b) * H + u0 + uq;
        float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + u0 + uq;
        if (RNN != DS2_RNN_TANH) st4(p.aux + so, o[4]);
        if (p.training) {
#pragma unroll
          for (int g = 0; g < G; ++g) st4(gp + g * H, o[g]);
        }
        st4(p.hseq + so, o[5]);
      };
      const bool defer = RES && p.defer && B <= 32;
      const int b_own = e >> 2;
      float sv[6][NDF];
      if (defer) {
        if (b_own < B) combine4(b_own, sv);
      } else {
        for (int b = b_own; b < B; b += 32) {
          combine4(b, sv);
          store4(b, sv);
        }
      }
      if (e == 0) trace_stamp(p.trace, p.T, step, 8);
      named_bar_sync(1, 128);          // CTA-scope: every epilogue thread's stores happen-before thread 0's release
      if (e == 0) {
        trace_stamp(p.trace, p.T, step, 9);
        fence_proxy_async_global();
        trace_stamp(p.trace, p.T, step, 10);
        // release is cumulative over the stores ordered by the named barrier
        red_release(ctr, 1u);
        trace_stamp(p.trace, p.T, step, 11);
        trace_stamp_ns(p.trace, p.T, step, 12);
      }
      if (defer) {
        if (b_own < B) store4(b_own, sv);
        if (e == 0) trace_stamp(p.trace, p.T, step, 13);
      }
    }
  }
  __syncthreads();
}

// A sweep whose barrier wait timed out leaves garbage behind: fail loudly.
// Runs right after every sweep launch; the trap makes the next CUDA call of the process return an error.
__global__ void sweep_check_kernel(const int* err) {
  if (*err != 0) {
    printf("ds2: recurrent sweep failed (code %d): results are invalid\n", *err);
    __trap();
  }
}

// ------------------------------------------------------------------------------------------------
// One persistent CTA per SM (they spin at the grid barrier and would only take issue slots from each other): ask for
// more than half of the 227 KB of shared memory even when the tiles are small.
static size_t one_cta_per_sm(size_t smem) { return smem < 116 * 1024 ? 116 * 1024 : smem; }

static long long* trace_ptr_from_env(const char* name) {
  const char* e = getenv(name);   // debug: device address of an int64 buffer of 6*T entries
  return e ? reinterpret_cast<long long*>(strtoull(e, nullptr, 10)) : nullptr;
}

// the epilogues use 8- / 16-byte vector accesses on these buffers
static bool vec_ok(const void* a, const void* b = nullptr, const void* c = nullptr, const void* d = nullptr) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
           reinterpret_cast<uintptr_t>(d)) & 15) == 0;
}

// The switches that force a variant the library picks by itself for other shapes (DESIGN §6.1): unset gives `dflt`,
// a value its integer, so that `=0` turns a switch off.
static int env_flag(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}
// DS2_SWEEP_DEFER=0: store everything before the barrier arrival (see PersistParams::defer)
static int sweep_defer_default() { return env_flag("DS2_SWEEP_DEFER", 1); }

// The 4 KB control block at the start of every sweep workspace, zeroed before each sweep: err (offset 0), the
// per-direction step counters and the per-CTA tile counters xcnt of the 4-CTA L2 exchange (at most XCNT_MAX CTAs).
constexpr size_t CTL_BAR = 128, CTL_XCNT = 1024, CTL_BYTES = 4096;
constexpr int XCNT_MAX = (int)(CTL_BYTES - CTL_XCNT) / 4;

static int sweep_nb(int B) { return (B + 31) / 32 * 32; }   // batch columns of the MMAs

// The fields every sweep fills the same way.  `units`: hidden units per CTA, or per group of CTAs of the split-K
// variants.
static PersistParams sweep_params(const SeqArgs& a, int units, const char* trace_env, void* ws) {
  PersistParams p{};
  p.T = a.T; p.B = a.B; p.NB = sweep_nb(a.B); p.H = a.H; p.D = a.D; p.NT = a.H / units; p.G = a.G;
  p.training = a.training;
  p.len = a.len; p.gates = a.gates; p.hseq = a.hseq; p.aux = a.aux; p.dy = a.dy; p.h0 = a.h0; p.c0 = a.c0;
  for (int d = 0; d < a.D; ++d) { p.b_ih[d] = a.b_ih[d]; p.b_hh[d] = a.b_hh[d]; }
  p.trace = trace_ptr_from_env(trace_env);
  p.defer = sweep_defer_default();
  p.err = static_cast<int*>(ws);
  p.bar = reinterpret_cast<unsigned int*>(static_cast<char*>(ws) + CTL_BAR);
  return p;
}

using SweepKernel = void (*)(const PersistParams);

// Opt in to 227 KB of dynamic shared memory, once per device.  A launcher opts in every instantiation it can pick, so
// that whichever shape comes first leaves none of them without it.  The occupancy queries below depend on the
// opt-in: call this before them.
static int opt_in_smem(DeviceOnce& once, std::initializer_list<SweepKernel> kerns) {
  if (once.first()) {
    for (SweepKernel k : kerns)
      DS2_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.done();
  }
  return DS2_OK;
}

// Launch configuration of a sweep for cudaLaunchKernelEx: cooperative (the grid barrier needs every CTA resident),
// in clusters of `cluster` CTAs when cluster > 1.
struct SweepConfig {
  cudaLaunchAttribute attrs[2];
  cudaLaunchConfig_t cfg{};
  SweepConfig(int cluster, int grid, size_t smem, cudaStream_t st) {
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(rp::THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = cluster; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
    attrs[1].id = cudaLaunchAttributeCooperative;
    attrs[1].val.cooperative = 1;
    cfg.attrs = cluster > 1 ? attrs : attrs + 1;
    cfg.numAttrs = cluster > 1 ? 2 : 1;
  }
  SweepConfig(const SweepConfig&) = delete;   // cfg.attrs points into the object
};

static size_t fwd_smem_bytes(int NB) {
  using namespace rp;
  size_t NBp = NB + 1;
  return 1024 + (size_t)STAGES * (A_BYTES + (size_t)NB * 128) + (5 * UT * NBp + NB + 4) * sizeof(float) +
         (2 * STAGES + 2) * sizeof(uint64_t) + 64 + tc::acc_image_bytes(NB);
}

static size_t res_smem_bytes(int NB, int H) {
  using namespace rp;
  size_t NBp = NB + 1;
  return 1024 + (size_t)(H / 64) * (A_BYTES + (size_t)NB * 128) + (5 * UT * NBp + NB + 4) * sizeof(float) +
         (32 + STAGES + 2) * sizeof(uint64_t) + 64 + tc::acc_image_bytes(NB);
}

// Workspace of the resident forward: [4 KB control][W16: D*G*H*H halfs][h16: (D*T + 2)*B*H halfs].  h16 is the
// (D,T,B,H) sequence with one extra time step before it and one after it: the operands fp16(h0[0]) of the forward
// direction's step t = 0 ("t = -1") and fp16(h0[1]) of the reverse direction's step t = T-1 ("t = T").
// Returns the bytes; with a base, also the addresses (h16: of time step 0, after the extra step).
struct ResFwdWs { __half* w16; __half* h16; };
static size_t res_fwd_carve(int G, int T, int B, int H, int D, void* base, ResFwdWs& w) {
  size_t off = CTL_BYTES;
  w.w16 = carve<__half>(base, off, (size_t)D * G * H * H * 2);
  w.h16 = carve<__half>(base, off, ((size_t)D * T + 2) * B * H * 2);
  if (base) w.h16 += (size_t)B * H;
  return off;
}

// Resident forward variants: the fp16 copy of W_hh (in the workspace) and the tensor maps of it and of the fp16 h
// sequence.  `chunks`: 64-wide K chunks a CTA streams per step; a multiple of 4 takes one 3-D box per group of 4.
// A box of W_hh holds 16 units; its rows are [gate][unit], or with `unit_major` [unit][4 gate rows] (a (k, gate, unit)
// map, the GRU's fourth row of a unit is zero fill).
// `state` (the kernels' ST): the h sequence maps start one time step earlier, so that row (tp + 1) * B of direction
// d's map is time step tp, tp = -1 .. T; the extra steps are filled with fp16(h0) (zeros where h0 is null).
static int f16_weight_maps(const SeqArgs& a, PersistParams& p, void* ws, int chunks, cudaStream_t st,
                           bool unit_major = false, bool state = false) {
  using namespace rp;
  const int G = a.G;
  const size_t BH = (size_t)a.B * a.H;
  ResFwdWs w;
  res_fwd_carve(G, a.T, a.B, a.H, a.D, ws, w);
  p.h16 = w.h16;
  const size_t wn = (size_t)G * a.H * a.H;
  p.box3 = chunks % 4 == 0;
  const int rows = (a.T + (state ? 2 : 0)) * a.B;
  for (int d = 0; d < a.D; ++d) {
    int rc = f32_to_f16_rows(G * a.H, a.H, a.w_hh[d], a.H, w.w16 + (size_t)d * wn, a.H, nullptr, st);
    if (rc) return rc;
    rc = unit_major
             ? make_tmap_f16(&p.tmW[d], w.w16 + (size_t)d * wn, 3, a.H, G, a.H, (size_t)a.H * a.H, (size_t)a.H, 64, 4, UT)
             : make_tmap_f16(&p.tmW[d], w.w16 + (size_t)d * wn, 3, a.H, a.H, G, (size_t)a.H, (size_t)a.H * a.H, 64, UT, G);
    if (rc) return rc;
    __half* hbase = p.h16 + (size_t)d * a.T * BH - (state ? BH : 0);
    rc = make_tmap_f16(&p.tmV[d], hbase, 2, a.H, rows, 1, (size_t)a.H, 0, 64, a.B, 1);
    if (rc) return rc;
    if (p.box3) {   // rows b >= B of a box belong to the next time step (or are zero-filled): those N columns are discarded
      rc = make_tmap_f16(&p.tmV3[d], hbase, 3, 64, rows, a.H / 64, (size_t)a.H, 64, 64, p.NB, 4);
      if (rc) return rc;
    }
    if (state) {   // forward: the step before t = 0; reverse: the step after t = T - 1
      __half* slot = d == 0 ? p.h16 - BH : p.h16 + (size_t)a.D * a.T * BH;
      if (a.h0) rc = f32_to_f16_rows(a.B, a.H, a.h0 + (size_t)d * BH, a.H, slot, a.H, nullptr, st);
      else DS2_CHECK_CUDA(cudaMemsetAsync(slot, 0, BH * sizeof(__half), st));
      if (rc) return rc;
    }
  }
  return DS2_OK;
}

// ------------------------------------------------------------------------------------------------
// Backward sweep.  A CTA owns 16 hidden units of one direction: rows u0..u0+15 of W_hh^T (H x G*H)
// are the (16 valid of 64) M rows, the gate-gradient vector of the previously processed step
// dGh[t_next] (B x G*H) is the N operand, K = G*H:
//     dh_rec[u, b] = sum_k W_hh^T[u, k] * dGh[t_next][b, k]
// Epilogue: dh = dY[t] + dh_rec (+ carried terms), gate backward from the saved activations, the
// gate gradients overwrite the activations in place (and are the next step's N operand).  The
// cell-state / hidden-state carry of the owned units stays in shared memory for the whole sweep.
template <int RNN>
__global__ void __launch_bounds__(rp::THREADS, 1) rnn_bwd_persist_kernel(const __grid_constant__ PersistParams p) {
  using namespace rp;
  using namespace tc;
  constexpr int G = num_gates(RNN);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);   // 1 KB aligned, still __shared__
  const int NB = p.NB, B = p.B, T = p.T, H = p.H, D = p.D;
  const int B_BYTES = NB * 128, STAGE_BYTES = A_BYTES + B_BYTES;
  const int NBp = NB + 1;
  float* ex = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [UT][NBp] dh_rec
  float* cst = ex + 4 * UT * NBp;                                       // [UT][NBp] carried dc (LSTM) / dh (GRU)
  uint64_t* full = reinterpret_cast<uint64_t*>(cst + UT * NBp);
  uint64_t* empty = full + STAGES;
  uint64_t* accum_bar = empty + STAGES;
  float* acc_img = reinterpret_cast<float*>(accum_bar + 1);   // accumulator image (tc::wg_store_acc)

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int d = p.d0 + blockIdx.x / p.NT, tile = blockIdx.x % p.NT, u0 = tile * UT;
  const int GH = G * H;
  const int NK = GH / BK;
  unsigned int* ctr = p.bar + 32 * d;   // one 128-byte line per direction

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmW[d]);
    tma_prefetch_desc(&p.tmV[d]);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 128); }   // every MMA-warpgroup thread arrives
    mbar_init(accum_bar, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < UT * NBp; i += THREADS) { cst[i] = 0.f; ex[i] = 0.f; }
  __syncthreads();
  const uint32_t tx_bytes = (uint32_t)(UT * 128 + B * 128);

  if (warp == 8) {                                        // TMA producer
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int step = 1; step < T; ++step) {
        const int t = d == 0 ? T - 1 - step : step;
        const int tn = d == 0 ? t + 1 : t - 1;
        for (int c = 0; c < NK; ++c) {
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], tx_bytes);
          tma_load_2d(smem + s * STAGE_BYTES, &p.tmW[d], &full[s], c * BK, u0);
          if (c == 0) {
            grid_wait_counter(ctr, (unsigned int)p.NT * (unsigned int)step, p.err);
            fence_proxy_async_global();
            trace_stamp(p.trace, p.T, step, 0);
          }
          const int k0 = c * BK;
          if (RNN == DS2_RNN_GRU && k0 >= 2 * H)
            tma_load_2d(smem + s * STAGE_BYTES + A_BYTES, &p.tmV2[d], &full[s], k0 - 2 * H, tn * B);
          else
            tma_load_2d(smem + s * STAGE_BYTES + A_BYTES, &p.tmV[d], &full[s], d * GH + k0, tn * B);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // MMA warpgroup: accumulators in registers, handed to the epilogue warps as an image in shared memory; the
    // accumulator width (batch padded to 32 * NCH) is chosen once, outside the step loop
    with_nch<4>(NB, [&](auto nch) {
      WgAcc<1, decltype(nch)::value> acc;
      {
        // The issue chain is the critical path of a step: the loop is free of div/mod and descriptor construction.
        const uint64_t a_base = smem_desc_sw128(smem_u32(smem));
        const uint64_t b_base = smem_desc_sw128(smem_u32(smem + A_BYTES));
        const uint64_t stage_step = (uint64_t)(STAGE_BYTES >> 4);
        int s = 0;
        uint32_t ph = 0;
        for (int step = 1; step < T; ++step) {
          for (int c = 0; c < NK; ++c) {
            mbar_wait(&full[s], ph);
            if (c == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 1);
            if (c == NK - 1 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
            const uint64_t ad = a_base + (uint64_t)s * stage_step, bd = b_base + (uint64_t)s * stage_step;
            wg_mma4<false>(acc, ad, bd, c > 0);
            wg_release_all(&empty[s]);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
          wg_publish(acc, acc_img, accum_bar);
        }
      }
    });
  } else {                                                // warps 0..3: epilogue
    const int q = warp % 4;
    const int e = threadIdx.x;
    uint32_t acc_phase = 0;
    for (int step = 0; step < T; ++step) {
      const int t = d == 0 ? T - 1 - step : step;
      const int tp = d == 0 ? t - 1 : t + 1;
      const bool tp_in = tp >= 0 && tp < T;
      if (q == 0 && step > 0) {          // rows 0..15 of the accumulator live in lanes 0..15 of quarter 0
        mbar_wait(accum_bar, acc_phase);
        if (lane == 0) trace_stamp(p.trace, p.T, step, 3);
        for (int cb = 0; cb < NB; cb += 32) {
          float acc[32];
          tmem_ld32(acc_img, acc_pitch(NB), (uint32_t)cb, acc);
          if (lane < UT) {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (cb + j < B) ex[lane * NBp + cb + j] = acc[j];
          }
        }
      }
      if (step > 0) acc_phase ^= 1;
      named_bar_sync(1, 128);
      if (e == 0) trace_stamp(p.trace, p.T, step, 4);
      for (int pi = e; pi < UT * B; pi += 128) {
        const int ui = pi % UT, b = pi / UT;
        const bool valid = t < p.len[b];
        const bool pin = tp_in && (d == 0 || tp < p.len[b]);
        const size_t si = (((size_t)d * T + t) * B + b) * H + u0 + ui;
        const size_t sp = (((size_t)d * T + (tp_in ? tp : 0)) * B + b) * H + u0 + ui;
        float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + u0 + ui;
        if (!valid) {
#pragma unroll
          for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
          if (RNN == DS2_RNN_GRU) p.aux[si] = 0.f;
        } else {
          float dh = p.dy[((size_t)t * B + b) * H + u0 + ui] + ex[ui * NBp + b];
          if (RNN == DS2_RNN_LSTM) {
            const float c_prev = pin ? p.aux[sp] : 0.f;
            LstmBwd r = lstm_cell_bwd(gp[0], gp[H], gp[2 * H], gp[3 * H], p.aux[si], c_prev, dh, cst[ui * NBp + b]);
            gp[0] = r.di; gp[H] = r.df; gp[2 * H] = r.dg; gp[3 * H] = r.d_o;
            cst[ui * NBp + b] = r.dc_prev;
          } else if (RNN == DS2_RNN_GRU) {
            const float h_prev = pin ? p.hseq[sp] : 0.f;
            dh += cst[ui * NBp + b];
            GruBwd r = gru_cell_bwd(gp[0], gp[H], gp[2 * H], p.aux[si], h_prev, dh);
            gp[0] = r.dr; gp[H] = r.dz; gp[2 * H] = r.dxn;
            p.aux[si] = r.dhn;
            cst[ui * NBp + b] = r.dh_prev;
          } else {
            const float h = p.hseq[si];
            gp[0] = dh * (1.f - h * h);
          }
        }
      }
      named_bar_sync(1, 128);          // CTA-scope: every epilogue thread's stores happen-before thread 0's release
      if (e == 0) {
        fence_proxy_async_global();
        red_release(ctr, 1u);            // release is cumulative over the stores ordered by the named barrier
        trace_stamp(p.trace, p.T, step, 5);
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// Backward sweep, split-K variant (the fast path): a 4-CTA cluster owns 64 hidden units; CTA `ks` of
// the cluster reduces over a quarter of K = G*H, so every CTA issues the same number of MMAs per
// step as the forward sweep with all 64 M rows useful.  The partial sums (64 units x B) are exchanged
// through distributed shared memory in push form: accumulator-image quarter q of every CTA holds the rows that CTA q
// of the cluster finishes, so epilogue warp q sends them straight into CTA q's shared memory with
// st.async (16-byte stores that complete_tx on the destination's mbarrier); each CTA then reduces the four
// slices it received from its own shared memory and finishes its 16 units (gate backward, carried dc / dh).
// (The earlier pull form — publish, cluster barrier, 4-byte ld.shared::cluster reads with a 132-byte lane
// stride — cost ~5.9k of the 16k cycles per step.)
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float ld_dsmem(uint32_t addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity, int* err) {
  uint32_t ok = 0, it = 0;
  long long t0 = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(tc::smem_u32(bar)), "r"(parity)
        : "memory");
    if (!ok && (++it & 1023u) == 0) {            // bounded: a protocol fault must not hang the GPU
      if (t0 == 0) t0 = clock64();
      if (*(volatile int*)err) return;
      if (clock64() - t0 > rp::SPIN_LIMIT) { *(volatile int*)err = 1; return; }
    }
  }
}
// Layout of the partial tiles exchanged inside a cluster: [source CTA][group of 4 columns][row position][4 columns].
// A lane owns an accumulator row, so for one group of 4 columns the 32 lanes of a warp store to (nearly)
// consecutive 16-byte slots (with a [row][column] layout every lane hit a different 144-byte row: ~170 cycles
// per st.async instruction).  Rows are skewed by one slot every 8 rows so that the reader's rows r, r+4, r+8,
// r+12 fall into different banks, and a column group is padded by one slot.
__host__ __device__ constexpr int xt_cgs(int rows) { return (rows + rows / 8) * 4 + 4; }                   // floats / group
__host__ __device__ constexpr int xt_slice(int rows, int nb) { return (nb / 4) * xt_cgs(rows); }           // floats / source
__device__ __forceinline__ int xt_off(int rows, int row, int col) {
  return (col >> 2) * xt_cgs(rows) + (row + (row >> 3)) * 4 + (col & 3);
}
// 16-byte store into a cluster peer's shared memory that also counts 16 bytes on the peer's mbarrier
// (st.async: data and completion travel together, no fence / separate arrive on the critical path)
__device__ __forceinline__ void st_async_v4(uint32_t cluster_addr, float a, float b, float c, float d, uint32_t cluster_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(
                   cluster_addr),
               "f"(a), "f"(b), "f"(c), "f"(d), "r"(cluster_bar)
               : "memory");
}
// 1-D bulk copy global -> this CTA's shared memory that counts its bytes on an mbarrier (16-byte aligned, size % 16 == 0)
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   tc::smem_u32(smem_dst)),
               "l"(src), "r"(bytes), "r"(tc::smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// RES = true: the CTA's slice of W_hh^T (64 units x K/4, fp16, 128 KB at H=1024) is resident in shared memory and
// the streamed operand is a SCALED fp16 copy of the gate gradients: dg16 = fp16(dGh * S_s), S_s a power of two
// chosen from the maximum |dGh| of the previously processed step (global atomicMax, final at the grid barrier;
// step 0 uses the bound max|dY|), so that the largest value sits near 2^8: 256x of fp16 headroom above, 2^-22 of
// the maximum still representable below.  fp16 carries the same 10-bit mantissa as TF32.
__device__ __forceinline__ __half to_half_sat(float v) {
  return __float2half_rn(fminf(fmaxf(v, -65000.f), 65000.f));
}
// scale exponent for a step whose maximum magnitude is m: m * 2^sx lands in [2^7, 2^8).  Exponent arithmetic on
// the float bits (m = f * 2^(E-126), f in [0.5, 1)) instead of frexpf / ldexpf / a division on the critical path.
__device__ __forceinline__ int pow2_exp_for(unsigned int m_bits, int sx_prev) {
  if (m_bits == 0u || m_bits >= 0x7f800000u) return sx_prev;     // 0, inf, nan: keep the previous scale
  const int E = (int)((m_bits >> 23) & 0xffu);
  return max(-100, min(100, 134 - E));
}
__device__ __forceinline__ float pow2f(int ex) { return __int_as_float((ex + 127) << 23); }   // |ex| <= 100

// CL = CTAs per cluster = K split: 4 (64 units per cluster, MMA M = 64) or 8 (128 units, M = 128: the same
// number of CTAs, but each reduces only K/8, i.e. half as many MMA instructions on the per-step critical path).
// XG (RES, CL = 4 only): launched without clusters, as plain cooperative CTAs; a group of CL consecutive CTAs keeps
// the roles of a cluster, but the partial dh_rec tiles travel through L2 (`xbuf`, counted in `xcnt`) instead of
// distributed shared memory.  For GPUs whose GPCs cannot hold every cluster of the grid at once (a 132-SM H100 with
// both directions of H = 1024: 32 clusters of 4), so that both directions still run in one launch.  The MMAs, sums
// and scales are the cluster path's: the results are bit-identical.
template <int RNN, bool RES, int CL, int NKR_T = 0, bool XG = false>   // NKR_T: see rnn_fwd_splitk_kernel
__global__ void __launch_bounds__(rp::THREADS, 1) rnn_bwd_splitk_kernel(const __grid_constant__ PersistParams p) {
  using namespace rp;
  using namespace tc;
  static_assert(!XG || (RES && CL == 4), "the L2 exchange is built for the resident 4-CTA variant");
  constexpr int G = num_gates(RNN);
  constexpr int UM = UT * CL;                  // units per cluster (all M rows valid): 64 or 128 = MMA M
  constexpr int A_BYTES = UM * 128;            // one K chunk of the weight tile (shadows rp::A_BYTES)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);   // 1 KB aligned, still __shared__
  const int NB = p.NB, B = p.B, T = p.T, H = p.H, D = p.D;
  const int B_BYTES = NB * 128, STAGE_BYTES = A_BYTES + B_BYTES;
  const int NBp = NB + 1;
  const int NKR = NKR_T ? NKR_T : (G * H / CL) / 64;                     // resident: 64 fp16 of K per chunk
  const int NG = grp_count(NKR);
  const int ring_bytes = RES ? NKR * STAGE_BYTES : STAGES * STAGE_BYTES;
  float* part = reinterpret_cast<float*>(smem + ring_bytes);             // [CL sources] partial dh_rec tiles (xt_* layout)
  float* cst = part + CL * xt_slice(UT, NB);                             // [16][NBp] carried dc / dh
  int* lens_s = reinterpret_cast<int*>(cst + UT * NBp);
  unsigned int* cta_max = reinterpret_cast<unsigned int*>(lens_s + ((NB + 1) & ~1));   // [2] (8 bytes)
  uint64_t* full = reinterpret_cast<uint64_t*>(cta_max + 2);            // resident: one per group of 4 chunks
  uint64_t* empty = full + (RES ? 32 : STAGES);                          // resident: [0] = weights landed
  uint64_t* accum_bar = empty + STAGES;
  uint64_t* part_bar = accum_bar + 1;
  float* acc_img = reinterpret_cast<float*>(part_bar + 1);   // accumulator image (tc::wg_store_acc)

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int ks = blockIdx.x % CL;                         // rank in the cluster == K split
  const int cl = blockIdx.x / CL;
  const int NTc = H / UM;                                 // clusters per direction
  const int d = p.d0 + cl / NTc, ut = cl % NTc;
  const int GH = G * H;
  const int Kc = GH / CL, NK = Kc / BK;
  const int kbase = ks * Kc;
  const int u0 = ut * UM + ks * UT;                       // the 16 units this CTA finishes
  unsigned int* ctr = p.bar + 32 * d;
  const unsigned int n_arrive = (unsigned int)(NTc * CL);
  const int ss = xt_slice(UT, NB);                        // floats of one partial tile
  // XG: CTA index over both directions (the directions may be launched one at a time); tile (cta, source, parity)
  // of xbuf holds what `source` computed for `cta`'s units in a step of that parity
  const int grp0 = (d * NTc + ut) * CL;
  auto xslot = [&](int cta, int src, int step) { return p.xbuf + ((size_t)(cta * CL + src) * 2 + (step & 1)) * ss; };

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmW[d]);
    tma_prefetch_desc(&p.tmV[d]);
    for (int i = 0; i < (RES ? 32 : STAGES); ++i) mbar_init(&full[i], 1);
    for (int i = 0; i < STAGES; ++i) mbar_init(&empty[i], RES ? 1 : 128);   // streaming: every MMA-warpgroup thread arrives
    mbar_init(accum_bar, 1);
    mbar_init(part_bar, XG ? 2 : 1);                     // XG: the producer's bulk copies + the warp that kept its rows
    fence_barrier_init();
    cta_max[0] = 0u;
  }
  for (int i = threadIdx.x; i < UT * NBp; i += THREADS) cst[i] = 0.f;
  for (int i = threadIdx.x; i < NB; i += THREADS) lens_s[i] = i < B ? p.len[i] : 0;
  __syncthreads();
  if constexpr (!XG) cluster_sync_all();                 // peers' mbarriers are initialised
  const uint32_t tx_bytes = (uint32_t)(UM * 128 + B * 128);

  if (warp == 8) {                                        // TMA producer
    if (RES) {
      if (lane == 0) {
        mbar_arrive_expect_tx(&empty[0], (uint32_t)(NKR * UM * 128));
        for (int c = 0; c < NKR; ++c) tma_load_2d(smem + c * A_BYTES, &p.tmW[d], &empty[0], kbase + c * 64, ut * UM);
        uint8_t* vbuf = smem + NKR * A_BYTES;
        for (int step = 1; step < T; ++step) {
          const int t = d == 0 ? T - 1 - step : step;
          const int tn = d == 0 ? t + 1 : t - 1;
          grid_wait_counter(ctr, n_arrive * (unsigned int)step, p.err);
          fence_proxy_async_global();
          trace_stamp(p.trace, p.T, step, 0);
          // every CTA's atomicMax of the previous step precedes its arrival: the maximum is final.  It is handed
          // to the epilogue warps through shared memory (published before the last group is armed, so the
          // full-barrier -> MMA -> accumulator-barrier chain orders it) instead of a ~300-cycle global load
          // on their critical path.
          const unsigned int gm = ld_relaxed(p.gmax + (size_t)d * (T + 1) + step);
          for (int g = 0; g < NG; ++g) {
            uint64_t* fb = full + g;
            const int c0 = grp_begin(g), c1 = min(NKR, grp_begin(g + 1));
            if (c1 == NKR) *(volatile unsigned int*)(cta_max + 1) = gm;
            if (p.box3) {
              mbar_arrive_expect_tx(fb, (uint32_t)(4 * B_BYTES));
              tma_load_3d(vbuf + c0 * B_BYTES, &p.tmV3[d], fb, 0, tn * B, (d * GH + kbase) / 64 + c0);
            } else {
              mbar_arrive_expect_tx(fb, (uint32_t)((c1 - c0) * B * 128));
              for (int c = c0; c < c1; ++c)
                tma_load_2d(vbuf + c * B_BYTES, &p.tmV[d], fb, d * GH + kbase + c * 64, tn * B);
            }
          }
          trace_stamp(p.trace, p.T, step, 1);
          if constexpr (XG) {
            // The CL - 1 partial tiles the other CTAs of the group send for this step: wait for them (relaxed polling,
            // then an acquire fence, as at the step barrier) and copy them into `part` with bulk copies that complete
            // on part_bar.  The epilogue read `part` of the previous step before its arrival at the barrier passed
            // above.  Two parities of xbuf are enough: a source writes the tile of step s + 2 only after its MMAs of
            // step s + 2, i.e. after every CTA of the direction arrived at the barrier that ends step s + 1, and this
            // CTA's arrival there follows the copies of step s (its epilogue waited for them on part_bar).
            grid_wait_counter(p.xcnt + grp0 + ks, (unsigned int)((CL - 1) * step), p.err);
            fence_proxy_async_global();
            mbar_arrive_expect_tx(part_bar, (uint32_t)((CL - 1) * ss * 4));
            for (int src = 0; src < CL; ++src)
              if (src != ks) bulk_load(part + src * ss, xslot(grp0 + ks, src, step), (uint32_t)(ss * 4), part_bar);
          }
        }
      }
    } else
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int step = 1; step < T; ++step) {
        const int t = d == 0 ? T - 1 - step : step;
        const int tn = d == 0 ? t + 1 : t - 1;
        for (int c = 0; c < NK; ++c) {
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], tx_bytes);
          const int k0 = kbase + c * BK;
          tma_load_2d(smem + s * STAGE_BYTES, &p.tmW[d], &full[s], k0, ut * UM);
          if (c == 0) {
            grid_wait_counter(ctr, n_arrive * (unsigned int)step, p.err);
            fence_proxy_async_global();
            trace_stamp(p.trace, p.T, step, 0);
          }
          if (RNN == DS2_RNN_GRU && k0 >= 2 * H)
            tma_load_2d(smem + s * STAGE_BYTES + A_BYTES, &p.tmV2[d], &full[s], k0 - 2 * H, tn * B);
          else
            tma_load_2d(smem + s * STAGE_BYTES + A_BYTES, &p.tmV[d], &full[s], d * GH + k0, tn * B);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // MMA warpgroup: accumulators in registers, handed to the epilogue warps as an image in shared memory; the
    // accumulator width (batch padded to 32 * NCH) is chosen once, outside the step loop
    with_nch<UM == 64 ? 4 : 2>(NB, [&](auto nch) {
      WgAcc<UM / 64, decltype(nch)::value> acc;
      if (RES) {
        {
          const uint64_t a_base = warp_uniform(smem_desc_sw128(smem_u32(smem)));
          const uint64_t b_base = warp_uniform(smem_desc_sw128(smem_u32(smem + NKR * A_BYTES)));
          const uint64_t a_step = (uint64_t)(A_BYTES >> 4), b_step = (uint64_t)(B_BYTES >> 4);
          mbar_wait(&empty[0], 0);
          uint32_t ph = 0;
          for (int step = 1; step < T; ++step) {
            if constexpr (NKR_T > 0) {
              constexpr int NGT = (NKR_T + 3) / 4;
  #pragma unroll
              for (int g = 0; g < NGT; ++g) {
                mbar_wait(full + g, ph);
                if (g == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
                if (g == NGT - 1 && lane == 0) trace_stamp(p.trace, p.T, step, 3);
  #pragma unroll
                for (int c = 4 * g; c < (4 * g + 4 < NKR_T ? 4 * g + 4 : NKR_T); ++c) {
                  const uint64_t ad = a_base + (uint64_t)c * a_step, bd = b_base + (uint64_t)c * b_step;
                  wg_mma4<true>(acc, ad, bd, c > 0);
                }
              }
            } else {
              for (int g = 0; g < NG; ++g) {
                mbar_wait(full + g, ph);
                if (g == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
                const int c0 = grp_begin(g), c1 = min(NKR, grp_begin(g + 1));
                if (c1 == NKR && lane == 0) trace_stamp(p.trace, p.T, step, 3);
                for (int c = c0; c < c1; ++c) {
                  const uint64_t ad = a_base + (uint64_t)c * a_step, bd = b_base + (uint64_t)c * b_step;
                  wg_mma4<true>(acc, ad, bd, c > 0);
                }
              }
            }
            wg_publish(acc, acc_img, accum_bar);
            if (lane == 0) trace_stamp(p.trace, p.T, step, 4);
            ph ^= 1;
          }
        }
      } else
      {
        const uint64_t a_base = smem_desc_sw128(smem_u32(smem));
        const uint64_t b_base = smem_desc_sw128(smem_u32(smem + A_BYTES));
        const uint64_t stage_step = (uint64_t)(STAGE_BYTES >> 4);
        int s = 0;
        uint32_t ph = 0;
        for (int step = 1; step < T; ++step) {
          for (int c = 0; c < NK; ++c) {
            mbar_wait(&full[s], ph);
            if (c == 0 && lane == 0) trace_stamp(p.trace, p.T, step, 1);
            if (c == NK - 1 && lane == 0) trace_stamp(p.trace, p.T, step, 2);
            const uint64_t ad = a_base + (uint64_t)s * stage_step, bd = b_base + (uint64_t)s * stage_step;
            wg_mma4<false>(acc, ad, bd, c > 0);
            wg_release_all(&empty[s]);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
          wg_publish(acc, acc_img, accum_bar);
        }
      }
    });
  } else {                                                // warps 0..3: epilogue
    const int q = warp % 4;
    const int e = threadIdx.x;
    const int ul = lane & 15, half = lane >> 4;
    uint32_t acc_phase = 0, part_phase = 0;
    // Destination of this lane's accumulator row: the CTA that finishes the row's unit, slice ks (= this CTA's rank)
    // of its tile.  M = 64 (CL 4): accumulator-image quarter q holds rows 16q..16q+15 in lanes 0..15 -> CTA q, the 32 columns are
    // split with lane+16 by shuffle.  M = 128 (CL 8): lane l of quarter q holds row 32q+l -> CTA 2q + l/16, all 32
    // columns of the row are sent by that lane.
    const int dst_cta = CL == 4 ? q : 2 * q + half;
    const uint32_t dst_row = XG ? 0u : mapa_u32(smem_u32(part), (uint32_t)dst_cta) + (uint32_t)(ks * ss * 4);
    const uint32_t dst_bar = XG ? 0u : mapa_u32(smem_u32(part_bar), (uint32_t)dst_cta);
    const uint32_t part_tx = (uint32_t)(CL * UT * NB * 4);               // bytes this CTA receives per step
    // bias gradients: this thread's 4 units x (gate) sums over all steps of its batch column(s)
    float bsum[5][4];
#pragma unroll
    for (int i = 0; i < 5; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) bsum[i][j] = 0.f;
    // resident: s_cur scales what this step writes, s_prev un-scales what this step's MMAs consumed
    int sx_prev = 0, sx_cur = 0;
    // step-0 scale: |dGh| <= |dh| = |dY[t_first]| for every cell type
    if (RES) sx_cur = pow2_exp_for(__ldg(p.dymax + (d == 0 ? T - 1 : 0)), 0);
    float s_cur = pow2f(sx_cur), inv_prev = 1.f;
    const float nscale = (RES && p.dgn16) ? __ldg(p.nscale) : 1.f;
    for (int step = 0; step < T; ++step) {
      const int t = d == 0 ? T - 1 - step : step;
      const int tp = d == 0 ? t - 1 : t + 1;
      const bool tp_in = tp >= 0 && tp < T;
      float lmax = 0.f;
      // the scale of this step's outputs must also cover this step's own upstream gradient: a frame of dY far above
      // its neighbours would otherwise saturate the fp16 copy (the previous step's maximum knows nothing of it)
      const unsigned int dym = RES ? __ldg(p.dymax + t) : 0u;
      // Saved activations / states / dY of this step do not depend on the recurrence, and every gate gradient is
      // linear in dh (LSTM: in dh and dc): fetch them and reduce them to per-pair coefficients BEFORE waiting for
      // the MMAs, so that global-load and special-function latencies hide behind the tensor-core phase and only
      // a handful of multiplies remain on the critical path.
      //   LSTM  k = {o(1-tc^2), tc o(1-o), g i(1-i), c_prev f(1-f), i(1-g^2), f}   tc = tanh(c_t)
      //   GRU   k = {cn hn r(1-r), (h_prev-n) z(1-z), cn, cn r, z}                  cn = (1-z)(1-n^2)
      //   tanh  k = {1-h^2}
      // Thread e owns the 4 consecutive units 4*(e&3)..+3 of batch column (e>>2) [+32 per block]: every global
      // access is one 8- or 16-byte vector.
      constexpr int NPF = 4;
      const bool single = B <= 32;
      const int uq = 4 * (e & 3), b_own = e >> 2;
      auto ld4 = [](const float* src, float (&v)[NPF]) {
        const float4 x = *reinterpret_cast<const float4*>(src);
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
      };
      auto load_coefs = [&](int b, float (&k)[6][NPF], float (&dyv)[NPF], bool& valid) {
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j < NPF; ++j) k[i][j] = 0.f;
#pragma unroll
        for (int j = 0; j < NPF; ++j) dyv[j] = 0.f;
        valid = b < B && t < lens_s[b < B ? b : 0];
        if (!valid) return;
        const bool pin = tp_in && (d == 0 || tp < lens_s[b]);
        const size_t si = (((size_t)d * T + t) * B + b) * H + u0 + uq;
        const size_t sp = (((size_t)d * T + (tp_in ? tp : 0)) * B + b) * H + u0 + uq;
        const float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + u0 + uq;
        ld4(p.dy + ((size_t)t * B + b) * H + u0 + uq, dyv);
        if (RNN == DS2_RNN_LSTM) {
          float gi[NPF], gf[NPF], gg[NPF], go[NPF], c[NPF], c_prev[NPF] = {0.f, 0.f, 0.f, 0.f}, tc[NPF];
          ld4(gp, gi); ld4(gp + H, gf); ld4(gp + 2 * H, gg); ld4(gp + 3 * H, go);
          ld4(p.aux + si, c);
          if (pin) ld4(p.aux + sp, c_prev);
#pragma unroll
          for (int j = 0; j < NPF; ++j) tc[j] = ex2_ftz(-2.f * LOG2E * c[j]);
#pragma unroll
          for (int j = 0; j < NPF; ++j) tc[j] = fmaf(2.f, rcp_ftz(1.f + tc[j]), -1.f);   // the forward used this tanh
#pragma unroll
          for (int j = 0; j < NPF; ++j) {
            k[0][j] = go[j] * (1.f - tc[j] * tc[j]); k[1][j] = tc[j] * go[j] * (1.f - go[j]);
            k[2][j] = gg[j] * gi[j] * (1.f - gi[j]); k[3][j] = c_prev[j] * gf[j] * (1.f - gf[j]);
            k[4][j] = gi[j] * (1.f - gg[j] * gg[j]); k[5][j] = gf[j];
          }
        } else if (RNN == DS2_RNN_GRU) {
          float r[NPF], z[NPF], n[NPF], hn[NPF], h_prev[NPF] = {0.f, 0.f, 0.f, 0.f};
          ld4(gp, r); ld4(gp + H, z); ld4(gp + 2 * H, n);
          ld4(p.aux + si, hn);
          if (pin) ld4(p.hseq + sp, h_prev);
#pragma unroll
          for (int j = 0; j < NPF; ++j) {
            const float cn = (1.f - z[j]) * (1.f - n[j] * n[j]);
            k[0][j] = cn * hn[j] * r[j] * (1.f - r[j]); k[1][j] = (h_prev[j] - n[j]) * z[j] * (1.f - z[j]);
            k[2][j] = cn; k[3][j] = cn * r[j]; k[4][j] = z[j];
          }
        } else {
          float hv[NPF];
          ld4(p.hseq + si, hv);
#pragma unroll
          for (int j = 0; j < NPF; ++j) k[0][j] = 1.f - hv[j] * hv[j];
        }
      };
      float kc[6][NPF], pdy[NPF];
      bool pvalid = false;
      if (single) load_coefs(b_own, kc, pdy, pvalid);
      if (step > 0) {
        if (!XG && e == 0) mbar_arrive_expect_tx(part_bar, part_tx);   // arm this step's phase (peers may already have sent)
        // send this CTA's partial tile: row (16q + ul), 32 columns split over the two half-warps
        mbar_wait(accum_bar, acc_phase);
        if (RES) {
          // this step's MMAs ran, so the grid barrier was passed: the maximum of step-1 the producer forwarded is final
          const unsigned int gm = *(volatile unsigned int*)(cta_max + 1);
          sx_prev = sx_cur;
          sx_cur = pow2_exp_for(max(gm, dym), sx_prev);      // non-negative floats order like their bit patterns
          s_cur = pow2f(sx_cur);
          inv_prev = pow2f(-sx_prev);
        }
        if (e == 0) trace_stamp(p.trace, p.T, step, 5);
        // XG: own rows straight into the own tile, the other CTAs' rows into xbuf
        float* const xdst = XG ? (q == ks ? part + ks * ss : xslot(grp0 + q, ks, step)) : nullptr;
        for (int cb = 0; cb < NB; cb += 32) {
          float acc[32];
          tmem_ld32(acc_img, acc_pitch(NB), ((uint32_t)(q * 32) << 16) + (uint32_t)cb, acc);
          if (CL == 4) {
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const float hi = __shfl_sync(0xffffffffu, acc[16 + j], ul);
              v[j] = half ? hi : acc[j];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int c0 = cb + half * 16 + 4 * i;      // NB is a multiple of 8: a group of 4 columns is in or out
              if (c0 >= NB) continue;
              if constexpr (XG) {
                *reinterpret_cast<float4*>(xdst + xt_off(UT, ul, c0)) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
              } else {
                st_async_v4(dst_row + (uint32_t)(xt_off(UT, ul, c0) * 4), v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3], dst_bar);
              }
            }
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int c0 = cb + 4 * i;
              if (c0 < NB)
                st_async_v4(dst_row + (uint32_t)(xt_off(UT, ul, c0) * 4), acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3], dst_bar);
            }
          }
        }
        acc_phase ^= 1;
        if (e == 0) trace_stamp(p.trace, p.T, step, 6);
        if constexpr (XG) {
          // Publish: the warp's stores happen-before lane 0's release (bar.warp.sync orders memory among the lanes);
          // a destination counts one arrival per source CTA and step.  The warp that kept its rows arrives on
          // part_bar instead.
          __syncwarp();
          if (lane == 0) {
            if (q == ks) {
              mbar_arrive(part_bar);
            } else {
              fence_proxy_async_global();
              red_release(p.xcnt + grp0 + q, 1u);
            }
          }
        }
        mbar_wait_cluster(part_bar, part_phase, p.err);   // all CL slices of this CTA's units have landed
        part_phase ^= 1;
      }
      if (e == 0) trace_stamp(p.trace, p.T, step, 7);
      // Four cells: recurrent term = sum of the four received slices, gate backward from the coefficients.  The
      // scaled fp16 copy (resident variant: the next step's MMA operand) is stored here; the fp32 gate gradients,
      // which only the weight-gradient GEMMs after the sweep read, are returned in o[] (o[4]: GRU dGh_n).
      auto st_h4 = [&](__half* dst, const float (&v)[NPF]) {     // 4 scaled, saturated halves = one 8-byte store
        const __half2 lo = __halves2half2(to_half_sat(v[0] * s_cur), to_half_sat(v[1] * s_cur));
        const __half2 hi = __halves2half2(to_half_sat(v[2] * s_cur), to_half_sat(v[3] * s_cur));
        uint2 pk;
        pk.x = *reinterpret_cast<const unsigned int*>(&lo);
        pk.y = *reinterpret_cast<const unsigned int*>(&hi);
        *reinterpret_cast<uint2*>(dst) = pk;
      };
      auto finish4 = [&](int b, const float (&k)[6][NPF], const float (&dyv)[NPF], bool valid, float (&o)[5][NPF]) {
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
          for (int j = 0; j < NPF; ++j) o[i][j] = 0.f;
        if (b >= B) return;
        __half* hp16 = RES ? p.dg16 + (((size_t)t * B + b) * D + d) * GH + u0 + uq : nullptr;
        if (!valid) {
          if (RES) {
#pragma unroll
            for (int g = 0; g < G; ++g) *reinterpret_cast<uint2*>(hp16 + g * H) = make_uint2(0u, 0u);
          }
          return;
        }
        float dh[NPF];
#pragma unroll
        for (int j = 0; j < NPF; ++j) {
          float rec = 0.f;
          if (step > 0) {
            const float* pr = part + xt_off(UT, uq + j, b);
            rec = (pr[0] + pr[ss]) + (pr[2 * ss] + pr[3 * ss]);
            if (CL == 8) rec += (pr[4 * ss] + pr[5 * ss]) + (pr[6 * ss] + pr[7 * ss]);
          }
          dh[j] = dyv[j] + (RES ? rec * inv_prev : rec);
        }
        if (RNN == DS2_RNN_LSTM) {
#pragma unroll
          for (int j = 0; j < NPF; ++j) {
            const int ci = (uq + j) * NBp + b;
            const float dc = fmaf(dh[j], k[0][j], cst[ci]);
            o[0][j] = dc * k[2][j]; o[1][j] = dc * k[3][j]; o[2][j] = dc * k[4][j]; o[3][j] = dh[j] * k[1][j];
            cst[ci] = dc * k[5][j];
            lmax = fmaxf(lmax, fmaxf(fmaxf(fabsf(o[0][j]), fabsf(o[1][j])), fmaxf(fabsf(o[2][j]), fabsf(o[3][j]))));
          }
          if (RES) {
#pragma unroll
            for (int g = 0; g < 4; ++g) st_h4(hp16 + g * H, o[g]);
          }
        } else if (RNN == DS2_RNN_GRU) {
#pragma unroll
          for (int j = 0; j < NPF; ++j) {
            const int ci = (uq + j) * NBp + b;
            const float dht = dh[j] + cst[ci];
            o[0][j] = dht * k[0][j]; o[1][j] = dht * k[1][j]; o[2][j] = dht * k[2][j]; o[4][j] = dht * k[3][j];
            cst[ci] = dht * k[4][j];
            lmax = fmaxf(lmax, fmaxf(fabsf(o[0][j]), fmaxf(fabsf(o[1][j]), fabsf(o[4][j]))));
          }
          if (RES) {
            st_h4(hp16, o[0]); st_h4(hp16 + H, o[1]);
            st_h4(hp16 + 2 * H, o[4]);                        // the h-side n-gate gradient (dGh_n)
          }
        } else {
#pragma unroll
          for (int j = 0; j < NPF; ++j) {
            o[0][j] = dh[j] * k[0][j];
            lmax = fmaxf(lmax, fabsf(o[0][j]));
          }
          if (RES) st_h4(hp16, o[0]);
        }
      };
      auto st4 = [](float* dst, const float (&v)[NPF]) {
        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      };
      auto store_dg = [&](int b, const float (&o)[5][NPF]) {
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
          for (int j = 0; j < NPF; ++j) bsum[i][j] += o[i][j];
        float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + u0 + uq;
#pragma unroll
        for (int g = 0; g < G; ++g) st4(gp + g * H, o[g]);
        if (RNN == DS2_RNN_GRU) st4(p.aux + (((size_t)d * T + t) * B + b) * H + u0 + uq, o[4]);
        if (RES && p.dgn16) {
          // precision-16 GEMM operands, produced where the values are: the row-major copy (dX) as 8-byte stores, the
          // transposed copies (dW_ih, dW_hh: the reduction index t*B+b must be contiguous) as 2-byte stores — 8
          // consecutive batch columns of a (gate, unit) come from 8 lanes of a warp and are merged in L2
          const size_t TBs = (size_t)T * B, col = (size_t)t * B + b;
          __half* r16 = p.dgn16 + (col * D + d) * GH + u0 + uq;
          __half* t16 = p.dgn16T + ((size_t)d * GH + u0 + uq) * TBs + col;
#pragma unroll
          for (int g = 0; g < G; ++g) {
            __half h[NPF];
#pragma unroll
            for (int j = 0; j < NPF; ++j) {
              h[j] = to_half_sat(o[g][j] * nscale);
              t16[((size_t)g * H + j) * TBs] = h[j];
            }
            const __half2 lo = __halves2half2(h[0], h[1]), hi = __halves2half2(h[2], h[3]);
            uint2 pk;
            pk.x = *reinterpret_cast<const unsigned int*>(&lo);
            pk.y = *reinterpret_cast<const unsigned int*>(&hi);
            *reinterpret_cast<uint2*>(r16 + g * H) = pk;
          }
          if (RNN == DS2_RNN_GRU) {
            __half* a16 = p.auxn16T + ((size_t)d * H + u0 + uq) * TBs + col;
#pragma unroll
            for (int j = 0; j < NPF; ++j) a16[(size_t)j * TBs] = to_half_sat(o[4][j] * nscale);
          }
        }
      };
      // the non-resident variants stream the fp32 gate gradients themselves: nothing can be deferred there
      const bool defer = RES && p.defer && single;
      float sv[5][NPF];
      if (single) {
        finish4(b_own, kc, pdy, pvalid, sv);
        if (!defer && b_own < B) store_dg(b_own, sv);
      } else {
        for (int b = b_own; b < B; b += 32) {
          load_coefs(b, kc, pdy, pvalid);
          finish4(b, kc, pdy, pvalid, sv);
          store_dg(b, sv);
        }
      }
      if (RES) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        if (lane == 0) atomicMax(cta_max, __float_as_uint(lmax));   // non-negative floats order like uints
      }
      if (e == 0) trace_stamp(p.trace, p.T, step, 8);
      named_bar_sync(1, 128);
      if (e == 0) {
        trace_stamp(p.trace, p.T, step, 9);
        if (RES) {
          atomicMax(p.gmax + (size_t)d * (T + 1) + step + 1, cta_max[0]);
          cta_max[0] = 0u;
        }
        fence_proxy_async_global();
        trace_stamp(p.trace, p.T, step, 10);
        red_release(ctr, 1u);
        trace_stamp(p.trace, p.T, step, 11);
        trace_stamp_ns(p.trace, p.T, step, 12);
      }
      if (defer) {
        if (b_own < B) store_dg(b_own, sv);
        if (e == 0) trace_stamp(p.trace, p.T, step, 13);
      }
    }
    if (p.dbias[d]) {
      // lanes with equal (lane & 3) hold the same 4 units for different batch columns: reduce over lane bits 2..4,
      // then the four warps through shared memory in a fixed order (the exchange tiles are free now).  Every
      // (gate, unit) of these 16 units belongs to this CTA alone: plain stores, bit-repeatable, no atomics.
      named_bar_sync(1, 128);                              // everybody is done reading `part`
      float* red = part;                                   // [4 warps][5][16]
#pragma unroll
      for (int i = 0; i < 5; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float v = bsum[i][j];
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 8);
          v += __shfl_xor_sync(0xffffffffu, v, 16);
          if (lane < 4) red[(q * 5 + i) * 16 + 4 * lane + j] = v;
        }
      }
      named_bar_sync(1, 128);
      if (e < 80) {
        const int i = e / 16, u = e % 16;
        const float v = (red[(0 * 5 + i) * 16 + u] + red[(1 * 5 + i) * 16 + u]) +
                        (red[(2 * 5 + i) * 16 + u] + red[(3 * 5 + i) * 16 + u]);
        if (i < G) p.dbias[d][(size_t)i * H + u0 + u] = v;
        else if (RNN == DS2_RNN_GRU && i == 4) p.dbias_hn[d][u0 + u] = v;
      }
    }
  }
  __syncthreads();
  if constexpr (!XG) cluster_sync_all();                 // nobody exits while a peer may still read its tile
}

// ------------------------------------------------------------------------------------------------
// Forward sweep, split-K variant (LSTM / GRU, resident fp16 weights).  A 2-CTA cluster owns 32 hidden units of one
// direction; CTA `rank` multiplies the G*32 gate rows (MMA M = 128) with its half of K = H, so a step issues H/32 MMAs
// instead of H/16 — the single-thread MMA issue chain is the longest part of a step.  The MMA warpgroup finishes the
// step itself, from its accumulator registers: m-block 0 holds the rows of the 16 units this CTA owns, m-block 1 those
// of the peer's 16 units.  After its last MMA the warpgroup pushes m-block 1 into the peer's `part` tile with st.async
// (complete_tx on the peer's mbarrier), waits for the peer's tile of its own rows, adds it, the input projection and
// the biases, and runs gates + cell update.  Warps 0-3 only store the fp32 outputs that later kernels read (B <= 32,
// deferred saves), so that the warpgroup goes from a step's barrier arrival straight to the next step's MMAs.
//
// Rows of an m-block are ordered row = 4 * unit + gate: tmW is a (k, gate, unit) map and the GRU's fourth gate row of
// a unit is the map's zero fill.  Thread l of warp w of the warpgroup holds accumulator rows 16 w + l/4 + 8 hh, i.e.
// gate (l >> 2) & 3 of units 4 w + l/16 + 2 hh, at columns 8 i + 2 (l & 3) + e of every 32-column chunk.  A transpose
// across the four lanes l ^ {0, 4, 8, 12} (quad_transpose) leaves each lane all gates of four cells: units
// 4 w + l/16 + 2 hh, columns 8 ((l >> 2) & 3) + 2 (l & 3) + e (fwd_cell_unit / fwd_cell_col).
// NKR_T: compile-time number of K chunks per CTA (0 = runtime): with constant chunk offsets the MMA descriptors are
// "uniform base + immediate" and the issue loop needs no vector arithmetic / R2UR per instruction.
__device__ __forceinline__ int fwd_cell_unit(int tid, int k) { return 4 * (tid >> 5) + ((tid >> 4) & 1) + 2 * (k >> 1); }
__device__ __forceinline__ int fwd_cell_col(int tid, int k) { return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + (k & 1); }

// The four cells' values of a thread (k = 2 hh + e: unit 4 w + ub + 2 hh, column e, ub = (tid >> 4) & 1) regrouped
// with lane tid ^ 16: u4[j] = unit 4 w + j at column ub (fwd_store_col)
__device__ __forceinline__ int fwd_store_col(int tid) { return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + ((tid >> 4) & 1); }
__device__ __forceinline__ void fwd_units4(const float (&v)[4], float (&u4)[4]) {
  const bool ub = (threadIdx.x >> 4) & 1;
  const float r0 = __shfl_xor_sync(0xffffffffu, ub ? v[0] : v[1], 16);   // the partner's column, units of hh = 0
  const float r1 = __shfl_xor_sync(0xffffffffu, ub ? v[2] : v[3], 16);   //   ... hh = 1
  u4[0] = ub ? r0 : v[0];
  u4[1] = ub ? v[1] : r0;
  u4[2] = ub ? r1 : v[2];
  u4[3] = ub ? v[3] : r1;
}

// Blocks of 4 floats, v[4 i .. 4 i + 3] = block i, transposed across the lanes x = (lane >> 2) & 3 of a group
// l ^ {0, 4, 8, 12}: block i of lane x ends as block x of lane i (one shfl.xor round per lane bit; exact moves).
__device__ __forceinline__ void quad_transpose(float (&v)[16]) {
  const int x = (threadIdx.x >> 2) & 3;
#pragma unroll
  for (int bit = 0; bit < 2; ++bit) {
    const bool hi = (x >> bit) & 1;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i & (1 << bit)) continue;
      const int i1 = i | (1 << bit);   // of the pair (i, i1) a lane sends the block whose bit differs from its own
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float r = __shfl_xor_sync(0xffffffffu, hi ? v[4 * i + k] : v[4 * i1 + k], 4 << bit);
        if (hi) v[4 * i + k] = r;
        else v[4 * i1 + k] = r;
      }
    }
  }
}

// ST: initial state p.h0 / p.c0, as in rnn_fwd_persist_kernel (step 0 runs the MMAs on fp16(h0), cs starts from
// c0 / h0, the reverse direction's padded steps write fp16(h0) into h16).  The body is shared by the two kernels below.
template <int RNN, int NKR_T, bool ST>
__device__ __forceinline__ void fwd_splitk_sweep(const PersistParams& p) {
  using namespace rp;
  using namespace tc;
  constexpr int G = num_gates(RNN);
  constexpr int AW = 128 * 128;                          // bytes of one K chunk of the weight tile (128 rows)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);   // 1 KB aligned, still __shared__
  const int NB = p.NB, B = p.B, T = p.T, H = p.H, D = p.D;
  const int B_BYTES = NB * 128;
  const int NKR = NKR_T ? NKR_T : H / 128;               // 64-wide fp16 chunks of this CTA's K half
  const int NG = grp_count(NKR);
  // the peer's partial sums of this CTA's rows, in the accumulator's fragment order: [32-column chunk][4][thread]
  float4* part = reinterpret_cast<float4*>(smem + NKR * (AW + B_BYTES));
  // B <= 32 with deferred saves: the MMA warpgroup hands a step's fp32 outputs ([6][thread]) to warps 0-3 here
  const bool stage_saves = p.defer && NB == 32;
  float4* stage = part + NB * 16;
  uint64_t* full = reinterpret_cast<uint64_t*>(stage + (stage_saves ? 6 * 128 : 0));   // one per group of 4 chunks (<= 8)
  uint64_t* wbar = full + 8;
  uint64_t* part_bar = wbar + 1;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int rank = blockIdx.x & 1, cl = blockIdx.x >> 1;
  const int NTc = H / 32;                                // clusters per direction
  const int d = p.d0 + cl / NTc, U0 = (cl % NTc) * 32;   // first unit of the cluster
  const int u0 = U0 + rank * UT;                         // the 16 units this CTA finishes
  const int GH = G * H;
  unsigned int* ctr = p.bar + 32 * d;
  const unsigned int n_arrive = (unsigned int)(NTc * 2);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmW[d]);
    tma_prefetch_desc(&p.tmV[d]);
    for (int i = 0; i < 8; ++i) mbar_init(&full[i], 1);
    mbar_init(wbar, 1);
    mbar_init(part_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();                                     // the peer's mbarriers are initialised
  const int kc0 = rank * NKR;                             // first K chunk (of H/64) of this CTA

  if (warp == 8) {                                        // TMA producer
    if (lane == 0) {
      // weights once: per chunk 64 rows (16 units x 4 gate rows) of this CTA's units, then 64 of the peer's
      mbar_arrive_expect_tx(wbar, (uint32_t)(NKR * 2 * 64 * 128));
      for (int c = 0; c < NKR; ++c) {
        tma_load_3d(smem + c * AW, &p.tmW[d], wbar, (kc0 + c) * 64, 0, u0);
        tma_load_3d(smem + c * AW + 64 * 128, &p.tmW[d], wbar, (kc0 + c) * 64, 0, U0 + (rank ^ 1) * UT);
      }
      uint8_t* hbuf = smem + NKR * AW;
      for (int step = ST ? 0 : 1; step < T; ++step) {
        const int t = d == 0 ? step : T - 1 - step;
        const int tp = d == 0 ? t - 1 : t + 1;
        const int row = (ST ? tp + 1 : tp) * B;           // ST: the maps start at time step -1
        // every CTA has finished the previous step, this one included: its MMAs no longer read hbuf
        grid_wait_counter(ctr, n_arrive * (unsigned int)step, p.err);
        fence_proxy_async_global();
        trace_stamp(p.trace, p.T, step, 0);
        for (int g = 0; g < NG; ++g) {
          uint64_t* fb = full + g;
          const int c0 = grp_begin(g), c1 = min(NKR, grp_begin(g + 1));
          if (p.box3) {
            mbar_arrive_expect_tx(fb, (uint32_t)(4 * B_BYTES));
            tma_load_3d(hbuf + c0 * B_BYTES, &p.tmV3[d], fb, 0, row, kc0 + c0);
          } else {
            mbar_arrive_expect_tx(fb, (uint32_t)((c1 - c0) * B * 128));
            for (int c = c0; c < c1; ++c) tma_load_2d(hbuf + c * B_BYTES, &p.tmV[d], fb, (kc0 + c) * 64, row);
          }
        }
        trace_stamp(p.trace, p.T, step, 1);
      }
    }
  } else if (warp >= 4) {
    // MMA warpgroup: the accumulator width (batch padded to 32 * NCH) is chosen once, outside the step loop
    with_nch<2>(NB, [&](auto nch) {
      constexpr int NCH = decltype(nch)::value;
      const int tid = threadIdx.x - 128;
      // biases of the cells' two units (k >> 1): x-side + h-side summed, except the GRU n gate (r multiplies the h side)
      float bsum[G][2], bhn[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int u = u0 + fwd_cell_unit(tid, 2 * hh);
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float bx = p.b_ih[d][g * H + u], bh = p.b_hh[d][g * H + u];
          bsum[g][hh] = (RNN == DS2_RNN_GRU && g == 2) ? bx : bx + bh;
          if (RNN == DS2_RNN_GRU && g == 2) bhn[hh] = bh;
        }
        if (RNN != DS2_RNN_GRU) bhn[hh] = 0.f;
      }
      float cs[NCH][4];                                  // cell (LSTM) / hidden (GRU) state of the cells
#pragma unroll
      for (int c = 0; c < NCH; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          cs[c][k] = 0.f;
          if constexpr (ST) {
            const float* s0 = RNN == DS2_RNN_LSTM ? p.c0 : p.h0;
            const int b = 32 * c + fwd_cell_col(tid, k);
            if (s0 && b < B) cs[c][k] = s0[((size_t)d * B + b) * H + u0 + fwd_cell_unit(tid, k)];
          }
        }
      const uint32_t dst_part = mapa_u32(smem_u32(part + tid), (uint32_t)(rank ^ 1));
      const uint32_t dst_bar = mapa_u32(smem_u32(part_bar), (uint32_t)(rank ^ 1));
      const uint32_t part_tx = (uint32_t)(64 * NB * 4);
      const uint64_t a_base = warp_uniform(smem_desc_sw128(smem_u32(smem)));
      const uint64_t b_base = warp_uniform(smem_desc_sw128(smem_u32(smem + NKR * AW)));
      const uint64_t a_step = (uint64_t)(AW >> 4), b_step = (uint64_t)(B_BYTES >> 4);
      const bool defer = stage_saves;                   // two chunks: stored before the arrival
      mbar_wait(wbar, 0);
      uint32_t ph = 0, part_phase = 0;
      for (int step = 0; step < T; ++step) {
        const int t = d == 0 ? step : T - 1 - step;
        // input projections of the cells of column chunk c: independent of the recurrence, so with one chunk they
        // are loaded before the MMA chain and land while it runs (with two, both chunks' accumulators and
        // projections would not fit in the registers together: each chunk's are loaded just before its cells)
        float gx[NCH][G][4];
        auto load_gx = [&](int c) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int b = 32 * c + fwd_cell_col(tid, k);
            const float* src = p.gates + (((size_t)t * B + b) * D + d) * GH + u0 + fwd_cell_unit(tid, k);
#pragma unroll
            for (int g = 0; g < G; ++g) gx[c][g][k] = b < B ? src[(size_t)g * H] : 0.f;
          }
        };
        if (NCH == 1) load_gx(0);
        // s[c][4 g + k]: recurrent sum of gate g of cell k (without ST zero at the first step: h_{-1} = 0)
        float s[NCH][16];
        if (ST || step > 0) {
          if (tid == 0) mbar_arrive_expect_tx(part_bar, part_tx);   // arm this step's phase (the peer may already have sent)
          WgAcc<2, NCH> acc;                             // live from the first MMA of the step to the partial sums only
          if constexpr (NKR_T > 0) {
            constexpr int NGT = (NKR_T + 3) / 4;
#pragma unroll
            for (int g = 0; g < NGT; ++g) {
              mbar_wait(full + g, ph);
              if (g == 0 && tid == 0) trace_stamp(p.trace, p.T, step, 2);
              if (g == NGT - 1 && tid == 0) trace_stamp(p.trace, p.T, step, 3);
#pragma unroll
              for (int c = 4 * g; c < (4 * g + 4 < NKR_T ? 4 * g + 4 : NKR_T); ++c) {
                const uint64_t ad = a_base + (uint64_t)c * a_step, bd = b_base + (uint64_t)c * b_step;
                wg_mma4<true>(acc, ad, bd, c > 0);
              }
            }
          } else {
            for (int c = 0; c < NKR; ++c) {
              if (c % 4 == 0) {                          // first chunk of a group
                mbar_wait(full + c / 4, ph);
                if (c == 0 && tid == 0) trace_stamp(p.trace, p.T, step, 2);
                if (c + 4 >= NKR && tid == 0) trace_stamp(p.trace, p.T, step, 3);
              }
              const uint64_t ad = a_base + (uint64_t)c * a_step, bd = b_base + (uint64_t)c * b_step;
              wg_mma4<true>(acc, ad, bd, c > 0);
            }
          }
          wg_commit();
          wg_wait<0>();
          ph ^= 1;
          if (tid == 0) trace_stamp(p.trace, p.T, step, 4);
          // the peer's rows, straight from the registers: thread tid of the peer reads back exactly these 16 values
#pragma unroll
          for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int j = 0; j < 4; ++j)
              st_async_v4(dst_part + (uint32_t)((4 * c + j) * 128 * 16), acc.r[1][c][4 * j], acc.r[1][c][4 * j + 1],
                          acc.r[1][c][4 * j + 2], acc.r[1][c][4 * j + 3], dst_bar);
          if (tid == 0) trace_stamp(p.trace, p.T, step, 6);
          mbar_wait_cluster(part_bar, part_phase, p.err);   // the peer's partial tile of this CTA's rows has landed
          part_phase ^= 1;
          if (tid == 0) trace_stamp(p.trace, p.T, step, 7);
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            // pr[rank] + pr[rank ^ 1]: IEEE addition is commutative, so this is pr[0] + pr[1] bit for bit
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 pv = part[(4 * c + j) * 128 + tid];
              s[c][4 * j] = acc.r[0][c][4 * j] + pv.x;
              s[c][4 * j + 1] = acc.r[0][c][4 * j + 1] + pv.y;
              s[c][4 * j + 2] = acc.r[0][c][4 * j + 2] + pv.z;
              s[c][4 * j + 3] = acc.r[0][c][4 * j + 3] + pv.w;
            }
            quad_transpose(s[c]);
          }
        } else {
#pragma unroll
          for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int i = 0; i < 16; ++i) s[c][i] = 0.f;
        }
        // ---- gates + cell update of 4 cells: o[0..G-1] saved gate values, o[4] aux (LSTM c / GRU h_n + b_hn), o[5] h
        auto cell4 = [&](int c, const float (&x)[G][4], const float (&r4)[16], float (&cp)[4], float (&o)[6][4]) {
          float pre[G][4], hn[4], hval[4];
          bool valid[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int b = 32 * c + fwd_cell_col(tid, k);
            valid[k] = b < B && t < p.len[b];
          }
#pragma unroll
          for (int g = 0; g < G; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float r = r4[4 * g + k];
              if (RNN == DS2_RNN_GRU && g == 2) { hn[k] = r + bhn[k >> 1]; pre[g][k] = x[g][k] + bsum[g][k >> 1]; }
              else pre[g][k] = (x[g][k] + r) + bsum[g][k >> 1];
            }
          if (RNN == DS2_RNN_LSTM) {
            float a[4][4], cval[4], th[4];
            // i, f, o: sigmoid; g: tanh = 2 sigmoid(2x) - 1  (one EX2 + one RCP per value, stage by stage)
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int k = 0; k < 4; ++k) a[g][k] = ex2_ftz((g == 2 ? -2.f * LOG2E : -LOG2E) * pre[g][k]);
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int k = 0; k < 4; ++k) a[g][k] = rcp_ftz(1.f + a[g][k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              a[2][k] = fmaf(2.f, a[2][k], -1.f);
              cval[k] = valid[k] ? fmaf(a[1][k], cp[k], a[0][k] * a[2][k]) : 0.f;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) th[k] = ex2_ftz(-2.f * LOG2E * cval[k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) th[k] = rcp_ftz(1.f + th[k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              hval[k] = valid[k] ? a[3][k] * fmaf(2.f, th[k], -1.f) : 0.f;
              if (valid[k]) cp[k] = cval[k];
#pragma unroll
              for (int g = 0; g < 4; ++g) o[g][k] = valid[k] ? a[g][k] : 0.f;
              o[4][k] = cval[k];
            }
          } else {
            float a[2][4], nv[4];
#pragma unroll
            for (int g = 0; g < 2; ++g)
#pragma unroll
              for (int k = 0; k < 4; ++k) a[g][k] = ex2_ftz(-LOG2E * pre[g][k]);
#pragma unroll
            for (int g = 0; g < 2; ++g)
#pragma unroll
              for (int k = 0; k < 4; ++k) a[g][k] = rcp_ftz(1.f + a[g][k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) nv[k] = ex2_ftz(-2.f * LOG2E * fmaf(a[0][k], hn[k], pre[2][k]));
#pragma unroll
            for (int k = 0; k < 4; ++k) nv[k] = rcp_ftz(1.f + nv[k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float nval = valid[k] ? fmaf(2.f, nv[k], -1.f) : 0.f;
              hval[k] = valid[k] ? fmaf(a[1][k], cp[k] - nval, nval) : 0.f;
              if (valid[k]) cp[k] = hval[k];
              o[0][k] = valid[k] ? a[0][k] : 0.f; o[1][k] = valid[k] ? a[1][k] : 0.f; o[2][k] = nval; o[3][k] = 0.f;
              o[4][k] = valid[k] ? hn[k] : 0.f;
            }
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) o[5][k] = hval[k];
        };
        // the fp32 saves that only later kernels read (gates when training, aux, the sequence output)
        // Outputs of a chunk's cells regrouped by one shfl.xor(16) round (fwd_units4): the lane with
        // ub = (tid >> 4) & 1 ends with column e = ub of the four consecutive units 4 w .. 4 w + 3, so every global
        // store of a thread is one 16-byte (fp32) or 8-byte (fp16) vector; scattered 4-byte stores cost more memory
        // transactions, and the release at the step barrier waits for them.
        const int bs = fwd_store_col(tid);               // + 32 c
        const int us = u0 + 4 * (tid >> 5);
        auto store4 = [&](int c, const float (&o)[6][4]) {
          const int b = 32 * c + bs;
          if (b < B) {
            const size_t so = (((size_t)d * T + t) * B + b) * H + us;
            float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + us;
            *reinterpret_cast<float4*>(p.aux + so) = make_float4(o[4][0], o[4][1], o[4][2], o[4][3]);
            if (p.training) {
#pragma unroll
              for (int g = 0; g < G; ++g)
                *reinterpret_cast<float4*>(gp + (size_t)g * H) = make_float4(o[g][0], o[g][1], o[g][2], o[g][3]);
            }
            *reinterpret_cast<float4*>(p.hseq + so) = make_float4(o[5][0], o[5][1], o[5][2], o[5][3]);
          }
        };
        float sv[NCH][6][4];
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          if (NCH > 1) load_gx(c);
          float o[6][4];
          cell4(c, gx[c], s[c], cs[c], o);
#pragma unroll
          for (int q = 0; q < 6; ++q)
            if (q < G || q >= 4) fwd_units4(o[q], sv[c][q]);
          const int b = 32 * c + bs;
          if (b < B) {                                   // fp16 h_t: the MMA operand of the next step
            float h4[4] = {sv[c][5][0], sv[c][5][1], sv[c][5][2], sv[c][5][3]};
            if constexpr (ST) {
              if (d == 1 && t >= p.len[b]) {
#pragma unroll
                for (int j = 0; j < 4; ++j) h4[j] = p.h0 ? p.h0[((size_t)B + b) * H + us + j] : 0.f;
              }
            }
            const __half2 lo = __floats2half2_rn(h4[0], h4[1]), hi = __floats2half2_rn(h4[2], h4[3]);
            uint2 pk;
            pk.x = *reinterpret_cast<const unsigned int*>(&lo);
            pk.y = *reinterpret_cast<const unsigned int*>(&hi);
            *reinterpret_cast<uint2*>(p.h16 + (((size_t)d * T + t) * B + b) * H + us) = pk;
          }
          if (!defer) store4(c, sv[c]);
        }
        if (tid == 0) trace_stamp(p.trace, p.T, step, 8);
        named_bar_sync(1, 128);          // CTA-scope: every thread's h16 stores happen-before thread 0's release
        if (tid == 0) {
          trace_stamp(p.trace, p.T, step, 9);
          fence_proxy_async_global();
          trace_stamp(p.trace, p.T, step, 10);
          red_release(ctr, 1u);
          trace_stamp(p.trace, p.T, step, 11);
          trace_stamp_ns(p.trace, p.T, step, 12);
        }
        if (defer) {                     // after the arrival: hand the saves to warps 0-3 (stage_saves)
          named_bar_sync(4, 256);        // they have stored the previous step's
#pragma unroll
          for (int q = 0; q < 6; ++q)
            if (q < G || q >= 4) stage[q * 128 + tid] = make_float4(sv[0][q][0], sv[0][q][1], sv[0][q][2], sv[0][q][3]);
          asm volatile("bar.arrive 3, 256;" ::: "memory");
        }
      }
    });
  } else if (stage_saves) {
    // warps 0-3: the fp32 saves (gates, aux, sequence output) of the cells of MMA-warpgroup thread threadIdx.x, off
    // the warpgroup's path from one step's arrival to the next step's MMAs
    const int tid = threadIdx.x;
    const int b = fwd_store_col(tid), us = u0 + 4 * (tid >> 5);
    for (int step = 0; step < T; ++step) {
      const int t = d == 0 ? step : T - 1 - step;
      asm volatile("bar.arrive 4, 256;" ::: "memory");   // the staging buffer is free
      named_bar_sync(3, 256);                            // this step's outputs are in it
      if (b < B) {
        const size_t so = (((size_t)d * T + t) * B + b) * H + us;
        float* gp = p.gates + (((size_t)t * B + b) * D + d) * GH + us;
        *reinterpret_cast<float4*>(p.aux + so) = stage[4 * 128 + tid];
        if (p.training) {
#pragma unroll
          for (int g = 0; g < G; ++g) *reinterpret_cast<float4*>(gp + (size_t)g * H) = stage[g * 128 + tid];
        }
        *reinterpret_cast<float4*>(p.hseq + so) = stage[5 * 128 + tid];
      }
      if (tid == 0) trace_stamp(p.trace, p.T, step, 13);
    }
  }
  __syncthreads();
  cluster_sync_all();                                     // nobody exits while the peer may still write into its tile
}

template <int RNN, int NKR_T = 0>
__global__ void __launch_bounds__(rp::THREADS, 1) rnn_fwd_splitk_kernel(const __grid_constant__ PersistParams p) {
  fwd_splitk_sweep<RNN, NKR_T, false>(p);
}
// With an initial state: compile-time chunk counts only, and only those whose ST body compiles without local memory
// (ptxas: H / 128 = 1, 5, 8, 9, i.e. H = 128, 640, 1024, 1152).  The runtime-count body and the counts 2-4, 6, 7, 10
// spill 8-596 bytes at the 168-register cap; a state at those H takes the 16-unit kernel where it fits.
constexpr int FWD_SPLITK_MAX_NKR = 10;   // shared memory holds at most 10 chunks (H = 1280)
template <int RNN, int NKR_T>
__global__ void __launch_bounds__(rp::THREADS, 1) rnn_fwd_splitk_state_kernel(const __grid_constant__ PersistParams p) {
  static_assert(NKR_T == 1 || NKR_T == 5 || NKR_T == 8 || NKR_T == 9, "an ST chunk count that compiles without spills");
  fwd_splitk_sweep<RNN, NKR_T, true>(p);
}
template <int RNN>
static const SweepKernel fwd_splitk_state_kernels[FWD_SPLITK_MAX_NKR] = {
    rnn_fwd_splitk_state_kernel<RNN, 1>, nullptr, nullptr, nullptr, rnn_fwd_splitk_state_kernel<RNN, 5>, nullptr,
    nullptr, rnn_fwd_splitk_state_kernel<RNN, 8>, rnn_fwd_splitk_state_kernel<RNN, 9>, nullptr};

static size_t fwd_splitk_smem_bytes(int NB, int H, bool defer) {
  return 1024 + (size_t)(H / 128) * (128 * 128 + (size_t)NB * 128) + (size_t)64 * NB * sizeof(float) +
         (defer && NB == 32 ? 6 * 128 * 16 : 0) + 10 * sizeof(uint64_t) + 64;
}

static size_t splitk_smem_bytes(int NB, int CL) {
  using namespace rp;
  size_t NBp = NB + 1;
  return 1024 + (size_t)STAGES * ((size_t)UT * CL * 128 + (size_t)NB * 128) +
         ((size_t)CL * xt_slice(UT, NB) + UT * NBp + NB + 16) * sizeof(float) + (2 * STAGES + 3) * sizeof(uint64_t) + 64 + tc::acc_image_bytes(NB);
}

// out[t] = float bits of max |x[t, :]| over the n floats of row t (one CTA per row, x >= 0 after fabs -> uint order)
__global__ void absmax_rows_kernel(size_t n, const float* __restrict__ x, unsigned int* __restrict__ out) {
  __shared__ float red[8];
  const float* row = x + (size_t)blockIdx.x * n;
  float m = 0.f;
  for (size_t i = threadIdx.x * 4; i + 3 < n; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  for (size_t i = (n & ~(size_t)3) + threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(row[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x / 32); ++w) m = fmaxf(m, red[w]);
    out[blockIdx.x] = __float_as_uint(m);
  }
}

static size_t splitk_res_smem_bytes(int NB, int Kc, int CL) {
  using namespace rp;
  size_t NBp = NB + 1;
  return 1024 + (size_t)(Kc / 64) * ((size_t)UT * CL * 128 + (size_t)NB * 128) +
         ((size_t)CL * xt_slice(UT, NB) + UT * NBp + NB + 16) * sizeof(float) + (32 + STAGES + 3) * sizeof(uint64_t) + 64 + tc::acc_image_bytes(NB);
}

// Workspace of the resident backward: [4 KB control][gmax: D*(T+1) uints][dymax: T uints][W^T fp16: D*H*GH]
// [dg16: T*B*D*GH][xbuf: D*H/16 CTAs x 4 sources x 2 parities partial tiles, the 4-CTA L2 exchange].
// Returns the bytes; with a base, also the addresses.
struct ResBwdWs { unsigned int* gmax; unsigned int* dymax; __half* wT16; __half* dg16; float* xbuf; };
static size_t res_bwd_carve(int G, int T, int B, int H, int D, void* base, ResBwdWs& w) {
  const size_t GH = (size_t)G * H;
  size_t off = CTL_BYTES;
  w.gmax = carve<unsigned int>(base, off, (size_t)D * (T + 1) * 4);
  w.dymax = carve<unsigned int>(base, off, (size_t)T * 4);
  w.wT16 = carve<__half>(base, off, (size_t)D * H * GH * 2);
  w.dg16 = carve<__half>(base, off, (size_t)T * B * D * GH * 2);
  w.xbuf = carve<float>(base, off, (size_t)D * (H / 16) * 4 * 2 * xt_slice(rp::UT, sweep_nb(B)) * sizeof(float));
  return off;
}

size_t rnn_sweep_tc_workspace_bytes(int rnn, int T, int B, int H, int D) {
  const int G = num_gates(rnn);
  ResFwdWs fw;
  ResBwdWs bw;
  const size_t fwd = res_fwd_carve(G, T, B, H, D, nullptr, fw), bwd = res_bwd_carve(G, T, B, H, D, nullptr, bw);
  return (fwd > bwd ? fwd : bwd) + 256;
}

// ------------------------------------------------------------------------------------------------
// Selection and launch.  choose_fwd / choose_bwd pick a sweep variant without side effects (they call nothing but the
// shared-memory opt-ins and the occupancy queries); launch_sweep then prepares that variant's operands and launches it.

// The operand preparation a sweep variant needs before its launch
enum class Prep {
  FWD_F32,   // maps over the fp32 W_hh and hseq: the 16-unit streaming forward
  FWD_F16,   // fp16 W_hh in the workspace (f16_weight_maps): the resident and the split-K forward
  BWD_F32,   // the fp32 W_hh^T and its maps (bwd_f32_maps): the 16-unit and the split-K streaming backward
  BWD_F16,   // the fp16 W_hh^T only, max |dY[t]| and the resident backward's workspace: the resident split-K backward
};

// A sweep variant as the selection returns it
struct SweepChoice {
  SweepKernel kern;
  int cluster;                      // 0: cooperative launch; 1, 2, 4, 8: cudaLaunchKernelEx in clusters of that size
  int group;                        // CTAs that share one slice of hidden units: 1, 2, 4 or 8 (not always a cluster)
  int per_dir;                      // CTAs per direction
  size_t smem;
  Prep prep;
  int rank;                         // place in the order of preference: a refused launch resumes the selection after it
  const char* what = nullptr;       // the variant, in the messages of a refused launch ...
  const char* fallback = nullptr;   // ... and what runs instead, when a refusal deserves a warning
  int launches = 0;                 // 1: both directions in one launch; D: one launch per direction
};

// CTAs of `c` that can be co-resident in a grid of `grid`: one per SM at most (see one_cta_per_sm), in whole clusters
// (a cluster cannot span two GPCs).  -1 when the device rejects the clusters or a CTA would need more than the 227 KB of
// shared memory it can have.  The occupancy queries depend on the opt-in: call opt_in_smem first.
static int co_resident(const SweepChoice& c, int grid, cudaStream_t st, int* fit) {
  *fit = -1;
  if (c.smem > 227 * 1024) return DS2_OK;
  if (c.cluster <= 1) {
    int per_sm = 0;
    DS2_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, c.kern, rp::THREADS, c.smem));
    *fit = per_sm * device_sm_count();
    return DS2_OK;
  }
  SweepConfig cfg(c.cluster, grid, c.smem, st);
  int max_clusters = 0;
  if (cudaOccupancyMaxActiveClusters(&max_clusters, c.kern, &cfg.cfg) == cudaSuccess) *fit = max_clusters * c.cluster;
  else (void)cudaGetLastError();
  return DS2_OK;
}

// The grid barrier needs every CTA of a launch resident: c->launches = 1 when both directions' CTAs can be, D when
// only one direction's can and `per_dir_ok`, otherwise 0 (the variant does not fit)
static int place(SweepChoice* c, int D, bool per_dir_ok, cudaStream_t st) {
  int fit = 0;
  if (int rc = co_resident(*c, D * c->per_dir, st, &fit)) return rc;
  c->launches = fit >= D * c->per_dir ? 1 : (per_dir_ok && fit >= c->per_dir ? D : 0);
  return DS2_OK;
}

// Forward: the 2-CTA split-K kernel (half the MMA chain per step), the 16-unit resident kernel, the 16-unit streaming
// kernel (DESIGN §5.1), from rank `from` on.  Returns 0 with *c, 1 when no variant takes the shape, or an error.
template <int RNN>
static int choose_fwd(const SeqArgs& a, size_t ws_bytes, int from, cudaStream_t st, SweepChoice* c) {
  constexpr int R = RNN == DS2_RNN_TANH ? DS2_RNN_LSTM : RNN;   // the split-K kernels exist for LSTM and GRU
  const int H = a.H, NB = sweep_nb(a.B);
  // NB: columns of the MMA warpgroup's accumulator (WgAcc), 64 for the variants with MMA M = 128
  if (H % 32 != 0 || NB > 128 || a.T < 2 || !vec_ok(a.gates, a.hseq, a.aux)) return 1;
  const bool state = a.h0 || a.c0;
  ResFwdWs w;
  const bool resident = !env_flag("DS2_NO_RESIDENT", 0) && ws_bytes >= res_fwd_carve(a.G, a.T, a.B, H, a.D, nullptr, w);
  if (from <= 0 && resident && RNN != DS2_RNN_TANH && env_flag("DS2_FWD_SPLITK", 1) && H % 128 == 0 && H / 128 <= 32 &&
      NB <= 64 && a.aux) {
    // with an initial state only the chunk counts of fwd_splitk_state_kernels; H = 1024: unrolled issue loop
    const SweepKernel* sk = fwd_splitk_state_kernels<R>;
    const int nkr = H / 128;
    const SweepKernel kern = state ? (nkr <= FWD_SPLITK_MAX_NKR ? sk[nkr - 1] : nullptr)
                                   : (H == 1024 ? rnn_fwd_splitk_kernel<R, 8> : rnn_fwd_splitk_kernel<R, 0>);
    static DeviceOnce once;
    if (kern) {
      if (int rc = opt_in_smem(once, {rnn_fwd_splitk_kernel<R, 8>, rnn_fwd_splitk_kernel<R, 0>, sk[0], sk[4], sk[7], sk[8]}))
        return rc;
      *c = {kern, 2, 2, H / 16, one_cta_per_sm(fwd_splitk_smem_bytes(NB, H, sweep_defer_default())), Prep::FWD_F16, 0,
            "split-K forward sweep", "the 16-unit kernel"};
      if (int rc = place(c, a.D, true, st)) return rc;
      if (c->launches) return DS2_OK;
    }
  }
  if (from <= 1 && resident && H % 64 == 0 && H / 64 <= 32) {
    static DeviceOnce once;
    if (int rc = opt_in_smem(once, {rnn_fwd_persist_kernel<RNN, true>, rnn_fwd_persist_kernel<RNN, true, true>})) return rc;
    *c = {state ? rnn_fwd_persist_kernel<RNN, true, true> : rnn_fwd_persist_kernel<RNN, true>, 0, 1, H / 16,
          one_cta_per_sm(res_smem_bytes(NB, H)), Prep::FWD_F16, 1};
    if (int rc = place(c, a.D, true, st)) return rc;
    if (c->launches) return DS2_OK;
  }
  // The streaming variant reads h_{t-1} from the fp32 output hseq, which must stay 0 at padded steps and has no step
  // before the first: it cannot carry an initial state.
  if (!state && ws_bytes >= CTL_BYTES) {
    static DeviceOnce once;
    if (int rc = opt_in_smem(once, {rnn_fwd_persist_kernel<RNN, false>})) return rc;
    *c = {rnn_fwd_persist_kernel<RNN, false>, 0, 1, H / 16, one_cta_per_sm(fwd_smem_bytes(NB)), Prep::FWD_F32, 2};
    if (int rc = place(c, a.D, true, st)) return rc;
    if (c->launches) return DS2_OK;
  }
  return 1;
}

// The split-K backward over groups of CL CTAs, resident (`res`) or streaming: *c with c->launches = 0 when the shape or
// the device does not take it.  8-CTA groups run only with both directions in one launch: they are only worth it when
// the directions run concurrently.
template <int RNN, int CL>
static int choose_bwd_splitk(const SeqArgs& a, size_t ws_bytes, bool res, cudaStream_t st, SweepChoice* c) {
  using namespace rp;
  const int GH = a.G * a.H, Kc = GH / CL, NB = sweep_nb(a.B);   // Kc: the K of one CTA
  if (a.H % (UT * CL) != 0 || GH % CL != 0 || NB > (CL == 8 ? 64 : 128)) return DS2_OK;
  if (CL == 8 && ((a.B + 7) / 8 * 8) % 16 != 0) return DS2_OK;   // M = 128: N % 16 == 0
  if (!vec_ok(a.gates, a.hseq, a.aux, a.dy)) return DS2_OK;
  if (!res) {
    if (Kc % BK != 0 || ws_bytes < CTL_BYTES) return DS2_OK;
    static DeviceOnce once;
    if (int rc = opt_in_smem(once, {rnn_bwd_splitk_kernel<RNN, false, CL>})) return rc;
    *c = {rnn_bwd_splitk_kernel<RNN, false, CL>, CL, CL, a.H / 16, one_cta_per_sm(splitk_smem_bytes(NB, CL)),
          Prep::BWD_F32, 0, "split-K backward sweep"};
    return place(c, a.D, CL != 8, st);
  }
  // <= 32 group barriers
  ResBwdWs w;
  if (Kc % 64 != 0 || Kc / 64 > 120 || ws_bytes < res_bwd_carve(a.G, a.T, a.B, a.H, a.D, nullptr, w)) return DS2_OK;
  // DS2_SPLITK_XCHG=cluster|global: force the partial-tile exchange through distributed shared memory or through L2
  const char* xe = getenv("DS2_SPLITK_XCHG");
  const bool force_cluster = xe && !strcmp(xe, "cluster"), force_global = xe && !strcmp(xe, "global");
  if (force_global && CL != 4) return DS2_OK;
  // H = 1024 (the BASELINE shapes): compile-time chunk count -> unrolled issue loop
  constexpr int G = num_gates(RNN);
  constexpr int NKU = (G * 1024 / CL) / 64;   // chunks per CTA at H = 1024: 16 / 12 / 4 (CL 4), 8 / 6 / 2 (CL 8)
  const bool unrolled = a.H == 1024;
  constexpr bool XG = CL == 4;                // only the 4-CTA variant has the L2 exchange
  static DeviceOnce once;
  int rc = opt_in_smem(once, {rnn_bwd_splitk_kernel<RNN, true, CL, NKU>, rnn_bwd_splitk_kernel<RNN, true, CL, 0>,
                              rnn_bwd_splitk_kernel<RNN, true, CL, NKU, XG>, rnn_bwd_splitk_kernel<RNN, true, CL, 0, XG>});
  if (rc) return rc;
  *c = {unrolled ? rnn_bwd_splitk_kernel<RNN, true, CL, NKU> : rnn_bwd_splitk_kernel<RNN, true, CL, 0>, CL, CL, a.H / 16,
        one_cta_per_sm(splitk_res_smem_bytes(NB, Kc, CL)), Prep::BWD_F16, 0, "resident split-K backward sweep",
        CL == 8 ? nullptr : "a slower variant"};
  // From what the device reports: (1) every cluster of the grid co-resident: cluster exchange, one launch.
  // (2) Otherwise the plain cooperative grid co-resident (a cluster cannot span two GPCs, so clusters of 4 can fail
  // where single CTAs fit: 32 clusters of 4 on a 132-SM H100): L2 exchange, one launch.  (3) Otherwise one launch
  // per direction with the cluster exchange.
  const int grid = a.D * c->per_dir;
  int fit = 0;
  if ((rc = co_resident(*c, grid, st, &fit))) return rc;
  if (fit < 0) return DS2_OK;
  if (XG && (force_global || (fit < grid && !force_cluster))) {
    SweepChoice xg = *c;
    xg.kern = unrolled ? rnn_bwd_splitk_kernel<RNN, true, CL, NKU, XG> : rnn_bwd_splitk_kernel<RNN, true, CL, 0, XG>;
    xg.cluster = 1;
    if ((rc = co_resident(xg, grid, st, &fit))) return rc;
    if (grid <= XCNT_MAX && (fit >= grid || force_global)) *c = xg;
    else if (force_global) return DS2_OK;
  }
  return place(c, a.D, CL != 8, st);
}

// Backward: the 8-CTA resident and streaming split-K kernels (DS2_SPLITK_CL=8, the default), the 4-CTA resident and
// streaming ones, the 16-unit kernel on W_hh^T (DESIGN §5.1), from rank `from` on.  Returns 0 with *c, 1 when no
// variant takes the shape, or an error.
template <int RNN>
static int choose_bwd(const SeqArgs& a, size_t ws_bytes, int from, cudaStream_t st, SweepChoice* c) {
  if (a.H % 32 != 0 || sweep_nb(a.B) > 128 || a.T < 2) return 1;
  const bool splitk = !env_flag("DS2_NO_SPLITK", 0), resident = !env_flag("DS2_NO_RESIDENT", 0);
  const bool cl8 = env_flag("DS2_SPLITK_CL", 8) == 8;
  for (int rank = from; rank < 5; ++rank) {
    int rc = DS2_OK;
    c->launches = 0;
    switch (rank) {
      case 0: if (splitk && cl8 && resident) rc = choose_bwd_splitk<RNN, 8>(a, ws_bytes, true, st, c); break;
      case 1: if (splitk && cl8) rc = choose_bwd_splitk<RNN, 8>(a, ws_bytes, false, st, c); break;
      case 2: if (splitk && resident) rc = choose_bwd_splitk<RNN, 4>(a, ws_bytes, true, st, c); break;
      case 3: if (splitk) rc = choose_bwd_splitk<RNN, 4>(a, ws_bytes, false, st, c); break;
      default:
        if (ws_bytes >= CTL_BYTES) {
          static DeviceOnce once;
          if ((rc = opt_in_smem(once, {rnn_bwd_persist_kernel<RNN>}))) return rc;
          *c = {rnn_bwd_persist_kernel<RNN>, 0, 1, a.H / 16, one_cta_per_sm(fwd_smem_bytes(sweep_nb(a.B))), Prep::BWD_F32, 0};
          rc = place(c, a.D, true, st);
        }
    }
    if (rc) return rc;
    if (c->launches) {
      c->rank = rank;
      return DS2_OK;
    }
  }
  return 1;
}

// Operands of the streaming backward kernels: the fp32 W_hh^T (H, G*H), transposed here into w_hhT, and the maps over
// it in boxes of `rows` unit rows, over the gate gradients (rows (t,b), full row width D*G*H: the direction offset is
// a coordinate) and, for the GRU, over the n-gate part of dGh in the aux buffer
static int bwd_f32_maps(const SeqArgs& a, PersistParams& p, int rows, cudaStream_t st) {
  using namespace rp;
  const int GH = a.G * a.H;
  for (int d = 0; d < a.D; ++d) {
    int rc = transpose(GH, a.H, a.w_hh[d], a.w_hhT[d], st);
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmW[d], a.w_hhT[d], a.H, GH, GH, rows, BK);
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmV[d], a.gates, a.T * a.B, a.D * GH, a.D * GH, a.B, BK);
    if (rc) return rc;
    if (a.G == 3) {
      rc = make_tmap_2d(&p.tmV2[d], a.aux + (size_t)d * a.T * a.B * a.H, a.T * a.B, a.H, a.H, a.B, BK);
      if (rc) return rc;
    }
  }
  return DS2_OK;
}

// The resident split-K backward: its workspace, the bias-gradient and fp16 gate-gradient outputs, the fp16 W_hh^T
// (the forward pass's copy when there is one, else made here by the same one-pass conversion), the maps over it and
// over the fp16 gate gradients, and max |dY[t]| per time step (the step-0 scale, and part of every later step's scale:
// spiky upstream gradients).  *ctl_bytes: the control block and gmax, which are zeroed.
static int prepare_res_bwd(const SweepChoice& c, const SeqArgs& a, void* ws, PersistParams& p, cudaStream_t st,
                           size_t* ctl_bytes) {
  using namespace rp;
  const int GH = a.G * a.H, CL = c.group;
  ResBwdWs w;
  res_bwd_carve(a.G, a.T, a.B, a.H, a.D, ws, w);
  p.gmax = w.gmax; p.dymax = w.dymax; p.dg16 = w.dg16; p.xbuf = w.xbuf;
  p.xcnt = reinterpret_cast<unsigned int*>(static_cast<char*>(ws) + CTL_XCNT);
  *ctl_bytes = reinterpret_cast<char*>(w.dymax) - static_cast<char*>(ws);
  for (int d = 0; d < a.D; ++d) { p.dbias[d] = a.dbias[d]; p.dbias_hn[d] = a.dbias_hn[d]; }
  if (a.f16_dg && a.f16_dgT && a.f16_scale && (a.G != 3 || a.f16_auxT)) {
    p.dgn16 = static_cast<__half*>(a.f16_dg);
    p.dgn16T = static_cast<__half*>(a.f16_dgT);
    p.auxn16T = static_cast<__half*>(a.f16_auxT);
    p.nscale = a.f16_scale;
  }
  const size_t wn = (size_t)a.H * GH;
  const bool cached = a.w_hhT16[0] && (a.D == 1 || a.w_hhT16[1]);   // fp16 W_hh^T left by the forward pass
  p.box3 = ((GH / CL) / 64) % 4 == 0;
  for (int d = 0; d < a.D; ++d) {
    const __half* wsrc = static_cast<const __half*>(a.w_hhT16[d]);
    if (!cached) {
      if (int rc = f32_to_f16_transpose(GH, a.H, a.w_hh[d], a.H, nullptr, 0, w.wT16 + (size_t)d * wn, GH, nullptr, st))
        return rc;
      wsrc = w.wT16 + (size_t)d * wn;
    }
    int rc = make_tmap_f16(&p.tmW[d], wsrc, 2, GH, a.H, 1, (size_t)GH, 0, 64, UT * CL, 1);
    if (rc) return rc;
    rc = make_tmap_f16(&p.tmV[d], p.dg16, 2, a.D * GH, a.T * a.B, 1, (size_t)a.D * GH, 0, 64, a.B, 1);
    if (rc) return rc;
    if (p.box3) {
      rc = make_tmap_f16(&p.tmV3[d], p.dg16, 3, 64, a.T * a.B, a.D * GH / 64, (size_t)a.D * GH, 64, 64, p.NB, 4);
      if (rc) return rc;
    }
  }
  DS2_LAUNCH(absmax_rows_kernel, a.T, 256, 0, st, (size_t)a.B * a.H, a.dy, p.dymax);
  return DS2_OK;
}

// Prepares the operands of the chosen variant, zeroes the control block, launches the sweep (c.launches launches:
// p.d0 is the first direction of each) and sweep_check_kernel.  cluster == 0: cudaLaunchCooperativeKernel, and a
// refused launch is an error.  cluster >= 1: cudaLaunchKernelEx in clusters of that size (1: no cluster dimension); a
// refused first launch returns 1, with a warning on stderr when c.fallback names what runs instead, and a refused
// second launch is an error.  `out` (backward): what the sweep produced besides the gate gradients.
static int launch_sweep(const SweepChoice& c, const SeqArgs& a, void* ws, cudaStream_t st, SweepBwdOut* out) {
  using namespace rp;
  const bool fwd = c.prep == Prep::FWD_F32 || c.prep == Prep::FWD_F16;
  PersistParams p = sweep_params(a, UT * c.group, fwd ? "DS2_TRACE_FWD" : "DS2_TRACE_BWD", ws);
  size_t ctl_bytes = CTL_BYTES;
  int rc = DS2_OK;
  switch (c.prep) {
    case Prep::FWD_F32:
      for (int d = 0; d < a.D && !rc; ++d) {
        rc = make_tmap_3d(&p.tmW[d], a.w_hh[d], a.H, a.H, a.G, (size_t)a.H, (size_t)a.H * a.H, BK, UT, a.G);
        if (!rc) rc = make_tmap_2d(&p.tmV[d], a.hseq + (size_t)d * a.T * a.B * a.H, a.T * a.B, a.H, a.H, a.B, BK);
      }
      break;
    case Prep::FWD_F16:
      rc = f16_weight_maps(a, p, ws, a.H / (64 * c.group), st, c.group == 2, a.h0 || a.c0);
      break;
    case Prep::BWD_F32:
      rc = bwd_f32_maps(a, p, UT * c.group, st);
      break;
    case Prep::BWD_F16:
      rc = prepare_res_bwd(c, a, ws, p, st, &ctl_bytes);
      break;
  }
  if (rc) return rc;
  DS2_CHECK_CUDA(cudaMemsetAsync(p.err, 0, ctl_bytes, st));
  const int grid = c.launches == 1 ? a.D * c.per_dir : c.per_dir;
  SweepConfig cfg(c.cluster, grid, c.smem, st);
  for (int li = 0; li < c.launches; ++li) {
    p.d0 = li;
    if (c.cluster == 0) {
      void* args[] = {&p};
      DS2_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)c.kern, dim3(grid), dim3(THREADS), args, c.smem, st));
    } else {
      const cudaError_t le = cudaLaunchKernelEx(&cfg.cfg, c.kern, p);
      if (le != cudaSuccess) {
        (void)cudaGetLastError();
        if (li == 0) {
          if (c.fallback)
            fprintf(stderr, "ds2_b200: WARNING %s launch failed (%s); using %s\n", c.what, cudaGetErrorString(le),
                    c.fallback);
          return 1;
        }
        set_error("%s: second launch failed: %s", c.what, cudaGetErrorString(le));
        return DS2_ERR_CUDA;
      }
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  DS2_LAUNCH(sweep_check_kernel, 1, 1, 0, st, p.err);
  if (out && c.prep == Prep::BWD_F16) *out = {a.dbias[0] != nullptr, p.dgn16 != nullptr};
  return DS2_OK;
}

// Launches the variant `choose` picks; when cudaLaunchKernelEx refuses it, the next one it picks after it
using ChooseSweep = int (*)(const SeqArgs&, size_t, int, cudaStream_t, SweepChoice*);
static int run_sweep(ChooseSweep choose, const SeqArgs& a, void* ws, size_t ws_bytes, cudaStream_t st,
                     SweepBwdOut* out = nullptr) {
  SweepChoice c{};
  for (int from = 0;; from = c.rank + 1) {
    int rc = choose(a, ws_bytes, from, st, &c);
    if (rc) return rc;
    rc = launch_sweep(c, a, ws, st, out);
    if (rc != 1) return rc;
  }
}

int rnn_sweep_fwd_tc(int rnn, const SeqArgs& a, void* ws, size_t ws_bytes, cudaStream_t st) {
  return run_sweep(rnn == DS2_RNN_LSTM ? choose_fwd<DS2_RNN_LSTM> : rnn == DS2_RNN_GRU ? choose_fwd<DS2_RNN_GRU>
                                                                                      : choose_fwd<DS2_RNN_TANH>,
                   a, ws, ws_bytes, st);
}

int rnn_sweep_bwd_tc(int rnn, const SeqArgs& a, void* ws, size_t ws_bytes, cudaStream_t st, SweepBwdOut* out) {
  *out = {false, false};
  return run_sweep(rnn == DS2_RNN_LSTM ? choose_bwd<DS2_RNN_LSTM> : rnn == DS2_RNN_GRU ? choose_bwd<DS2_RNN_GRU>
                                                                                      : choose_bwd<DS2_RNN_TANH>,
                   a, ws, ws_bytes, st, out);
}

}  // namespace ds2
