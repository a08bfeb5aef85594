// One BatchRNN layer (model.py:80-102): [BatchNorm1d over T*B rows] -> input projection GEMM ->
// recurrent sweep per direction with per-utterance length masking (replaces pack/pad, SURVEY §2b K8)
// -> sum of directions.  Backward: reverse sweep producing gate gradients in place of the saved
// gate activations, then three dense GEMMs (dW_ih, dW_hh, dX) and the BatchNorm backward.
//
// This file holds the host orchestration and the generic FFMA step kernels (any H, any B): one
// launch per time step covering both directions.  rnn_persistent_tc.cu provides the wgmma
// persistent sweep that replaces the step launches when the shape is eligible.  The backward gives
// every sweep the layer's W_hh and workspace for the fp32 W_hh^T (SeqArgs): a sweep that reads the
// transpose makes it.  The tensor-core backward sweep reports whether it also accumulated the bias
// gradients and wrote the fp16 gate-gradient copies (SweepBwdOut); the layer computes what it did not.
//
// reserve layout (floats):  gates (T,B,D,G*H) | hseq (D,T,B,H) | aux (D,T,B,H: LSTM cell states /
//                           GRU W_hn h + b_hn; absent for tanh) | bn mean,invstd (2*In)
#include <cuda_fp16.h>

#include <mutex>
#include <unordered_set>

#include "common.cuh"
#include "rnn_cells.cuh"
#include "rnn_common.cuh"

namespace ds2 {

constexpr int UT = 8;   // hidden units per CTA
constexpr int KC = 64;  // reduction chunk staged in shared memory

// grid (ceil(H/UT), D), block (32, UT)
template <int RNN>
__global__ void __launch_bounds__(32 * UT) rnn_step_fwd_kernel(SeqArgs a, int step) {
  constexpr int G = num_gates(RNN);
  __shared__ float hs[32][KC + 1];
  __shared__ float ws[G * UT][KC + 1];
  const int d = blockIdx.y, T = a.T, B = a.B, H = a.H, D = a.D;
  const int t = d == 0 ? step : T - 1 - step;
  const int tp = d == 0 ? t - 1 : t + 1;
  const bool tp_in = tp >= 0 && tp < T;
  const int lane = threadIdx.x, uy = threadIdx.y, tid = uy * 32 + lane;
  const int u0 = blockIdx.x * UT, u = u0 + uy;
  const float* __restrict__ W = a.w_hh[d];
  const float* hprev = a.hseq + ((size_t)d * T + (tp_in ? tp : 0)) * B * H;
  const float* cprev = a.aux ? a.aux + ((size_t)d * T + (tp_in ? tp : 0)) * B * H : nullptr;
  const int GH = G * H;

  for (int bt = 0; bt < (B + 31) / 32; ++bt) {
    const int b = bt * 32 + lane;
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    for (int k0 = 0; k0 < H; k0 += KC) {
      for (int idx = tid; idx < 32 * KC; idx += 32 * UT) {
        int kk = idx % KC, bb = idx / KC, gb = bt * 32 + bb, gk = k0 + kk;
        float v = 0.f;
        if (gb < B && gk < H) {
          bool pin = tp_in && (d == 0 || tp < a.len[gb]);
          v = pin ? hprev[(size_t)gb * H + gk] : (a.h0 ? a.h0[((size_t)d * B + gb) * H + gk] : 0.f);
        }
        hs[bb][kk] = v;
      }
      for (int idx = tid; idx < G * UT * KC; idx += 32 * UT) {
        int kk = idx % KC, rr = idx / KC, g = rr / UT, gu = u0 + rr % UT, gk = k0 + kk;
        ws[rr][kk] = (gu < H && gk < H) ? W[((size_t)g * H + gu) * H + gk] : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int kk = 0; kk < KC; ++kk) {
        float hv = hs[lane][kk];
#pragma unroll
        for (int g = 0; g < G; ++g) acc[g] = fmaf(hv, ws[g * UT + uy][kk], acc[g]);
      }
      __syncthreads();
    }
    if (b < B && u < H) {
      const bool valid = t < a.len[b];
      const bool pin = tp_in && (d == 0 || tp < a.len[b]);
      float* gp = a.gates + (((size_t)t * B + b) * D + d) * GH + u;
      float* hp = a.hseq + (((size_t)d * T + t) * B + b) * H + u;
      float* xp = a.aux ? a.aux + (((size_t)d * T + t) * B + b) * H + u : nullptr;
      const float* bi = a.b_ih[d] + u;
      const float* bh = a.b_hh[d] + u;
      if (!valid) {
        *hp = 0.f;
        if (xp) *xp = 0.f;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
      } else if constexpr (RNN == DS2_RNN_LSTM) {
        float c_prev = pin ? cprev[(size_t)b * H + u] : (a.c0 ? a.c0[((size_t)d * B + b) * H + u] : 0.f);
        LstmFwd r = lstm_cell_fwd(gp[0] + bi[0] + acc[0] + bh[0], gp[H] + bi[H] + acc[1] + bh[H],
                                  gp[2 * H] + bi[2 * H] + acc[2] + bh[2 * H],
                                  gp[3 * H] + bi[3 * H] + acc[3] + bh[3 * H], c_prev);
        gp[0] = r.i; gp[H] = r.f; gp[2 * H] = r.g; gp[3 * H] = r.o;
        *hp = r.h;
        *xp = r.c;
      } else if constexpr (RNN == DS2_RNN_GRU) {
        float h_prev = pin ? hprev[(size_t)b * H + u] : (a.h0 ? a.h0[((size_t)d * B + b) * H + u] : 0.f);
        float hn = acc[2] + bh[2 * H];
        GruFwd r = gru_cell_fwd(gp[0] + bi[0], gp[H] + bi[H], gp[2 * H] + bi[2 * H], acc[0] + bh[0],
                                acc[1] + bh[H], hn, h_prev);
        gp[0] = r.r; gp[H] = r.z; gp[2 * H] = r.n;
        *hp = r.h;
        *xp = hn;
      } else {
        float h = tanhf(gp[0] + bi[0] + acc[0] + bh[0]);
        gp[0] = h;
        *hp = h;
      }
    }
  }
}

// Backward step on the transposed recurrent matrix w_hhT[d] (H, G*H).
template <int RNN>
__global__ void __launch_bounds__(32 * UT) rnn_step_bwd_kernel(SeqArgs a, int step) {
  constexpr int G = num_gates(RNN);
  __shared__ float gs[32][KC + 1];
  __shared__ float ws[UT][KC + 1];
  const int d = blockIdx.y, T = a.T, B = a.B, H = a.H, D = a.D;
  const int t = d == 0 ? T - 1 - step : step;
  const int tn = d == 0 ? t + 1 : t - 1;   // processed just before (later in this direction's time)
  const int tp = d == 0 ? t - 1 : t + 1;   // source of the previous state in the forward sweep
  const bool tn_in = tn >= 0 && tn < T, tp_in = tp >= 0 && tp < T;
  const int lane = threadIdx.x, uy = threadIdx.y, tid = uy * 32 + lane;
  const int u0 = blockIdx.x * UT, u = u0 + uy;
  const int GH = G * H;
  const float* __restrict__ WT = a.w_hhT[d];

  for (int bt = 0; bt < (B + 31) / 32; ++bt) {
    const int b = bt * 32 + lane;
    float acc = 0.f;
    if (tn_in) {
      for (int k0 = 0; k0 < GH; k0 += KC) {
        for (int idx = tid; idx < 32 * KC; idx += 32 * UT) {
          int kk = idx % KC, bb = idx / KC, gb = bt * 32 + bb, row = k0 + kk;
          float v = 0.f;
          if (gb < B && row < GH) {
            if (RNN == DS2_RNN_GRU && row >= 2 * H)
              v = a.aux[(((size_t)d * T + tn) * B + gb) * H + (row - 2 * H)];   // dGh_n
            else
              v = a.gates[(((size_t)tn * B + gb) * D + d) * GH + row];
          }
          gs[bb][kk] = v;
        }
        for (int idx = tid; idx < UT * KC; idx += 32 * UT) {
          int kk = idx % KC, rr = idx / KC, gu = u0 + rr, row = k0 + kk;
          ws[rr][kk] = (gu < H && row < GH) ? WT[(size_t)gu * GH + row] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < KC; ++kk) acc = fmaf(gs[lane][kk], ws[uy][kk], acc);
        __syncthreads();
      }
    }
    if (b < B && u < H) {
      const bool valid = t < a.len[b];
      const bool pin = tp_in && (d == 0 || tp < a.len[b]);
      float* gp = a.gates + (((size_t)t * B + b) * D + d) * GH + u;
      const size_t si = (((size_t)d * T + t) * B + b) * H + u;
      const size_t sp = (((size_t)d * T + (tp_in ? tp : 0)) * B + b) * H + u;
      float* carry = a.carry ? a.carry + ((size_t)d * B + b) * H + u : nullptr;
      if (!valid) {
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
        if (RNN == DS2_RNN_GRU) a.aux[si] = 0.f;
      } else {
        float dh = a.dy[((size_t)t * B + b) * H + u] + acc;
        if constexpr (RNN == DS2_RNN_LSTM) {
          float c_prev = pin ? a.aux[sp] : 0.f;
          LstmBwd r = lstm_cell_bwd(gp[0], gp[H], gp[2 * H], gp[3 * H], a.aux[si], c_prev, dh, *carry);
          gp[0] = r.di; gp[H] = r.df; gp[2 * H] = r.dg; gp[3 * H] = r.d_o;
          *carry = r.dc_prev;
        } else if constexpr (RNN == DS2_RNN_GRU) {
          float h_prev = pin ? a.hseq[sp] : 0.f;
          dh += *carry;
          GruBwd r = gru_cell_bwd(gp[0], gp[H], gp[2 * H], a.aux[si], h_prev, dh);
          gp[0] = r.dr; gp[H] = r.dz; gp[2 * H] = r.dxn;
          a.aux[si] = r.dhn;
          *carry = r.dh_prev;
        } else {
          float h = a.hseq[si];
          gp[0] = dh * (1.f - h * h);
        }
      }
    }
  }
}

__global__ void sum_dirs_kernel(size_t n, int D, const float* __restrict__ hseq, float* __restrict__ y) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) y[i] = D == 2 ? hseq[i] + hseq[n + i] : hseq[i];
}

// hn[d,b,u] = state after the last valid step (fwd: t=len-1, reverse: t=0); h0 when len == 0
__global__ void final_state_kernel(int T, int B, int H, int D, const int32_t* __restrict__ len,
                                   const float* __restrict__ seq, const float* __restrict__ init,
                                   float* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)D * B * H) return;
  int u = (int)(i % H), b = (int)((i / H) % B), d = (int)(i / ((size_t)H * B));
  int L = min(len[b], T);
  float v;
  if (L <= 0) v = init ? init[i] : 0.f;
  else v = seq[(((size_t)d * T + (d == 0 ? L - 1 : 0)) * B + b) * H + u];
  out[i] = v;
}

// dst[f] = sum_r src[r*ld + f]   (dst zeroed by the caller); grid (ceil(F/32), chunks), block (32,8)
__global__ void colsum_strided_kernel(int rows, int F, const float* __restrict__ src, size_t ld,
                                      float* __restrict__ dst) {
  __shared__ float red[8][33];
  int f = blockIdx.x * 32 + threadIdx.x;
  int per = cdiv_dev(rows, gridDim.y), r0 = blockIdx.y * per, r1 = min(rows, r0 + per);
  float acc = 0.f;
  if (f < F)
    for (int r = r0 + threadIdx.y; r < r1; r += 8) acc += src[(size_t)r * ld + f];
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && f < F) {
    for (int i = 1; i < 8; ++i) acc += red[i][threadIdx.x];
    atomicAdd(&dst[f], acc);
  }
}

static int colsum(int rows, int F, const float* src, size_t ld, float* dst, cudaStream_t st) {
  DS2_CHECK_CUDA(cudaMemsetAsync(dst, 0, sizeof(float) * F, st));
  int chunks = rows / 256;
  chunks = chunks < 1 ? 1 : (chunks > 64 ? 64 : chunks);
  DS2_LAUNCH(colsum_strided_kernel, dim3(cdiv(F, 32), chunks), dim3(32, 8), 0, st, rows, F, src, ld, dst);
  return DS2_OK;
}

struct Reserve {
  float *gates, *hseq, *aux, *bnstats;
  __half* wT16;   // (D, H, G*H) fp16 W_hh^T, written by a tensor-core-mode training forward for the backward sweep
  size_t total;
};
static Reserve carve_reserve(const ds2_rnn_desc* d, float* base) {
  const size_t D = d->bidirectional ? 2 : 1, G = num_gates(d->rnn_type);
  const size_t TB = (size_t)d->T * d->B;
  Reserve r;
  size_t off = 0;
  r.gates = base + off; off += TB * D * G * d->H;
  r.hseq = base + off; off += D * TB * d->H;
  if (d->rnn_type != DS2_RNN_TANH) { r.aux = base + off; off += D * TB * d->H; } else r.aux = nullptr;
  r.bnstats = base + off; off += 2 * (size_t)d->In;
  off = (off + 3) & ~(size_t)3;                           // 16-byte aligned (TMA source)
  r.wT16 = reinterpret_cast<__half*>(base + off); off += (D * G * d->H * d->H + 1) / 2;
  r.total = off;
  return r;
}

// Which reserve buffers hold a valid fp16 W_hh^T (the forward pass that wrote it registers the pointer, the backward
// pass that consumes the reserve removes it): a backward without the copy simply converts the weights itself.
static std::mutex g_wT16_mu;
static std::unordered_set<const void*> g_wT16_valid;
static void wT16_set(const void* reserve, bool valid) {
  std::lock_guard<std::mutex> lk(g_wT16_mu);
  if (valid) g_wT16_valid.insert(reserve); else g_wT16_valid.erase(reserve);
}
static bool wT16_take(const void* reserve) {
  std::lock_guard<std::mutex> lk(g_wT16_mu);
  return g_wT16_valid.erase(reserve) > 0;
}

// Workspace of one pass, each buffer 256-byte aligned, then what the sweep and the fp32 / TF32 GEMMs use (gws):
//   fwd  xbn (TB,In) | sums (4*In doubles) | fp16: x16 (TB,In) | W_ih16 (D*G*H,In)
//   bwd  xbn | xhat | dxbn (TB,In) | sums (2*In doubles) | W_hh^T (H,G*H) per direction | carry (D,B,H) |
//        fp16: dG16 (TB,D*G*H) | dG16^T | x16^T (In,TB) | h16^T (D*H,TB) | GRU aux16^T (D*H,TB) | W_ih16^T (In,D*G*H) |
//        scale (16 floats)
// The BN buffers are there whether or not the layer has BatchNorm; the fp16 operand copies exactly when the pass runs
// its GEMMs on them (f16).  Returns the bytes; with a base, also the addresses.
struct LayerWs {
  float *xbn, *xhat, *dxbn;
  double* sums;
  float* w_hhT[2];
  float* carry;
  bool f16;
  __half *x16, *w16, *dG16, *dG16T, *x16T, *h16T, *aux16T, *w16T;
  float* scale;
};
static size_t layer_ws_carve(const ds2_rnn_desc* d, bool bwd, void* base, LayerWs& w) {
  const size_t D = d->bidirectional ? 2 : 1, TB = (size_t)d->T * d->B, In = d->In, H = d->H;
  const size_t GH = num_gates(d->rnn_type) * H, DGH = D * GH;
  w = LayerWs{};
  size_t off = 0;
  w.xbn = carve<float>(base, off, TB * In * 4);
  if (bwd) {
    w.xhat = carve<float>(base, off, TB * In * 4);
    w.dxbn = carve<float>(base, off, TB * In * 4);
  }
  w.sums = carve<double>(base, off, (bwd ? 2 : 4) * In * 8);
  if (bwd) {
    for (size_t dir = 0; dir < D; ++dir) w.w_hhT[dir] = carve<float>(base, off, GH * H * 4);
    w.carry = carve<float>(base, off, D * d->B * H * 4);
  }
  w.f16 = f16_gemm_mode() && d->B % 8 == 0 && In % 8 == 0 && H % 8 == 0 && (!bwd || TB >= 128);
  if (w.f16 && !bwd) {
    w.x16 = carve<__half>(base, off, TB * In * 2);
    w.w16 = carve<__half>(base, off, DGH * In * 2);
  } else if (w.f16) {
    w.dG16 = carve<__half>(base, off, TB * DGH * 2);
    w.dG16T = carve<__half>(base, off, TB * DGH * 2);
    w.x16T = carve<__half>(base, off, TB * In * 2);
    w.h16T = carve<__half>(base, off, D * H * TB * 2);
    if (d->rnn_type == DS2_RNN_GRU) w.aux16T = carve<__half>(base, off, D * H * TB * 2);
    w.w16T = carve<__half>(base, off, In * DGH * 2);
    w.scale = carve<float>(base, off, 16 * 4);
  }
  return off;
}

// wgmma persistent sweeps (rnn_persistent_tc.cu).  Return 1 when the shape is not eligible.
int rnn_sweep_fwd_tc(int rnn, const SeqArgs& a, void* ws, size_t ws_bytes, cudaStream_t st);
int rnn_sweep_bwd_tc(int rnn, const SeqArgs& a, void* ws, size_t ws_bytes, cudaStream_t st, SweepBwdOut* out);
size_t rnn_sweep_tc_workspace_bytes(int rnn, int T, int B, int H, int D);

static int sweep_fwd(int rnn, const SeqArgs& a, cudaStream_t st) {
  dim3 grid(cdiv(a.H, UT), a.D), block(32, UT);
  for (int s = 0; s < a.T; ++s) {
    if (rnn == DS2_RNN_LSTM) DS2_LAUNCH(rnn_step_fwd_kernel<DS2_RNN_LSTM>, grid, block, 0, st, a, s);
    else if (rnn == DS2_RNN_GRU) DS2_LAUNCH(rnn_step_fwd_kernel<DS2_RNN_GRU>, grid, block, 0, st, a, s);
    else DS2_LAUNCH(rnn_step_fwd_kernel<DS2_RNN_TANH>, grid, block, 0, st, a, s);
  }
  return DS2_OK;
}
// The FFMA backward reads the fp32 W_hh^T: transposed here, again if a tensor-core preparation made it before declining
static int sweep_bwd(int rnn, const SeqArgs& a, cudaStream_t st) {
  for (int dir = 0; dir < a.D; ++dir) {
    int rc = transpose(a.G * a.H, a.H, a.w_hh[dir], a.w_hhT[dir], st);
    if (rc) return rc;
  }
  dim3 grid(cdiv(a.H, UT), a.D), block(32, UT);
  for (int s = 0; s < a.T; ++s) {
    if (rnn == DS2_RNN_LSTM) DS2_LAUNCH(rnn_step_bwd_kernel<DS2_RNN_LSTM>, grid, block, 0, st, a, s);
    else if (rnn == DS2_RNN_GRU) DS2_LAUNCH(rnn_step_bwd_kernel<DS2_RNN_GRU>, grid, block, 0, st, a, s);
    else DS2_LAUNCH(rnn_step_bwd_kernel<DS2_RNN_TANH>, grid, block, 0, st, a, s);
  }
  return DS2_OK;
}

}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_rnn_reserve_floats(const ds2_rnn_desc* d) {
  if (!d) return 0;
  return carve_reserve(d, nullptr).total;
}

size_t ds2_rnn_workspace_bytes(const ds2_rnn_desc* d) {
  if (!d) return 0;
  const int D = d->bidirectional ? 2 : 1, TB = d->T * d->B, Kr = (d->T - 1) * d->B, In = d->In, H = d->H;
  const int GH = num_gates(d->rnn_type) * H, rows_x = d->rnn_type == DS2_RNN_GRU ? 2 * H : GH;
  // what each ds2_gemm of the layer needs (gemm_tc's operand transposes, gemm_simt's split-K slabs): the input
  // projection, dW_ih, dW_hh (GRU: its r, z rows and its n rows apart) and dX
  const size_t gemm[] = {ds2_gemm_workspace_bytes(0, 1, TB, GH, In), ds2_gemm_workspace_bytes(1, 0, GH, In, TB),
                         ds2_gemm_workspace_bytes(1, 0, rows_x, H, Kr), ds2_gemm_workspace_bytes(1, 0, H, H, Kr),
                         ds2_gemm_workspace_bytes(0, 0, TB, In, GH)};
  size_t gemm_max = 0;
  for (size_t g : gemm) gemm_max = g > gemm_max ? g : gemm_max;
  LayerWs w;
  const size_t fwd = layer_ws_carve(d, false, nullptr, w), bwd = layer_ws_carve(d, true, nullptr, w);
  return (fwd > bwd ? fwd : bwd) + rnn_sweep_tc_workspace_bytes(d->rnn_type, d->T, d->B, H, D) + gemm_max + 4096;
}

static int check_desc(const ds2_rnn_desc* d) {
  DS2_REQUIRE(d, "rnn: null descriptor");
  DS2_REQUIRE(d->rnn_type >= DS2_RNN_LSTM && d->rnn_type <= DS2_RNN_TANH, "rnn: unknown rnn_type %d", d->rnn_type);
  DS2_REQUIRE(d->T > 0 && d->B > 0 && d->In > 0 && d->H > 0, "rnn: bad shape T=%d B=%d In=%d H=%d", d->T, d->B,
              d->In, d->H);
  return DS2_OK;
}

int ds2_rnn_layer_fwd(const ds2_rnn_desc* d, const float* x, const int32_t* len, const float* bn_gamma,
                      const float* bn_beta, float* bn_rmean, float* bn_rvar, const float* const* w_ih,
                      const float* const* w_hh, const float* const* b_ih, const float* const* b_hh, const float* h0,
                      const float* c0, float* y, float* hn, float* cn, float* reserve, void* ws, size_t ws_bytes,
                      void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  DS2_REQUIRE(ws_bytes >= ds2_rnn_workspace_bytes(d), "rnn fwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  const int D = d->bidirectional ? 2 : 1, G = num_gates(d->rnn_type), T = d->T, B = d->B, In = d->In, H = d->H;
  const int TB = T * B, GH = G * H;
  Reserve R = carve_reserve(d, reserve);
  LayerWs W;
  const size_t used = layer_ws_carve(d, false, ws, W);
  void* gws = static_cast<char*>(ws) + used;
  const size_t gws_bytes = ws_bytes - used;
  const float* xin = x;
  if (bn_gamma) {
    rc = bn_rows_fwd(TB, In, x, bn_gamma, bn_beta, bn_rmean, bn_rvar, d->training, d->bn_momentum, d->bn_eps, W.xbn,
                     nullptr, R.bnstats, W.sums, st);
    if (rc) return rc;
    xin = W.xbn;
  }
  // input projection for every time step and both directions: gates[:, d*GH:(d+1)*GH] = xin . W_ih[d]^T
  {
    DS2_PROF("rnn_fwd_proj_gemm", st);
    bool done = false;
    if (W.f16) {
      // precision 16: fp16 copies of the layer input and of both directions' W_ih (stacked: one N = D*G*H GEMM)
      rc = f32_to_f16_rows(TB, In, xin, In, W.x16, In, nullptr, st);
      if (rc) return rc;
      for (int dir = 0; dir < D; ++dir) {
        rc = f32_to_f16_rows(GH, In, w_ih[dir], In, W.w16 + (size_t)dir * GH * In, In, nullptr, st);
        if (rc) return rc;
      }
      rc = gemm_tc_f16(TB, D * GH, In, 1.f, W.x16, In, W.w16, In, 0.f, R.gates, D * GH, nullptr, st);
      if (rc < 0) return rc;
      done = rc == 0;
    }
    for (int dir = 0; dir < D && !done; ++dir) {
      rc = ds2_gemm(0, 1, TB, GH, In, 1.f, xin, In, w_ih[dir], In, 0.f, R.gates + (size_t)dir * GH, D * GH, gws,
                    gws_bytes, stream);
      if (rc) return rc;
    }
  }
  SeqArgs a{};
  a.T = T; a.B = B; a.H = H; a.D = D; a.G = G; a.len = len;
  a.gates = R.gates; a.hseq = R.hseq; a.aux = R.aux;
  for (int dir = 0; dir < D; ++dir) { a.w_hh[dir] = w_hh[dir]; a.b_ih[dir] = b_ih[dir]; a.b_hh[dir] = b_hh[dir]; }
  a.h0 = h0; a.c0 = c0; a.training = d->training;
  {
    DS2_PROF("rnn_fwd_sweep", st);
    rc = 1;
    if (tensor_core_mode()) {
      rc = rnn_sweep_fwd_tc(d->rnn_type, a, gws, gws_bytes, st);
      if (rc == 1) note_fallback("forward sweep", d->rnn_type, T, B, H, D);
    }
    if (rc == 1) rc = sweep_fwd(d->rnn_type, a, st);
    if (rc) return rc;
  }
  // fp16 W_hh^T for the backward sweep of this step (the weights cannot change in between): one pass here instead of a
  // transpose + a conversion on the backward critical path; on the side stream when there is one
  wT16_set(reserve, false);
  if (d->training && tensor_core_mode() && H % 8 == 0) {
    cudaStream_t side = as_stream(g_side_stream.load());
    cudaStream_t cst = st;
    if (side) {
      rc = side_fork(st, side);
      if (rc) return rc;
      cst = side;
    }
    for (int dir = 0; dir < D; ++dir) {
      rc = f32_to_f16_transpose(GH, H, w_hh[dir], (size_t)H, nullptr, 0, R.wT16 + (size_t)dir * H * GH, (size_t)GH,
                                nullptr, cst);
      if (rc) return rc;
    }
    if (side) {
      rc = side_mark_workspace(reserve, side);
      if (rc) return rc;
    }
    wT16_set(reserve, true);
  }
  size_t n = (size_t)TB * H;
  int blocks = (int)((n + 1023) / 1024);
  blocks = blocks > 132 * 16 ? 132 * 16 : blocks;
  DS2_LAUNCH(sum_dirs_kernel, blocks, 256, 0, st, n, D, R.hseq, y);
  if (hn) DS2_LAUNCH(final_state_kernel, cdiv((long long)D * B * H, 256), 256, 0, st, T, B, H, D, len, R.hseq, h0, hn);
  if (cn && d->rnn_type == DS2_RNN_LSTM)
    DS2_LAUNCH(final_state_kernel, cdiv((long long)D * B * H, 256), 256, 0, st, T, B, H, D, len, R.aux, c0, cn);
  return DS2_OK;
}

int ds2_rnn_layer_bwd(const ds2_rnn_desc* d, const float* x, const int32_t* len, const float* bn_gamma,
                      const float* bn_beta, const float* const* w_ih, const float* const* w_hh,
                      const float* const* b_ih, const float* const* b_hh, const float* dy, float* reserve, float* dx,
                      float* dbn_gamma, float* dbn_beta, float* const* dw_ih, float* const* dw_hh,
                      float* const* db_ih, float* const* db_hh, void* ws, size_t ws_bytes, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  DS2_REQUIRE(ws_bytes >= ds2_rnn_workspace_bytes(d), "rnn bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  cudaStream_t side = as_stream(g_side_stream.load());
  if (side) {   // deferred weight-gradient GEMMs of an earlier layer may still read operand copies in this workspace
    rc = side_wait_for_workspace(ws, st);
    if (rc) return rc;
  }
  const int D = d->bidirectional ? 2 : 1, G = num_gates(d->rnn_type), T = d->T, B = d->B, In = d->In, H = d->H;
  const int TB = T * B, GH = G * H;
  Reserve R = carve_reserve(d, reserve);
  LayerWs W;
  const size_t used = layer_ws_carve(d, true, ws, W);
  void* gws = static_cast<char*>(ws) + used;
  const size_t gws_bytes = ws_bytes - used;

  // W_hh^T: the fp16 copy from the forward pass when there is one; the sweep that needs another form makes it
  const bool have_wT16 = tensor_core_mode() && wT16_take(reserve);
  if (have_wT16 && side) {   // written on the side stream by the forward pass
    rc = side_wait_for_workspace(reserve, st);
    if (rc) return rc;
  }
  DS2_CHECK_CUDA(cudaMemsetAsync(W.carry, 0, sizeof(float) * (size_t)D * B * H, st));
  SeqArgs a{};
  a.T = T; a.B = B; a.H = H; a.D = D; a.G = G; a.len = len;
  a.gates = R.gates; a.hseq = R.hseq; a.aux = R.aux;
  for (int dir = 0; dir < D; ++dir) {
    a.w_hh[dir] = w_hh[dir]; a.w_hhT[dir] = W.w_hhT[dir]; a.b_ih[dir] = b_ih[dir]; a.b_hh[dir] = b_hh[dir];
  }
  a.dy = dy; a.carry = W.carry; a.training = 1;
  if (have_wT16)
    for (int dir = 0; dir < D; ++dir) a.w_hhT16[dir] = R.wT16 + (size_t)dir * H * GH;
  // bias gradients are column sums of the gate gradients: the tensor-core sweep can accumulate them on the fly
  const bool gru = d->rnn_type == DS2_RNN_GRU;
  for (int dir = 0; dir < D; ++dir) {
    a.dbias[dir] = db_ih[dir];
    a.dbias_hn[dir] = gru ? db_hh[dir] + 2 * H : nullptr;
    DS2_CHECK_CUDA(cudaMemsetAsync(db_ih[dir], 0, sizeof(float) * GH, st));
    if (gru) DS2_CHECK_CUDA(cudaMemsetAsync(db_hh[dir] + 2 * H, 0, sizeof(float) * H, st));
  }
  // ---- precision 16: scaled fp16 copies of the gate gradients (row-major for dX, transposed for the weight
  // gradients), transposed fp16 copies of the layer input / the hidden sequence / W_ih; every GEMM K-major fp16.
  // The split-K sweep writes the gate-gradient copies itself (scale from max|dY|); after other sweeps they are
  // converted from the fp32 gate gradients.
  const bool f16 = W.f16;
  if (f16) {
    rc = pow2_scale_for(TB, H, dy, (size_t)H, reinterpret_cast<unsigned int*>(W.scale + 8), W.scale, 5, st);
    if (rc) return rc;
    a.f16_dg = W.dG16; a.f16_dgT = W.dG16T; a.f16_auxT = W.aux16T; a.f16_scale = W.scale;
  }
  SweepBwdOut made{false, false};
  {
    DS2_PROF("rnn_bwd_sweep", st);
    rc = 1;
    if (tensor_core_mode()) {
      rc = rnn_sweep_bwd_tc(d->rnn_type, a, gws, gws_bytes, st, &made);
      if (rc == 1) note_fallback("backward sweep", d->rnn_type, T, B, H, D);
    }
    if (rc == 1) rc = sweep_bwd(d->rnn_type, a, st);
    if (rc) return rc;
  }

  // the layer input as the projection saw it (BN applied) and its normalised form for the BN backward
  const float* xin = x;
  if (bn_gamma) {
    // recompute xhat and xbn from the saved batch statistics
    rc = bn_rows_reapply(TB, In, x, bn_gamma, bn_beta, R.bnstats, W.xbn, W.xhat, st);
    if (rc) return rc;
    xin = W.xbn;
  }
  DS2_PROF("rnn_bwd_gemms", st);
  if (f16) {
    const size_t DGH = (size_t)D * GH;
    if (!made.f16) {
      unsigned int* absmax_ws = reinterpret_cast<unsigned int*>(W.scale + 8);
      rc = pow2_scale_for(TB, (int)DGH, R.gates, DGH, absmax_ws, W.scale, 10, st);
      if (rc) return rc;
      rc = f32_to_f16_transpose(TB, (int)DGH, R.gates, DGH, W.dG16, DGH, W.dG16T, (size_t)TB, W.scale, st);
      if (rc) return rc;
    }
    for (int dir = 0; dir < D; ++dir) {
      rc = f32_to_f16_transpose(GH, In, w_ih[dir], (size_t)In, nullptr, 0, W.w16T + (size_t)dir * GH, DGH, nullptr, st);
      if (rc) return rc;
    }
  }
  // weight-gradient GEMMs: nobody needs dW_ih / dW_hh before the optimizer, so (precision-16 path, caller opted in)
  // they go to the side stream together with the operand copies only they read (x16T, h16T), ordered after the sweep,
  // and overlap the next layer's sweep.  The side stream then reads x / reserve until ds2_join_side_stream.
  cudaStream_t gst = st;
  if (f16 && side && d->deferred_dw) {
    rc = side_fork(st, side);
    if (rc) return rc;
    gst = side;
  }
  if (f16) {
    rc = f32_to_f16_transpose(TB, In, xin, (size_t)In, nullptr, 0, W.x16T, (size_t)TB, nullptr, gst);
    if (rc) return rc;
    for (int dir = 0; dir < D; ++dir) {
      rc = f32_to_f16_transpose(TB, H, R.hseq + (size_t)dir * TB * H, (size_t)H, nullptr, 0, W.h16T + (size_t)dir * H * TB,
                                (size_t)TB, nullptr, gst);
      if (rc) return rc;
      if (gru && !made.f16) {
        rc = f32_to_f16_transpose(TB, H, R.aux + (size_t)dir * TB * H, (size_t)H, nullptr, 0,
                                  W.aux16T + (size_t)dir * H * TB, (size_t)TB, W.scale, gst);
        if (rc) return rc;
      }
    }
  }
  // C (M,N) = A^T . B over K rows of (t,b): on the fp16 copies A16 (M,K) and B16 (N,K) (row stride TB) on gst when
  // the pass has them and gemm_tc_f16 takes the shape, otherwise with ds2_gemm on the fp32 A (K,M) and B (K,N) on st
  auto weight_grad = [&](int M, int N, int K, const __half* A16, const __half* B16, const float* A, int lda,
                         const float* Bf, int ldb, float* C, int ldc) {
    int r = 1;
    if (f16) {
      r = gemm_tc_f16(M, N, K, 1.f, A16, TB, B16, TB, 0.f, C, ldc, W.scale + 1, gst);
      if (r < 0) return r;
    }
    return r == 1 ? ds2_gemm(1, 0, M, N, K, 1.f, A, lda, Bf, ldb, 0.f, C, ldc, gws, gws_bytes, stream) : r;
  };
  // element `off` of an fp16 copy; null when the pass has no fp16 copies
  auto f16_at = [&](const __half* p, size_t off) { return f16 ? p + off : nullptr; };
  bool dx_done = false;
  if (f16 && dx) {   // dX = dG (TB x D*GH) . [W_ih fwd ; W_ih rev] : one K = D*G*H GEMM for both directions
    rc = gemm_tc_f16(TB, In, D * GH, 1.f, W.dG16, D * GH, W.w16T, D * GH, 0.f, bn_gamma ? W.dxbn : dx, In, W.scale + 1,
                     st);
    if (rc < 0) return rc;
    dx_done = rc == 0;
  }
  for (int dir = 0; dir < D; ++dir) {
    const float* dG = R.gates + (size_t)dir * GH;   // (TB, GH) with row stride D*GH : dGx
    const int ldg = D * GH;
    const float* aux_d = R.aux ? R.aux + (size_t)dir * TB * H : nullptr;   // GRU: dGh_n (TB,H)
    const float* hseq_d = R.hseq + (size_t)dir * TB * H;
    // dW_ih = dGx^T . xin
    rc = weight_grad(GH, In, TB, f16_at(W.dG16T, (size_t)dir * GH * TB), W.x16T, dG, ldg, xin, In, dw_ih[dir], In);
    if (rc) return rc;
    if (!made.dbias) {
      rc = colsum(TB, GH, dG, ldg, db_ih[dir], st);
      if (rc) return rc;
    }
    // dW_hh = sum_t dGh[t]^T . h_prev[t]; h_prev[t] = hseq[t-1] (forward) / hseq[t+1] (reverse).  In the transposed
    // fp16 copies a shift by one time step is a shift by B columns.
    const int Kr = (T - 1) * B;
    const size_t a_off = dir == 0 ? (size_t)B : 0, h_off = dir == 0 ? 0 : (size_t)B;
    const int rows_x = gru ? 2 * H : GH;   // rows whose dGh == dGx
    if (Kr > 0) {
      rc = weight_grad(rows_x, H, Kr, f16_at(W.dG16T, (size_t)dir * GH * TB + a_off),
                       f16_at(W.h16T, (size_t)dir * H * TB + h_off), dG + a_off * ldg, ldg, hseq_d + h_off * H, H,
                       dw_hh[dir], H);
      if (rc) return rc;
      if (gru) {
        rc = weight_grad(H, H, Kr, f16_at(W.aux16T, (size_t)dir * H * TB + a_off),
                         f16_at(W.h16T, (size_t)dir * H * TB + h_off), aux_d + a_off * H, H,
                         hseq_d + h_off * H, H, dw_hh[dir] + (size_t)2 * H * H, H);
        if (rc) return rc;
      }
    } else {
      DS2_CHECK_CUDA(cudaMemsetAsync(dw_hh[dir], 0, sizeof(float) * (size_t)GH * H, st));
    }
    if (gru) {
      DS2_CHECK_CUDA(cudaMemcpyAsync(db_hh[dir], db_ih[dir], sizeof(float) * 2 * H, cudaMemcpyDeviceToDevice, st));
      if (!made.dbias) {
        rc = colsum(TB, H, aux_d, H, db_hh[dir] + 2 * H, st);
        if (rc) return rc;
      }
    } else {
      DS2_CHECK_CUDA(cudaMemcpyAsync(db_hh[dir], db_ih[dir], sizeof(float) * GH, cudaMemcpyDeviceToDevice, st));
    }
    // dX (pre-BN-affine) += dGx . W_ih
    if (dx && !dx_done) {
      rc = ds2_gemm(0, 0, TB, In, GH, 1.f, dG, ldg, w_ih[dir], In, dir == 0 ? 0.f : 1.f, bn_gamma ? W.dxbn : dx, In,
                    gws, gws_bytes, stream);
      if (rc) return rc;
    }
  }
  if (gst != st) {
    rc = side_mark_workspace(ws, side);
    if (rc) return rc;
  }
  if (bn_gamma) {
    DS2_REQUIRE(dx && dbn_gamma && dbn_beta, "rnn bwd: BN layer needs dx, dbn_gamma, dbn_beta");
    rc = bn_rows_bwd(TB, In, W.xhat, bn_gamma, R.bnstats, W.dxbn, dx, dbn_gamma, dbn_beta, W.sums, st);
    if (rc) return rc;
  }
  return DS2_OK;
}

}  // extern "C"
