// Gate math shared by every recurrent kernel (FFMA step kernels and the wgmma persistent kernels).
// PyTorch conventions (SURVEY.md Appendix B): LSTM rows [i,f,g,o]; GRU rows [r,z,n] with
// n = tanh(x_n + r * (W_hn h + b_hn)); tanh-RNN single gate.
#pragma once
#include "common.cuh"

namespace ds2 {

struct LstmFwd { float i, f, g, o, c, h; };

// pre-activations (x part + h part + both biases already summed) and previous cell -> gates, c, h
__device__ __forceinline__ LstmFwd lstm_cell_fwd(float pi, float pf, float pg, float po, float c_prev) {
  LstmFwd r;
  r.i = sigmoidf_(pi);
  r.f = sigmoidf_(pf);
  r.g = tanhf(pg);
  r.o = sigmoidf_(po);
  r.c = fmaf(r.f, c_prev, r.i * r.g);
  r.h = r.o * tanhf(r.c);
  return r;
}

struct LstmBwd { float di, df, dg, d_o, dc_prev; };

// dh: total gradient w.r.t. h_t ; dc_in: carried gradient w.r.t. c_t from step t+1
__device__ __forceinline__ LstmBwd lstm_cell_bwd(float i, float f, float g, float o, float c, float c_prev,
                                                 float dh, float dc_in) {
  LstmBwd r;
  float tc = tanhf(c);
  float dc = fmaf(dh * o, 1.f - tc * tc, dc_in);
  r.d_o = dh * tc * o * (1.f - o);
  r.di = dc * g * i * (1.f - i);
  r.df = dc * c_prev * f * (1.f - f);
  r.dg = dc * i * (1.f - g * g);
  r.dc_prev = dc * f;
  return r;
}

struct GruFwd { float r, z, n, h; };

// xr,xz,xn: input projections (+b_ih); hr,hz: W_h{r,z} h + b_h{r,z}; hn: W_hn h + b_hn
__device__ __forceinline__ GruFwd gru_cell_fwd(float xr, float xz, float xn, float hr, float hz, float hn,
                                               float h_prev) {
  GruFwd g;
  g.r = sigmoidf_(xr + hr);
  g.z = sigmoidf_(xz + hz);
  g.n = tanhf(fmaf(g.r, hn, xn));
  g.h = fmaf(g.z, h_prev - g.n, g.n);  // (1-z)*n + z*h_prev
  return g;
}

struct GruBwd { float dr, dz, dxn, dhn, dh_prev; };  // dr,dz: pre-activation grads (same for x and h side)

__device__ __forceinline__ GruBwd gru_cell_bwd(float r, float z, float n, float hn, float h_prev, float dh) {
  GruBwd g;
  g.dz = dh * (h_prev - n) * z * (1.f - z);
  float dn_pre = dh * (1.f - z) * (1.f - n * n);
  g.dxn = dn_pre;
  g.dhn = dn_pre * r;
  g.dr = dn_pre * hn * r * (1.f - r);
  g.dh_prev = dh * z;
  return g;
}

}  // namespace ds2
