// Arguments of one recurrent sweep (all time steps of one layer, both directions).
#pragma once
#include <stdint.h>

#include "../../include/ds2_b200.h"

namespace ds2 {

// Gate rows per hidden unit: LSTM i, f, g, o; GRU r, z, n; tanh one
constexpr int num_gates(int rnn) { return rnn == DS2_RNN_LSTM ? 4 : (rnn == DS2_RNN_GRU ? 3 : 1); }

struct SeqArgs {
  int T, B, H, D, G;
  const int32_t* len;
  float* gates;  // (T,B,D,G*H): input projections in, gate activations (fwd) / gate gradients (bwd) out
  float* hseq;   // (D,T,B,H) per-direction outputs, zero at masked steps
  float* aux;    // (D,T,B,H) LSTM cell states / GRU W_hn h + b_hn (-> dGh_n after bwd); null for tanh
  const float* w_hh[2];   // the layer's (G*H,H) recurrent weights
  float* w_hhT[2];        // bwd: (H,G*H) workspace for the fp32 W_hh^T of the streaming and FFMA backward sweeps,
                          // each of which transposes w_hh into it itself (the resident ones read fp16 only)
  const float* b_ih[2];
  const float* b_hh[2];
  const float* h0;        // (D,B,H) or null
  const float* c0;
  const float* dy;        // bwd: (T,B,H)
  float* carry;           // bwd: (D,B,H) dc (LSTM) / dh (GRU)
  int training;
  // bwd, optional: bias gradients accumulated inside the sweep (column sums of the gate gradients over (t,b)).
  // dbias[d]: (G*H) zeroed by the caller; dbias_hn[d]: GRU only, (H) sum of the h-side n-gate gradient.
  float* dbias[2];
  float* dbias_hn[2];
  // bwd, optional (precision-16 GEMM operands): fp16 copies of the gate gradients, multiplied by the power of two
  // f16_scale[0] (device), written by the sweep as it produces them — f16_dg (T*B, D*G*H) row-major, f16_dgT
  // (D*G*H, T*B) transposed, f16_auxT (D*H, T*B) GRU h-side n-gate gradient transposed.
  void* f16_dg;
  void* f16_dgT;
  void* f16_auxT;
  const float* f16_scale;
  // bwd, optional: fp16 copy of the transposed recurrent matrix (H, G*H) made by the forward pass of the same step.
  // The fp16-resident sweep takes it as it is instead of converting w_hh.
  const void* w_hhT16[2];
};

// What a tensor-core backward sweep produced besides the gate gradients: the caller computes what it did not
struct SweepBwdOut {
  bool dbias;   // accumulated the bias gradients into SeqArgs::dbias / dbias_hn
  bool f16;     // wrote the fp16 gate-gradient copies SeqArgs::f16_dg / f16_dgT / f16_auxT
};

}  // namespace ds2
