/*
 * ds2_b200.h — C-ABI of the H100-native DeepSpeech2 train-step path (libds2_b200.so).
 *
 * The reference (SeanNaren/deepspeech.pytorch) has no FFI layer of its own: its hot path is the
 * Python class deepspeech_pytorch/model.py::DeepSpeech calling third-party torch ops.  This header
 * is the boundary a maintainer binds *beneath* that class (ctypes stub in INTEGRATION.md): each
 * entry point replaces the torch call sites named in its comment (reference file:line).
 *
 * Conventions
 *   - every function returns 0 on success or a negative DS2_ERR_* code; ds2_last_error() returns a
 *     thread-local message for the last failure on the calling thread;
 *   - all tensor pointers are DEVICE pointers to dense row-major fp32 unless suffixed `_host` or
 *     typed otherwise; lengths are int32 on the device; CTC targets are int64 (reference
 *     data_loader.py:269);
 *   - `stream` is a cudaStream_t passed as void*; nothing synchronises the device or allocates
 *     memory: scratch comes from the caller (ds2_*_workspace_bytes), saved-for-backward tensors are
 *     caller-owned buffers listed per call;
 *   - re-entrant per stream; no global mutable state except the lazily created TMA descriptor
 *     encoder handle.
 *
 * Precision: DS2_PREC_FP32 = fp32 FFMA everywhere (bit-for-bit independent of tensor cores);
 *            DS2_PREC_TF32 = dense GEMMs (input projections, recurrent products, weight gradients)
 *            on wgmma tensor cores with TF32 operands / fp32 accumulation — the same arithmetic
 *            class the reference's stock CUDA path uses (cuDNN allow_tf32=True).
 *            DS2_PREC_F16 = the reference's `precision: 16` (configs/librispeech.yaml:12, torch autocast): the
 *            dense GEMMs of the recurrent stack (input projections, weight gradients, data gradients) take fp16
 *            operand copies (gradients scaled by a power of two per tensor), fp32 accumulation; the recurrent
 *            products already use fp16 operands; conv front-end / fc head as in TF32 mode; parameters,
 *            activations, gradients and the optimizer stay fp32 (what autocast keeps in fp32 too).
 */
#ifndef DS2_B200_H_
#define DS2_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DS2_OK                 0
#define DS2_ERR_INVALID       -1   /* bad argument / unsupported shape                           */
#define DS2_ERR_CUDA          -2   /* a CUDA runtime / driver call failed                         */
#define DS2_ERR_UNSORTED      -3   /* lengths not sorted descending (pack_padded_sequence raises) */
#define DS2_ERR_WORKSPACE     -4   /* workspace too small                                         */

enum { DS2_RNN_LSTM = 0, DS2_RNN_GRU = 1, DS2_RNN_TANH = 2 };   /* reference enums.py:18-21 */
enum { DS2_PREC_FP32 = 0, DS2_PREC_TF32 = 1, DS2_PREC_F16 = 2 };

/* Fixed geometry of the reference front-end (model.py:157-164). */
#define DS2_NUM_FREQ   161
#define DS2_CONV_CH     32
#define DS2_CONV1_D     81
#define DS2_CONV2_D     41
#define DS2_RNN_IN0   1312   /* 32 * 41, feature index = c*41 + d (model.py:219-221) */

const char* ds2_version(void);
const char* ds2_last_error(void);
/* Fails (DS2_ERR_CUDA) when no sm_90 (H100) device is usable: there is no CPU fallback. */
int ds2_device_check(int* sm_count, int* cc_major, int* cc_minor);
int ds2_set_precision(int prec);
int ds2_get_precision(void);
/* Kernel-launch counter (all kernels launched by this library since the last reset). */
int64_t ds2_launch_count(int reset);
/* Number of tensor-core-mode recurrent sweeps that had to take the one-launch-per-time-step FFMA kernels
 * because their shape is not eligible for the persistent tensor-core kernels (also reported once per shape on
 * stderr): a benchmark line with a non-zero count did not run the path it claims.                      */
int64_t ds2_fallback_count(int reset);

/* Optional side stream for deferred work.  With a side stream set, ds2_rnn_layer_bwd(deferred_dw != 0) queues the
 * weight-gradient GEMMs (dW_ih, dW_hh: nobody needs them before the optimizer / the gradient exchange) on it, ordered
 * after the layer's sweep and operand copies; they then run in the shadow of the next layer's latency-bound sweep.
 * The caller (a) alternates between two workspaces for consecutive layers (the library orders the reuse of a
 * workspace after the side work that read it), (b) calls ds2_join_side_stream(stream) before anything on `stream`
 * (or any other stream ordered after it) reads those gradients, (c) keeps `x` and `reserve` of that call valid until
 * the side stream has passed this point (the transposed fp16 copies of the layer input and of the hidden sequence are
 * made on the side stream too).  NULL disables (default).                                                        */
int ds2_set_side_stream(void* stream);
int ds2_join_side_stream(void* stream);

/* Device-time ranges around the kernel groups of each block (cudaEvent pairs on the launching stream).
 * ds2_prof_report synchronises, writes "tag:total_ms:count;..." into buf and clears the records.     */
int ds2_prof_enable(int on);
int ds2_prof_report(char* buf, size_t cap);

/* ---- lengths: DeepSpeech.get_seq_lens, model.py:299-310 (host integers, bit-exact) ---------- */
int ds2_seq_lens_host(const int32_t* in_len_host, int n, int32_t* out_len_host);

/* ---- conv front-end: MaskConv(Conv2d,BN2d,Hardtanh,Conv2d,BN2d,Hardtanh) model.py:53-69,157-164
 * and the (B,C,D,T)->(T,B,C*D) re-layout of model.py:219-221.
 *   x          (B,1,161,T)
 *   out_len    (B) int32, = get_seq_lens(lengths)
 *   w1 (32,1,41,11) b1 (32) ; w2 (32,32,21,11) b2 (32)
 *   bnK        gamma,beta,running_mean,running_var (32 each); running stats updated in place when
 *              training (momentum, unbiased variance), read when !training
 *   y          (T', B, 1312)   T' = (T-1)/2+1, zero for t >= out_len[b]
 *   saved      z1 (B,32,81,T') masked pre-BN conv1 ; a1 (B,32,81,T') activation ;
 *              z2 (B,32,41,T') masked pre-BN conv2 ; stats (4*32): mean1,invstd1,mean2,invstd2
 *   workspace  ds2_conv_frontend_workspace_bytes(B,T)
 */
size_t ds2_conv_frontend_workspace_bytes(int B, int T);
int ds2_conv_frontend_fwd(int B, int T, const float* x, const int32_t* out_len,
                          const float* w1, const float* b1, const float* bn1_gamma, const float* bn1_beta,
                          float* bn1_rmean, float* bn1_rvar,
                          const float* w2, const float* b2, const float* bn2_gamma, const float* bn2_beta,
                          float* bn2_rmean, float* bn2_rvar,
                          int training, float momentum, float eps,
                          float* y, float* z1, float* a1, float* z2, float* stats,
                          void* workspace, size_t workspace_bytes, void* stream);
/* dy (T',B,1312) -> parameter gradients (written, not accumulated).  No gradient w.r.t. x. */
int ds2_conv_frontend_bwd(int B, int T, const float* x, const int32_t* out_len,
                          const float* w1, const float* bn1_gamma, const float* bn1_beta,
                          const float* w2, const float* bn2_gamma, const float* bn2_beta,
                          const float* z1, const float* a1, const float* z2, const float* stats,
                          const float* dy,
                          float* dw1, float* db1, float* dbn1_gamma, float* dbn1_beta,
                          float* dw2, float* db2, float* dbn2_gamma, float* dbn2_beta,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---- one BatchRNN layer: model.py:80-102 ([BN1d] -> pack -> LSTM/GRU/RNN -> pad -> sum dirs) --
 * Lengths must be sorted descending (checked by the Python shell like pack_padded_sequence does).
 *   x (T,B,In)  len (B) int32  y (T,B,H)   T = max(len)
 *   per direction d in [0,dirs): w_ih[d] (G*H,In)  w_hh[d] (G*H,H)  b_ih[d], b_hh[d] (G*H)
 *   bn_*: NULL for the first layer (model.py:177)
 *   h0/c0 (dirs,B,H) or NULL;  hn/cn (dirs,B,H) outputs (cn only for LSTM)
 *   reserve: ds2_rnn_reserve_floats() floats, written by fwd (training) and consumed by bwd.  In the tensor-core
 *            modes a training fwd also leaves an fp16 copy of W_hh^T there for the bwd sweep of the same step (the
 *            weights must not change between the two calls; a bwd on a reserve that no fwd of this process filled
 *            converts the weights itself).  With a side stream set that copy is made on it: `w_hh` stays valid
 *            until the side stream has passed this point.
 */
typedef struct {
  int rnn_type;      /* DS2_RNN_*                     */
  int bidirectional; /* 0/1                           */
  int T, B, In, H;
  int training;      /* BN batch statistics + reserve */
  float bn_momentum, bn_eps;
  int deferred_dw;   /* bwd: 1 = dW_ih / dW_hh may be queued on the side stream (see ds2_set_side_stream) */
} ds2_rnn_desc;

size_t ds2_rnn_reserve_floats(const ds2_rnn_desc* d);
size_t ds2_rnn_workspace_bytes(const ds2_rnn_desc* d);
int ds2_rnn_layer_fwd(const ds2_rnn_desc* d, const float* x, const int32_t* len,
                      const float* bn_gamma, const float* bn_beta, float* bn_rmean, float* bn_rvar,
                      const float* const* w_ih, const float* const* w_hh,
                      const float* const* b_ih, const float* const* b_hh,
                      const float* h0, const float* c0,
                      float* y, float* hn, float* cn, float* reserve,
                      void* workspace, size_t workspace_bytes, void* stream);
int ds2_rnn_layer_bwd(const ds2_rnn_desc* d, const float* x, const int32_t* len,
                      const float* bn_gamma, const float* bn_beta,
                      const float* const* w_ih, const float* const* w_hh,
                      const float* const* b_ih, const float* const* b_hh,
                      const float* dy, float* reserve,
                      float* dx, float* dbn_gamma, float* dbn_beta,
                      float* const* dw_ih, float* const* dw_hh, float* const* db_ih, float* const* db_hh,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- Lookahead + Hardtanh(0,20): model.py:105-130,189-193 ------------------------------------
 *   y[t,b,c] = clamp(sum_k w[c,k] * x[t+k,b,c], 0, 20);  x,y (T,B,H), w (H,1,ctx)             */
int ds2_lookahead_fwd(int T, int B, int H, int ctx, const float* x, const float* w, float* y, void* stream);
/* dz: caller scratch (T,B,H), receives dy masked by the Hardtanh interior (must not alias dx). */
int ds2_lookahead_bwd(int T, int B, int H, int ctx, const float* x, const float* w, const float* dy,
                      float* dz, float* dx, float* dw, void* stream);

/* ---- fc head: SequenceWise(BatchNorm1d(H), Linear(H,C,bias=False)) model.py:195-201 ----------
 *   x (T,B,H) -> logits (T,B,C).   saved: xhat (T*B,H) normalised input, stats (2*H: mean,invstd)
 *   softmax != 0 applies InferenceBatchSoftmax (model.py:72-77, eval only).                     */
size_t ds2_fc_head_workspace_bytes(int rows, int H, int C);
int ds2_fc_head_fwd(int rows, int H, int C, const float* x, const float* bn_gamma, const float* bn_beta,
                    float* bn_rmean, float* bn_rvar, const float* w, int training, float momentum, float eps,
                    int softmax, float* logits, float* xhat, float* stats,
                    void* workspace, size_t workspace_bytes, void* stream);
int ds2_fc_head_bwd(int rows, int H, int C, const float* bn_gamma, const float* bn_beta, const float* w,
                    const float* xhat,
                    const float* stats, const float* dlogits, float* dx, float* dbn_gamma, float* dbn_beta,
                    float* dw, void* workspace, size_t workspace_bytes, void* stream);

/* ---- CTC: log_softmax + CTCLoss(blank, reduction='sum', zero_infinity=True) model.py:245-248 --
 *   logits (T,B,C) ; targets int64 1-D concatenated ; in_len,tgt_len (B) int32 device
 *   nll (B) per-utterance loss (0 where infeasible) ; grad (T,B,C) = d(sum nll)/d(logits)
 *   = softmax - posterior for t < in_len[b], 0 otherwise (and 0 for infeasible utterances).
 *   max_tgt_len: upper bound of tgt_len (host knows it from the batch collate).                 */
size_t ds2_ctc_workspace_bytes(int T, int B, int C, int max_tgt_len);
int ds2_ctc_loss_fwd_bwd(int T, int B, int C, const float* logits, const int64_t* targets,
                         const int32_t* in_len, const int32_t* tgt_len, int max_tgt_len, int blank,
                         float* nll, float* grad, void* workspace, size_t workspace_bytes, void* stream);

/* ---- greedy decode (row N2): argmax -> collapse repeats -> drop blank, decoder.py:144-181 -----
 *   probs (B,T,C); out_len (B) ; labels/offsets (B,T) int32, counts (B) int32                   */
int ds2_greedy_decode(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                      int32_t* labels, int32_t* offsets, int32_t* counts, void* stream);

/* ---- optimizer on flat fp32 buffers (row N1): clip_grad_norm_(max_norm) + AdamW / SGD-Nesterov,
 * model.py:273-297, configs/librispeech.yaml:12.  grad_scale multiplies g first (1/world for DDP
 * mean).  norm_ws: >= ds2_optim_workspace_bytes(); grad_norm_out (1 float, device) gets the
 * pre-clip total norm.                                                                          */
size_t ds2_optim_workspace_bytes(void);
int ds2_adamw_step(int64_t n, float* p, const float* g, float* m, float* v, float lr, float beta1, float beta2,
                   float eps, float weight_decay, int step, float grad_scale, float max_norm,
                   float* grad_norm_out, void* norm_ws, void* stream);
int ds2_sgd_nesterov_step(int64_t n, float* p, const float* g, float* momentum_buf, float lr, float momentum,
                          float weight_decay, int first_step, float grad_scale, float max_norm,
                          float* grad_norm_out, void* norm_ws, void* stream);

/* ---- input pipeline (row N3): raw PCM -> padded, length-sorted spectrogram batch ---------------
 * Replaces SpectrogramParser.compute_spectrogram (data_loader.py:73-94: librosa.stft(n_fft = win_length, hop,
 * window, center=True) -> |.| -> log1p -> (x - mean)/std, torch's unbiased std) for every utterance of a batch and
 * the zero-padding copy of _collate_fn (data_loader.py:247-270).
 *   wave      concatenated fp32 PCM of the n_utts utterances (device)
 *   offsets   (n_utts+1) int64 sample offsets into wave (device)
 *   dst_row   (n_utts) int32: batch row of each utterance (the host sorts by length, descending, stable)
 *   window    (n_fft) fp32 analysis window (device), e.g. periodic Hamming
 *   pad_reflect  1: librosa pad_mode="reflect" (librosa < 0.10), 0: "constant" zeros (librosa >= 0.10)
 *   out       (n_utts, 1, n_fft/2+1, Tmax) fp32, frames t >= 1 + len/hop of a row are written as zeros
 *   max_samples  length of the longest utterance (grid sizing); Tmax >= max_samples/hop + 1              */
size_t ds2_spectrogram_workspace_bytes(int n_utts);
int ds2_spectrogram_batch(int n_utts, const float* wave, const int64_t* offsets, const int32_t* dst_row,
                          int max_samples, int n_fft, int hop, const float* window, int pad_reflect, int normalize,
                          float* out, int Tmax, void* workspace, size_t workspace_bytes, void* stream);

/* ---- dense GEMM used by the blocks above, exported for tests / the roofline bench ------------
 *   C[M,N] = alpha * op(A) op(B) + beta * C ; row-major ; transX: 0 = as stored, 1 = transposed.
 *   Dispatches on ds2_get_precision(): fp32 FFMA kernel or the wgmma TF32 kernel.            */
size_t ds2_gemm_workspace_bytes(int transA, int transB, int M, int N, int K);
int ds2_gemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda,
             const float* B, int ldb, float beta, float* C, int ldc,
             void* workspace, size_t workspace_bytes, void* stream);

/* fp16-operand variant (the precision-16 mode's GEMM): A16 (M,K) and B16 (N,K) are K-major half matrices on the
 * device, C = alpha * A16 . B16^T + beta * C in fp32.  lda / ldb multiples of 8, 16-byte aligned bases.       */
int ds2_gemm_f16(int M, int N, int K, float alpha, const void* A16, int lda, const void* B16, int ldb, float beta,
                 float* C, int ldc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DS2_B200_H_ */
