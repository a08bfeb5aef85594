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

/* ---- CTC forced alignment: the Viterbi path of each known target through the CTC lattice ---------------------
 *   x (T,B,C) fp32: logits (apply_log_softmax = 1: the log-softmax of ds2_ctc_loss_fwd_bwd is applied first) or
 *   log-probabilities used as given (apply_log_softmax = 0; -inf allowed).  targets, in_len, tgt_len, max_tgt_len and
 *   blank as for ds2_ctc_loss_fwd_bwd; in_len is clamped to [0, T] and frames t >= in_len[b] are never read.
 *   Extended sequence of S = 2L+1 states (blank, y1, blank, ..., yL, blank); fp64 scores
 *     score_t(s) = max(score_{t-1}(s), score_{t-1}(s-1), score_{t-1}(s-2)) + (double)lp[t][ext[s]]
 *   where s-2 counts only if ext[s] != blank && ext[s] != ext[s-2]; at t = 0 only states 0 and 1 are live; ties
 *   prefer s, then s-1, then s-2; the path ends in S-1 if score(S-1) >= score(S-2), else in S-2.
 *   Outputs (device):
 *     frame_labels (B,T) int32    label on the path, blank included; -1 for t >= in_len[b]      (may be NULL)
 *     frame_log_probs (B,T) fp32  log-prob of that label; 0 where the label is -1                 (may be NULL)
 *     token_spans (B,max_tgt_len,2) int32  [start, end) frames of target token k; -1 for k >= tgt_len[b]
 *     path_score (B) fp64         the path's total log-prob
 *   An utterance without a finite path (too few frames, every path through a -inf entry, in_len 0 with a non-empty
 *   target), or with tgt_len outside [0, max_tgt_len] or a target label outside [0, C), gets path_score = -inf, all
 *   labels and spans -1; the rest of the batch is aligned.  L = 0 gives the all-blank path (score 0 when in_len = 0).
 *   Limits: max_tgt_len <= DS2_CTC_ALIGN_MAX_TGT_LEN and C <= DS2_CTC_ALIGN_MAX_CLASSES (the two fp64 DP rows live in
 *   shared memory); beyond them the call returns DS2_ERR_INVALID.  Deterministic (no atomics); three launches.
 *   Workspace (bytes), each term rounded up to a multiple of 256:
 *     T*B*C*4 (log-probs) + B*T*ceil((2*max_tgt_len+1)/32)*8 (2-bit backpointers) + B*8 (target offsets)
 *   e.g. 3,904,256 bytes at T = 500, B = 32, C = 29, max_tgt_len = 250.                                                     */
#define DS2_CTC_ALIGN_MAX_TGT_LEN 6144
#define DS2_CTC_ALIGN_MAX_CLASSES 1024
size_t ds2_ctc_align_workspace_bytes(int T, int B, int C, int max_tgt_len);
int ds2_ctc_align(int T, int B, int C, const float* x, int apply_log_softmax, const int64_t* targets,
                  const int32_t* in_len, const int32_t* tgt_len, int max_tgt_len, int blank,
                  int32_t* frame_labels, float* frame_log_probs, int32_t* token_spans, double* path_score,
                  void* workspace, size_t workspace_bytes, void* stream);

/* ---- greedy decode (row N2): argmax -> collapse repeats -> drop blank, decoder.py:144-181 -----
 *   probs (B,T,C); out_len (B) ; labels/offsets (B,T) int32, counts (B) int32                   */
int ds2_greedy_decode(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                      int32_t* labels, int32_t* offsets, int32_t* counts, void* stream);
/* streaming greedy decode (row N9): the probabilities of each session's newly decided frames, packed session after
 * session: rows [row_off[s], row_off[s+1]) of probs (rows, C) belong to session s, whose carried argmax is
 * carry[slot[s]] (-1 at the stream start; ds2_greedy_decode's frame-0 rule).  labels (rows) int32 gets the label a
 * row emits (argmax, lowest index on ties, not blank, not equal to the previous frame's argmax) or -1; the last
 * row's argmax goes back to carry.  Over a stream the emitted labels equal ds2_greedy_decode of the whole output. */
int ds2_greedy_decode_stream(int n_sess, int C, const float* probs, const int32_t* row_off, const int32_t* slot,
                             int blank, int32_t* carry, int32_t* labels, void* stream);

/* ---- beam-search decode (row N5): CTC prefix beam search without a language model, what decoder.py:56-118
 * (BeamCTCDecoder) gets from ctcdecode with an empty lm_path; the rules are in csrc/beam_decode.cu.
 *   probs (B,T,C) fp32 probabilities; out_len (B) or NULL (= T), clamped to [0, T]
 *   1 <= beam_width W <= 128, 2 <= C <= 64, 0 <= blank < C, cutoff_top_n >= 1, 0 < cutoff_prob <= 1
 *   labels/timesteps (B,W,T) int32 (zero past each beam's length), lengths (B,W) int32, scores (B,W) fp64
 *   (-log-likelihood, +inf for unused slots), n_beams (B) int32 -- ctcdecode's (beam_results, beam_scores,
 *   timesteps, out_lens).  Deterministic; no allocation, no synchronisation; one launch.
 *   Workspace: per utterance a node pool of T*W + 1 nodes (24 B each) and a hash of the next power of two
 *   >= 2 (T*W + 1) slots (12 B each), which the call clears: ~2.8 MB at T = 500, W = 100; ~98 MB at T = 20000. */
size_t ds2_beam_decode_workspace_bytes(int B, int T, int C, int beam_width);
int ds2_beam_decode(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                    int beam_width, int cutoff_top_n, float cutoff_prob,
                    int32_t* labels, int32_t* timesteps, int32_t* lengths,
                    double* scores, int32_t* n_beams,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ---- ARPA n-gram language model for beam search (row N6): the tables of csrc/lm.cuh in a caller buffer.
 *   order 1..5; counts[order] (host) the number of n-grams of each order, counts[0] = n_words < 2^24;
 *   ids[n-1] (device) counts[n-1] x n int32 word ids, oldest first; logp[n-1] / backoff[n-1] (device) fp32 log10
 *   values as written (a NULL backoff array = all 0); duplicate n-grams are the caller's to refuse; bos = id of <s>;
 *   trie_mask / trie_first / trie_word (device, n_nodes each): the vocabulary trie, node 0 the root, children of a
 *   node contiguous in label order from trie_first, trie_word = word id of the node's prefix or -1.
 *   The build clears and fills the buffer on `stream` (a few launches); the inputs may be freed once it has run.
 *   Bytes: 4 per hash slot (a power of two >= 2 x the n-gram count), 24 per n-gram, 16 per trie node. */
size_t ds2_lm_bytes(int order, const int64_t* counts, int64_t n_nodes);
int ds2_lm_build(int order, const int64_t* counts, const int32_t* const* ids, const float* const* logp,
                 const float* const* backoff, int n_words, int bos, int64_t n_nodes, const uint64_t* trie_mask,
                 const int32_t* trie_first, const int32_t* trie_word, void* buffer, size_t buffer_bytes,
                 void* stream);

/* ---- beam-search decode with the language model (rules L0-L5 in csrc/beam_decode.cu): the arguments of
 * ds2_beam_decode plus the buffer of ds2_lm_build, its order, alpha, beta (fp64) and the space label, which must not
 * be the blank.  Scores are -(CTC log-likelihood + alpha * sum lm + beta * #words), best first.  Workspace: that of
 * ds2_beam_decode plus 8 B per pool node.  Deterministic; no allocation, no synchronisation; one launch. */
size_t ds2_beam_decode_lm_workspace_bytes(int B, int T, int C, int beam_width);
int ds2_beam_decode_lm(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                       int beam_width, int cutoff_top_n, float cutoff_prob,
                       const void* lm, int lm_order, double alpha, double beta, int space,
                       int32_t* labels, int32_t* timesteps, int32_t* lengths,
                       double* scores, int32_t* n_beams,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- many (alpha, beta) pairs per launch (row N6), for search_lm_params.py:100-118, which reruns
 * validation.py:run_evaluation with ds2_beam_decode_lm once per pair: the arguments of ds2_beam_decode_lm with K >= 1
 * pairs instead of one.
 *   pairs (K,2) fp64 (alpha_k, beta_k) on the HOST, each finite (checked here, then copied into the workspace)
 *   labels (K,B,T) int32: the best beam of (pair k, utterance b), zero after its length; lengths (K,B) int32.
 *   Each (k, b) is bit-identical to beam 0 of ds2_beam_decode_lm with (alpha_k, beta_k).
 *   Items are (utterance, pair), utterance-major: pass the utterances sorted by length, longest first, so the
 *   longest items start first.  One launch of as many CTAs as can be resident on the current device (occupancy x
 *   SMs, at most B*K); each CTA runs its items one after another in its own node pool and hash.
 *   Workspace: the pairs plus ds2_beam_decode_lm's workspace for that many CTAs (not for B*K utterances); it
 *   depends on the current device.  Deterministic; one launch (after a K x 16 B host-to-device copy).           */
size_t ds2_beam_decode_lm_grid_workspace_bytes(int B, int T, int C, int beam_width, int K);
int ds2_beam_decode_lm_grid(int B, int T, int C, const float* probs, const int32_t* out_len, int blank,
                            int beam_width, int cutoff_top_n, float cutoff_prob,
                            const void* lm, int lm_order, int K, const double* pairs, int space,
                            int32_t* labels, int32_t* lengths,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- streaming beam search (row N9): ds2_beam_decode(_lm) resumed across calls, one CTA per session -------------
 * The search of a session is the one ds2_beam_decode(_lm) runs on the concatenation of its calls' rows: the same
 * rules 1-7 / L0-L5, tie rules and fp64 arithmetic, so after a final call its W beams (labels, timesteps, lengths,
 * scores, n_beams) equal the one-shot search on the whole output bit for bit, and the best beam reported after t
 * frames is the one-shot search's first beam on the first t frames (including the L5 end term and reorder).
 *   items     (n_sess, 5) int32 on the device: {row0, n_frames, slot, flags, out_row}.  Rows [row0, row0+n_frames) of
 *             probs (rows, C) are the session's new frames (n_frames may be 0).  flags bit 0: the session's first call
 *             (reset: its hash is cleared and the list starts from the empty prefix); bit 1: final (write all W beams
 *             to output rows out_row .. out_row+W-1, as ds2_beam_decode writes them; otherwise only the current best
 *             to row out_row).  Slots of one call must differ.
 *   labels, timesteps (rows_out, Tout) int32; lengths (rows_out) int32; scores (rows_out) double; n_beams (n_sess).
 *             Tout >= the frames the session has decoded so far (a beam is at most that long); timesteps are stream
 *             frame indices.
 *   state     ds2_beam_decode(_lm)_stream_state_bytes(max_sessions, max_frames, beam_width), kept across calls:
 *             per slot a node pool of max_frames * W + 1 nodes with its (parent, label) hash, never compacted (rule
 *             2: a returning prefix keeps its node, so nodes of dropped prefixes stay), and the list record (lb, lnb,
 *             sc, lab, node, pnode, pslot, kids; with the LM amask, lmv, tn, ctx; n_list, pool_next, frames so far).
 *             Per slot: NP = max_frames*W + 1 nodes of 24 bytes (+8 with the LM) plus HC = the power of two >= 2 NP
 *             hash entries of 12 bytes: 600 s (30 001 frames) at W = 100 is about 173 MB (197 MB with the LM).
 *             A session must not see more than max_frames frames in total.  No workspace.                    */
size_t ds2_beam_decode_stream_state_bytes(int max_sessions, int max_frames, int beam_width);
size_t ds2_beam_decode_lm_stream_state_bytes(int max_sessions, int max_frames, int beam_width);
int ds2_beam_decode_stream(int n_sess, int C, const float* probs, const int32_t* items, int blank, int beam_width,
                           int cutoff_top_n, float cutoff_prob, int max_sessions, int max_frames, int Tout,
                           int32_t* labels, int32_t* timesteps, int32_t* lengths, double* scores, int32_t* n_beams,
                           void* state, size_t state_bytes, void* stream);
int ds2_beam_decode_lm_stream(int n_sess, int C, const float* probs, const int32_t* items, int blank, int beam_width,
                              int cutoff_top_n, float cutoff_prob, const void* lm, int lm_order, double alpha,
                              double beta, int space, int max_sessions, int max_frames, int Tout, int32_t* labels,
                              int32_t* timesteps, int32_t* lengths, double* scores, int32_t* n_beams, void* state,
                              size_t state_bytes, void* stream);

/* ---- WER / CER edit counts (validation.py:48-126, the Lev.distance calls of WordErrorRate / CharErrorRate) ----
 * Rows are hypotheses: labels (R,T) int32 with lengths (R) int32 (clamped to [0, T]), R = K x B, row k*B + b
 * scored against reference b.  References: targets flat int64 (n_targets) with target_sizes (B) int32, all on the
 * device, as the collate produces them; max_target_size >= every target size.  Blank labels are dropped from the
 * references (GreedyDecoder.convert_to_strings); a word is a maximal run of labels other than `space` (pass
 * space = C when the labels have no space).  Per row:
 *   [0] char_edits  Levenshtein distance with the spaces removed from both sides   [1] ref_chars  (non-space)
 *   [2] word_edits  Levenshtein distance between the word sequences                [3] ref_words
 * row_counts (R,4) int64 is written when non-NULL; pair_counts (K,4) int64, when non-NULL, is ADDED to (the
 * caller zeroes it once; batches accumulate).  Bit-parallel (Myers / Hyyroe) in 64-bit words, one warp per row;
 * no length limit.  Deterministic (integer sums).  Workspace: ds2_error_counts_workspace_bytes.  A reference
 * longer than max_target_size is not scored: its rows get -1 in row_counts and add nothing to pair_counts.       */
size_t ds2_error_counts_workspace_bytes(int K, int B, int64_t n_targets, int max_target_size);
int ds2_error_counts(int K, int B, int T, const int32_t* labels, const int32_t* lengths, const int64_t* targets,
                     int64_t n_targets, const int32_t* target_sizes, int max_target_size, int blank, int space,
                     int64_t* row_counts, int64_t* pair_counts, void* workspace, size_t workspace_bytes,
                     void* stream);

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

/* ---- streaming spectrogram (row N9, DESIGN.md §5.11): the frames of live streams, a call at a time ---------
 * Frame j of a stream covers samples [j*hop - n_fft/2, j*hop + n_fft/2), zero outside the stream: the frames of
 * ds2_spectrogram_batch with pad_reflect = 0, through the same DFT code, so un-normalised frames are bit-identical.
 * The host keeps each session's undecided PCM tail and packs tail + new audio into `wave`; a call emits the frames
 * j = first_frame .. first_frame + n_frames - 1 of each session (the host emits a frame once its last sample has
 * arrived, and at the stream end the frames up to 1 + n // hop with zero padding).
 *   out       (n_sess, F, Tcap) fp32, session s's frames at columns 0 .. n_frames-1, normalised by `norm`:
 *               1  fixed: (x - mean) / std with the record's mean / std;
 *               0  running: frame j with the mean and unbiased std of all values of frames 0..j of the stream,
 *                  from fp64 sums carried per session in `state` and added frame by frame in stream order, so the
 *                  result does not depend on how the stream was split into calls (a causal departure from the
 *                  offline per-utterance statistics and from per-chunk statistics);
 *              -1  none (the raw log-magnitudes).
 *   state     ds2_spectrogram_stream_state_bytes(max_sessions): DS2_STREAM_SPECT_STATE_DOUBLES fp64 per slot
 *             (running sum, sum of squares); a call with first_frame == 0 starts the slot's sums from zero.
 *   workspace ds2_spectrogram_stream_workspace_bytes(n_sess, Tcap) = n_sess * Tcap * 16 bytes (frame sums),
 *             rounded up to 256; max_frames = the largest n_frames (grid sizing), Tcap >= max_frames.       */
#define DS2_STREAM_SPECT_STATE_DOUBLES 2
typedef struct {
  int64_t wave_off;     /* first sample of the session's packed PCM in wave                                */
  int64_t wave_len;     /* packed samples: stream samples [base, base + wave_len)                          */
  int64_t base;         /* stream index of the first packed sample                                         */
  int64_t first_frame;  /* stream index of the first frame of this call                                    */
  int32_t n_frames;     /* frames emitted by this call (0: nothing to do)                                  */
  int32_t slot;         /* state record of the session                                                     */
  int32_t norm;         /* 1 fixed, 0 running, -1 none                                                     */
  float mean, std;      /* fixed normalisation                                                             */
  int32_t reserved[3];
} Ds2StreamSpect;

size_t ds2_spectrogram_stream_state_bytes(int max_sessions);
size_t ds2_spectrogram_stream_workspace_bytes(int n_sess, int Tcap);
int ds2_spectrogram_stream(int n_sess, const float* wave, const Ds2StreamSpect* sessions, int max_frames, int n_fft,
                           int hop, const float* window, float* out, int Tcap, void* state, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- input pipeline: SpecAugment on a padded spectrogram batch ----------------------------------
 * Replaces, per utterance, spec_augment (loader/spec_augment.py:68-115 with sparse_image_warp.py:88-410, the
 * reference's defaults), which SpectrogramParser.parse_audio (data_loader.py:161-163) applies to each normalised
 * (F, T) spectrogram before collation:
 *   time warp   control point c = (F/2, fp32(p + d)) with p = in[u, F/2, idx] (the VALUE is used as the time
 *               coordinate), x-flow fx = fp32(c1 - p); order-2 polyharmonic fit [[0, b^T], [b, Z]] [w; v] =
 *               [fx; 0], b = (c0, c1, 1); dense x-flow phi(r) w + v0 j + v1 i + v2 with phi(r) = r log(r) / 2 and
 *               r = sum over the whole (F, T) grid of (j^2 + i^2) - 2 (j c0 + i c1) + |c|^2; the y-flow is 0.
 *               Output (j, i) is the bilinear sample at (j, i - flow), floor clamped to [0, size - 2] and alpha
 *               to [0, 1] on the utterance's own width T; the last row takes alpha_y = 1.
 *   masks       rows [f0, f0 + f) and frames [t0, t0 + t) become 0 (width 0: no mask).
 * The random numbers are the caller's (deepspeech_pytorch_b200.input_pipeline.spec_augment_draws draws them from
 * python's `random`, numpy and torch in the reference's order).
 *   in, out   (n_utts, 1, F, Tmax) fp32, must not overlap; frames t >= frames[u] of `out` are written as 0
 *   frames    int32 frame count T of each utterance (device), 11 <= T <= Tmax
 *   draws     one Ds2SpecAugDraws per utterance (device)
 * Deterministic: no atomics, the same inputs give bit-identical outputs.                                   */
typedef struct {
  int32_t idx;  /* random.randrange(5, T - 5): the frame whose row-F/2 value is the control point's time   */
  int32_t d;    /* random.randrange(-5, 5): the warp distance                                              */
  int32_t f0, f; /* frequency mask: rows [f0, f0 + f)                                                      */
  int32_t t0, t; /* time mask: frames [t0, t0 + t); t = 0 when the reference skipped it                    */
  float Z[9];   /* torch.randn((1, 3, 3)) / 1e10, row-major                                               */
  int32_t reserved;
} Ds2SpecAugDraws;

size_t ds2_spec_augment_workspace_bytes(int n_utts);
int ds2_spec_augment(int n_utts, int F, int Tmax, const float* in, const int32_t* frames,
                     const Ds2SpecAugDraws* draws, float* out, void* workspace, size_t workspace_bytes, void* stream);

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
/* the same with alpha multiplied by *alpha_dev, a float on the device (the layers pass the inverse of the
 * power-of-two scale of a scaled fp16 operand this way); alpha_dev may be NULL.                                */
int ds2_gemm_f16_scaled(int M, int N, int K, float alpha, const void* A16, int lda, const void* B16, int ldb,
                        float beta, float* C, int ldc, const float* alpha_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DS2_B200_H_ */
