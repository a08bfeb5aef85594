// Input pipeline (SURVEY.md §8f row N3): raw PCM -> the padded, length-sorted spectrogram batch the train step
// consumes, on the GPU.  Replaces, per utterance, SpectrogramParser.compute_spectrogram
// (reference deepspeech_pytorch/loader/data_loader.py:73-94:  librosa.stft(n_fft = win_length = sample_rate *
// window_size, hop = sample_rate * window_stride, window, center=True) -> magnitude -> log1p -> (x - mean) / std with
// torch's unbiased std) and, per batch, the zero-padding copy of _collate_fn (data_loader.py:247-270: utterance i
// goes to row dst_row[i] of a (B,1,F,Tmax) tensor, frames >= its own length are zero).
//
// Kernel 1 (spect_logmag_kernel): a CTA takes 16 consecutive frames of one utterance, builds the centred, windowed
// frames in shared memory (reflect or zero padding at the ends, librosa's pad_mode) and evaluates the n_fft-point real
// DFT directly: thread = frequency bin, 16 frames in registers, twiddles from a shared-memory table indexed by
// (k*n mod n_fft).  n_fft = 320 = 2^6*5 is tiny: a direct fp32 DFT is 3.3 GFMA for 32 x 1000 frames (~0.1 ms of the
// FP32 pipes) and keeps fp32 accuracy; magnitude, log1p and the per-utterance sum / sum of squares (double
// atomics) are fused.  Kernel 2 (spect_normalize_pad_kernel) normalises in place and writes the zero padding.
#include <math_constants.h>

#include "common.cuh"

namespace ds2 {

namespace sp {
constexpr int FT = 16;        // frames per CTA
constexpr int THREADS = 192;  // >= n_fft/2 + 1 bins (161 for the reference's 20 ms window at 16 kHz)
constexpr int MAX_NFFT = 384;
}  // namespace sp

// Frames f0 .. f0+FT-1 of one signal y[0, L) into xw[n][f], windowed: frame f0 + f starts at sample
// start + f * hop (start may be negative), samples outside [0, L) are zero (reflected when pad_reflect).
__device__ __forceinline__ void spect_load_frames(float (*xw)[sp::FT], const float* __restrict__ y, long long L,
                                                  long long start, int n_valid, int n_fft, int hop,
                                                  const float* __restrict__ window, int pad_reflect) {
  using namespace sp;
  for (int idx = threadIdx.x; idx < n_fft * FT; idx += THREADS) {
    const int f = idx / n_fft, n = idx % n_fft;      // consecutive threads -> consecutive samples
    float v = 0.f;
    if (f < n_valid) {
      long long i = start + (long long)f * hop + n;
      if (pad_reflect) {
        if (i < 0) i = -i;
        if (i >= L) i = 2 * (L - 1) - i;
        v = (i >= 0 && i < L) ? y[i] : 0.f;
      } else {
        v = (i >= 0 && i < L) ? y[i] : 0.f;
      }
      v *= window[n];
    }
    xw[n][f] = v;
  }
}

// log1p(|DFT bin k|) of the FT frames in xw: thread = bin, frames in registers, twiddles cs/sn indexed by
// (k*n mod n_fft).  Shared by the batch and the streaming spectrogram, so their frames are bit-identical.
__device__ __forceinline__ void spect_dft_logmag(const float (*xw)[sp::FT], const float* cs, const float* sn,
                                                 int n_fft, int k, float (&v)[sp::FT]) {
  using namespace sp;
  float re[FT], im[FT];
#pragma unroll
  for (int f = 0; f < FT; ++f) re[f] = im[f] = 0.f;
  int ph = 0;                                       // (k * n) mod n_fft
  for (int n = 0; n < n_fft; ++n) {
    const float c = cs[ph], s = sn[ph];
#pragma unroll
    for (int f4 = 0; f4 < FT; f4 += 4) {
      const float4 x = *reinterpret_cast<const float4*>(&xw[n][f4]);
      re[f4] = fmaf(x.x, c, re[f4]); im[f4] = fmaf(x.x, s, im[f4]);
      re[f4 + 1] = fmaf(x.y, c, re[f4 + 1]); im[f4 + 1] = fmaf(x.y, s, im[f4 + 1]);
      re[f4 + 2] = fmaf(x.z, c, re[f4 + 2]); im[f4 + 2] = fmaf(x.z, s, im[f4 + 2]);
      re[f4 + 3] = fmaf(x.w, c, re[f4 + 3]); im[f4 + 3] = fmaf(x.w, s, im[f4 + 3]);
    }
    ph += k;
    if (ph >= n_fft) ph -= n_fft;
  }
#pragma unroll
  for (int f = 0; f < FT; ++f)   // np.log1p(|D|), contracted explicitly so that every caller rounds alike
    v[f] = log1pf(sqrtf(fmaf(re[f], re[f], __fmul_rn(im[f], im[f]))));
}

__device__ __forceinline__ void spect_twiddles(float* cs, float* sn, int n_fft) {
  for (int j = threadIdx.x; j < n_fft; j += sp::THREADS) sincospif(2.f * (float)j / (float)n_fft, &sn[j], &cs[j]);
}

__global__ void __launch_bounds__(sp::THREADS) spect_logmag_kernel(
    const float* __restrict__ wave, const long long* __restrict__ offs, const int32_t* __restrict__ dst_row, int n_fft,
    int hop, const float* __restrict__ window, int pad_reflect, float* __restrict__ out, int Tmax,
    double* __restrict__ sums) {
  using namespace sp;
  __shared__ __align__(16) float xw[MAX_NFFT][FT];   // [n][frame]: one LDS.128 feeds 4 frames
  __shared__ float cs[MAX_NFFT], sn[MAX_NFFT];
  const int u = blockIdx.y, f0 = blockIdx.x * FT;
  const long long o0 = offs[u], L = offs[u + 1] - o0;
  const int n_frames = (int)(L / hop) + 1;           // librosa.stft(center=True): 1 + len // hop
  if (f0 >= n_frames) return;
  const int F = n_fft / 2 + 1, half = n_fft / 2;
  spect_twiddles(cs, sn, n_fft);
  spect_load_frames(xw, wave + o0, L, (long long)f0 * hop - half, n_frames - f0, n_fft, hop, window, pad_reflect);
  __syncthreads();
  const int k = threadIdx.x;
  float s1 = 0.f, s2 = 0.f;
  if (k < F) {
    float v[FT];
    spect_dft_logmag(xw, cs, sn, n_fft, k, v);
    float* dst = out + ((size_t)dst_row[u] * F + k) * Tmax + f0;
#pragma unroll
    for (int f = 0; f < FT; ++f) {
      if (f0 + f < n_frames) {
        dst[f] = v[f];
        s1 += v[f];
        s2 = fmaf(v[f], v[f], s2);
      }
    }
  }
  // per-utterance sum and sum of squares: fp32 inside a thread (<= 16 values), double across threads
  double d1 = warp_sum_d((double)s1), d2 = warp_sum_d((double)s2);
  if (threadIdx.x % 32 == 0) {
    atomicAdd(&sums[2 * u], d1);
    atomicAdd(&sums[2 * u + 1], d2);
  }
}

// in place: x <- (x - mean) / std for t < n_frames[u] (torch.Tensor.std: unbiased), 0 for the padding t >= n_frames
__global__ void spect_normalize_pad_kernel(int B, int F, int Tmax, const long long* __restrict__ offs,
                                           const int32_t* __restrict__ dst_row, int hop, int normalize,
                                           const double* __restrict__ sums, float* __restrict__ out) {
  const int u = blockIdx.y;
  const int n_frames = (int)((offs[u + 1] - offs[u]) / hop) + 1;
  const double n = (double)n_frames * F;
  const double mean = sums[2 * u] / n;
  const double var = n > 1.0 ? (sums[2 * u + 1] - n * mean * mean) / (n - 1.0) : 0.0;
  const float m = normalize ? (float)mean : 0.f;
  const float inv = normalize ? (float)(1.0 / sqrt(var > 0.0 ? var : 0.0)) : 1.f;
  float* base = out + (size_t)dst_row[u] * F * Tmax;
  const size_t total = (size_t)F * Tmax;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % Tmax);
    base[i] = t < n_frames ? (base[i] - m) * inv : 0.f;
  }
}


// ------------------------------------------------------------------ streaming (DESIGN.md §5.11)
// Kernel 1: a CTA takes FT frames of one session.  The frames are those of the offline kernel with pad_reflect = 0,
// with the session's packed PCM y[0, wave_len) holding stream samples [base, base + wave_len).  Writes the
// un-normalised log-magnitudes to out (n_sess, F, Tcap) and each frame's sum and sum of squares over its F bins
// (fp64, fixed order) to fsum[2 * (s * Tcap + f)].
__global__ void __launch_bounds__(sp::THREADS) spect_stream_logmag_kernel(
    const float* __restrict__ wave, const Ds2StreamSpect* __restrict__ sess, int n_fft, int hop,
    const float* __restrict__ window, float* __restrict__ out, int Tcap, double* __restrict__ fsum) {
  using namespace sp;
  __shared__ __align__(16) float xw[MAX_NFFT][FT];
  __shared__ float cs[MAX_NFFT], sn[MAX_NFFT];
  __shared__ double red[THREADS / 32][FT][2];
  const int s = blockIdx.y, f0 = blockIdx.x * FT;
  const Ds2StreamSpect m = sess[s];
  if (f0 >= m.n_frames) return;
  const int F = n_fft / 2 + 1, half = n_fft / 2;
  spect_twiddles(cs, sn, n_fft);
  const long long start = (m.first_frame + f0) * (long long)hop - half - m.base;
  spect_load_frames(xw, wave + m.wave_off, m.wave_len, start, m.n_frames - f0, n_fft, hop, window, 0);
  __syncthreads();
  const int k = threadIdx.x;
  float v[FT];
#pragma unroll
  for (int f = 0; f < FT; ++f) v[f] = 0.f;
  if (k < F) {
    spect_dft_logmag(xw, cs, sn, n_fft, k, v);
    float* dst = out + ((size_t)s * F + k) * Tcap + f0;
#pragma unroll
    for (int f = 0; f < FT; ++f)
      if (f0 + f < m.n_frames) dst[f] = v[f];
  }
  const int w = threadIdx.x / 32, lane = threadIdx.x % 32;
#pragma unroll
  for (int f = 0; f < FT; ++f) {
    const double a = warp_sum_d((double)v[f]), b = warp_sum_d((double)v[f] * (double)v[f]);
    if (lane == 0) { red[w][f][0] = a; red[w][f][1] = b; }
  }
  __syncthreads();
  if (threadIdx.x < FT && f0 + threadIdx.x < m.n_frames) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < THREADS / 32; ++i) { a += red[i][threadIdx.x][0]; b += red[i][threadIdx.x][1]; }
    double* d = fsum + 2 * ((size_t)s * Tcap + f0 + threadIdx.x);
    d[0] = a;
    d[1] = b;
  }
}

// Kernel 2: one CTA per session.  Thread 0 walks the call's frames in stream order, adding each frame's sums to the
// session's running fp64 sums, and turns them into that frame's (mean, 1/std) (unbiased std over all values of frames
// 0..j); the walk is sequential so the sums do not depend on how the stream was split into calls.  Then every thread
// normalises.  norm = 1: the session's fixed mean / std; -1: no normalisation.
__global__ void spect_stream_normalize_kernel(int F, int Tcap, const Ds2StreamSpect* __restrict__ sess,
                                              double* __restrict__ state, double* __restrict__ fsum,
                                              float* __restrict__ out) {
  const int s = blockIdx.x;
  const Ds2StreamSpect m = sess[s];
  if (m.n_frames <= 0 || m.norm < 0) return;
  double* st = state + (size_t)DS2_STREAM_SPECT_STATE_DOUBLES * m.slot;
  float2* mi = reinterpret_cast<float2*>(fsum + 2 * (size_t)s * Tcap);   // (mean, 1/std) replaces frame f's sums
  if (threadIdx.x == 0) {
    double s1 = m.first_frame == 0 ? 0.0 : st[0], s2 = m.first_frame == 0 ? 0.0 : st[1];
    for (int f = 0; f < m.n_frames; ++f) {
      const double* d = fsum + 2 * ((size_t)s * Tcap + f);
      s1 += d[0];
      s2 += d[1];
      float mf, inv;
      if (m.norm == 1) {
        mf = m.mean;
        inv = 1.f / m.std;
      } else {
        const double n = (double)(m.first_frame + f + 1) * F;
        const double mean = s1 / n;
        const double var = (s2 - n * mean * mean) / (n - 1.0);
        mf = (float)mean;
        inv = (float)(1.0 / sqrt(var > 0.0 ? var : 0.0));
      }
      mi[f] = make_float2(mf, inv);
    }
    st[0] = s1;
    st[1] = s2;
  }
  __syncthreads();
  float* base = out + (size_t)s * F * Tcap;
  for (int i = threadIdx.x; i < F * m.n_frames; i += blockDim.x) {
    const int k = i / m.n_frames, f = i % m.n_frames;
    const float2 p = mi[f];
    base[(size_t)k * Tcap + f] = (base[(size_t)k * Tcap + f] - p.x) * p.y;
  }
}

}  // namespace ds2

extern "C" {
using namespace ds2;

size_t ds2_spectrogram_workspace_bytes(int n_utts) { return align_up((size_t)n_utts * 2 * sizeof(double), 256); }

int ds2_spectrogram_batch(int n_utts, const float* wave, const int64_t* offsets, const int32_t* dst_row,
                          int max_samples, int n_fft, int hop, const float* window, int pad_reflect, int normalize,
                          float* out, int Tmax, void* workspace, size_t workspace_bytes, void* stream) {
  DS2_REQUIRE(n_utts > 0 && wave && offsets && dst_row && window && out, "spectrogram: null argument");
  DS2_REQUIRE(n_fft >= 2 && n_fft % 2 == 0 && n_fft <= sp::MAX_NFFT && n_fft / 2 + 1 <= sp::THREADS,
              "spectrogram: n_fft %d not supported (even, <= %d)", n_fft, sp::MAX_NFFT);
  DS2_REQUIRE(hop > 0 && max_samples >= 0 && Tmax >= max_samples / hop + 1,
              "spectrogram: Tmax %d < frames of the longest utterance (%d)", Tmax, max_samples / hop + 1);
  DS2_REQUIRE(workspace_bytes >= ds2_spectrogram_workspace_bytes(n_utts), "spectrogram: workspace too small");
  cudaStream_t st = as_stream(stream);
  double* sums = static_cast<double*>(workspace);
  DS2_CHECK_CUDA(cudaMemsetAsync(sums, 0, (size_t)n_utts * 2 * sizeof(double), st));
  const int max_frames = max_samples / hop + 1;
  DS2_LAUNCH(spect_logmag_kernel, dim3(cdiv(max_frames, sp::FT), n_utts), sp::THREADS, 0, st, wave,
             reinterpret_cast<const long long*>(offsets), dst_row, n_fft, hop, window, pad_reflect, out, Tmax, sums);
  const int F = n_fft / 2 + 1;
  int bx = cdiv((long long)F * Tmax, 256 * 4);
  bx = bx < 1 ? 1 : (bx > 132 ? 132 : bx);
  DS2_LAUNCH(spect_normalize_pad_kernel, dim3(bx, n_utts), 256, 0, st, n_utts, F, Tmax,
             reinterpret_cast<const long long*>(offsets), dst_row, hop, normalize, sums, out);
  return DS2_OK;
}

size_t ds2_spectrogram_stream_state_bytes(int max_sessions) {
  return align_up((size_t)max_sessions * DS2_STREAM_SPECT_STATE_DOUBLES * sizeof(double), 256);
}

size_t ds2_spectrogram_stream_workspace_bytes(int n_sess, int Tcap) {
  return align_up((size_t)n_sess * Tcap * 2 * sizeof(double), 256);
}

int ds2_spectrogram_stream(int n_sess, const float* wave, const Ds2StreamSpect* sessions, int max_frames, int n_fft,
                           int hop, const float* window, float* out, int Tcap, void* state, void* workspace,
                           size_t workspace_bytes, void* stream) {
  DS2_REQUIRE(n_sess > 0 && wave && sessions && window && out && state, "spectrogram_stream: null argument");
  DS2_REQUIRE(n_fft >= 2 && n_fft % 2 == 0 && n_fft <= sp::MAX_NFFT && n_fft / 2 + 1 <= sp::THREADS,
              "spectrogram_stream: n_fft %d not supported (even, <= %d)", n_fft, sp::MAX_NFFT);
  DS2_REQUIRE(hop > 0 && max_frames >= 0 && Tcap >= max_frames && Tcap > 0,
              "spectrogram_stream: Tcap %d < max_frames %d", Tcap, max_frames);
  DS2_REQUIRE(workspace_bytes >= ds2_spectrogram_stream_workspace_bytes(n_sess, Tcap),
              "spectrogram_stream: workspace too small");
  if (max_frames == 0) return DS2_OK;
  cudaStream_t st = as_stream(stream);
  double* fsum = static_cast<double*>(workspace);
  DS2_LAUNCH(spect_stream_logmag_kernel, dim3(cdiv(max_frames, sp::FT), n_sess), sp::THREADS, 0, st, wave, sessions,
             n_fft, hop, window, out, Tcap, fsum);
  DS2_LAUNCH(spect_stream_normalize_kernel, n_sess, 256, 0, st, n_fft / 2 + 1, Tcap, sessions,
             static_cast<double*>(state), fsum, out);
  return DS2_OK;
}

}  // extern "C"
