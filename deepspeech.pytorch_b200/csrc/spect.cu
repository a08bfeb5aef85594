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
  for (int j = threadIdx.x; j < n_fft; j += THREADS) sincospif(2.f * (float)j / (float)n_fft, &sn[j], &cs[j]);
  const float* y = wave + o0;
  for (int idx = threadIdx.x; idx < n_fft * FT; idx += THREADS) {
    const int f = idx / n_fft, n = idx % n_fft;      // consecutive threads -> consecutive samples
    float v = 0.f;
    if (f0 + f < n_frames) {
      long long i = (long long)(f0 + f) * hop + n - half;
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
  __syncthreads();
  const int k = threadIdx.x;
  float s1 = 0.f, s2 = 0.f;
  if (k < F) {
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
    float* dst = out + ((size_t)dst_row[u] * F + k) * Tmax + f0;
#pragma unroll
    for (int f = 0; f < FT; ++f) {
      if (f0 + f < n_frames) {
        const float v = log1pf(sqrtf(re[f] * re[f] + im[f] * im[f]));   // np.log1p(|D|)
        dst[f] = v;
        s1 += v;
        s2 = fmaf(v, v, s2);
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

}  // extern "C"
