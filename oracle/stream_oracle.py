"""TEST INFRASTRUCTURE — float64 restatement of the streaming spectrogram's running normalisation
(deepspeech.pytorch_b200/streaming.py, csrc/spect.cu `spect_stream_normalize_kernel`).  Not product code.

Frame j of a stream is normalised with the mean and the unbiased standard deviation of all values of frames 0..j:
a causal replacement for the offline per-utterance statistics."""
import numpy as np


def running_normalize(frames: np.ndarray) -> np.ndarray:
    """frames (F, T) un-normalised log-magnitudes -> (F, T) float64, column j with the statistics of columns 0..j"""
    x = np.asarray(frames, dtype=np.float64)
    F, T = x.shape
    s1 = np.cumsum(x.sum(axis=0))
    s2 = np.cumsum((x * x).sum(axis=0))
    n = F * np.arange(1, T + 1, dtype=np.float64)
    mean = s1 / n
    var = (s2 - n * mean * mean) / (n - 1.0)
    return (x - mean[None, :]) / np.sqrt(np.maximum(var, 0.0))[None, :]
