"""Input pipeline on the GPU (SURVEY.md §8f row N3): raw PCM of a minibatch -> the batch tuple
`(inputs, targets, input_percentages, target_sizes)` that `DeepSpeech.training_step` consumes.

Replaces, for a whole minibatch at once,
  * `SpectrogramParser.compute_spectrogram` (reference deepspeech_pytorch/loader/data_loader.py:73-94): STFT with
    n_fft = win_length = sample_rate * window_size (320), hop = sample_rate * window_stride (160), the configured
    window, centred frames; magnitude; log1p; per-utterance (x - mean) / std (torch's unbiased std) — which the
    reference runs per utterance in librosa / numpy inside DataLoader worker processes, and
  * `_collate_fn` (data_loader.py:247-270): sort by length (descending, stable), zero-pad into (B,1,F,Tmax), flat
    int64 targets in the sorted order, `input_percentages` = frames / Tmax (fp32), int32 `target_sizes`.

The host side only does integer bookkeeping: utterances are packed back to back into ONE grow-only pinned staging
buffer in sorted order, copied with a single asynchronous H2D transfer, and `ds2_spectrogram_batch` (csrc/spect.cu)
writes the padded batch tensor directly.  No CPU fallback: without the library / a GPU this raises.
"""
import ctypes as C
import math
from typing import List, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import check, get_lib, ptr


def analysis_window(name: str, n: int) -> np.ndarray:
    """scipy.signal.get_window(name, n, fftbins=True) — the periodic window librosa.stft builds
    (reference SpectrogramWindow values: hamming / hann / blackman / bartlett), float32."""
    k = np.arange(n, dtype=np.float64)
    x = 2.0 * math.pi * k / n                       # periodic: denominator n, not n - 1
    if name == "hamming":
        w = 0.54 - 0.46 * np.cos(x)
    elif name == "hann":
        w = 0.5 - 0.5 * np.cos(x)
    elif name == "blackman":
        w = 0.42 - 0.5 * np.cos(x) + 0.08 * np.cos(2 * x)
    elif name == "bartlett":
        w = 1.0 - np.abs(2.0 * k / n - 1.0)
    else:
        raise ValueError(f"unsupported window {name!r}")
    return w.astype(np.float32)


class SpectrogramBatcher:
    """callable: (waves, transcripts) -> (inputs cuda (B,1,F,Tmax), targets int64, input_percentages f32,
    target_sizes int32) — the `_collate_fn` tuple, with `inputs` already on the device."""

    def __init__(self, spect_cfg, normalize: bool = True, pad_mode: str = "constant", device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.Ds2Error("SpectrogramBatcher: needs a CUDA device; there is no CPU path")
        self.n_fft = int(spect_cfg.sample_rate * spect_cfg.window_size)
        self.hop = int(spect_cfg.sample_rate * spect_cfg.window_stride)
        wname = spect_cfg.window.value if hasattr(spect_cfg.window, "value") else str(spect_cfg.window)
        self.window = torch.from_numpy(analysis_window(wname, self.n_fft)).to(self.device)
        if pad_mode not in ("constant", "reflect"):
            raise ValueError("pad_mode must be 'constant' (librosa >= 0.10) or 'reflect' (librosa < 0.10)")
        self.pad_reflect = int(pad_mode == "reflect")
        self.normalize = int(bool(normalize))
        self._stage = None          # pinned PCM staging buffer (grow-only)
        self._meta = None           # pinned int64 offsets + int32 rows

    @staticmethod
    def order_and_frames(n_samples: Sequence[int], hop: int):
        """integer bookkeeping of the collate: frames per utterance (librosa centre framing: 1 + len // hop) and the
        stable descending order `sorted(batch, key=frames, reverse=True)` produces (ties keep the original order)"""
        frames = [1 + int(n) // hop for n in n_samples]
        order = sorted(range(len(frames)), key=lambda i: frames[i], reverse=True)
        return order, frames

    def __call__(self, waves: List, transcripts: List[Sequence[int]]):
        B = len(waves)
        assert B > 0 and len(transcripts) == B
        lens = [int(len(w)) for w in waves]
        if self.pad_reflect and min(lens) <= self.n_fft // 2:
            raise _lib.Ds2Error("reflect padding needs utterances longer than n_fft/2 samples (librosa raises too)")
        order, frames = self.order_and_frames(lens, self.hop)
        total = sum(lens)
        if self._stage is None or self._stage.numel() < total:
            self._stage = torch.empty(int(total * 1.25) + 1024, dtype=torch.float32).pin_memory()
        if self._meta is None or self._meta.numel() < 2 * (B + 1):
            self._meta = torch.empty(4 * (B + 1), dtype=torch.int64).pin_memory()
        stage = self._stage.numpy()
        offs = self._meta[:B + 1]
        rows = self._meta[B + 1:2 * (B + 1)].view(torch.int32)[:B]
        pos = 0
        for slot, i in enumerate(order):            # packed in SORTED order: utterance `slot` goes to batch row `slot`
            w = waves[i]
            w = w.detach().cpu().numpy() if isinstance(w, torch.Tensor) else np.asarray(w)
            stage[pos:pos + lens[i]] = w.astype(np.float32, copy=False)
            offs[slot] = pos
            rows[slot] = slot
            pos += lens[i]
        offs[B] = pos
        Tmax = frames[order[0]]
        F = self.n_fft // 2 + 1
        dev = self.device
        with torch.cuda.device(dev):
            wave_d = self._stage[:total].to(dev, non_blocking=True)
            offs_d = offs.to(dev, non_blocking=True)
            rows_d = rows.to(dev, non_blocking=True)
            out = torch.empty(B, 1, F, Tmax, device=dev)
            lib = get_lib()
            nws = lib.ds2_spectrogram_workspace_bytes(B)
            ws = torch.empty(nws, dtype=torch.uint8, device=dev)
            check(lib.ds2_spectrogram_batch(B, ptr(wave_d), ptr(offs_d), ptr(rows_d), max(lens), self.n_fft, self.hop,
                                            ptr(self.window), self.pad_reflect, self.normalize, ptr(out), Tmax, ptr(ws),
                                            nws, C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  "ds2_spectrogram_batch")
        # host-side part of _collate_fn (data_loader.py:256-270), in the sorted order
        input_percentages = torch.tensor([frames[i] / float(Tmax) for i in order], dtype=torch.float32)
        target_sizes = torch.tensor([len(transcripts[i]) for i in order], dtype=torch.int32)
        flat = [int(c) for i in order for c in transcripts[i]]
        targets = torch.tensor(flat, dtype=torch.long)
        self.h2d_bytes = total * 4 + (B + 1) * 8 + B * 4
        return out, targets, input_percentages, target_sizes
