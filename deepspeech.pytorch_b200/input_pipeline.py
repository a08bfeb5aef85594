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

With `augmentation_conf.spec_augment` set, it also replaces the reference's per-utterance `spec_augment`
(loader/spec_augment.py:68-115, applied by SpectrogramParser.parse_audio, data_loader.py:161-163): the host draws the
random numbers (`spec_augment_draws`, the reference's generators in the reference's order) and `ds2_spec_augment`
(csrc/spec_augment.cu) does the time warp and the masks on the batch.
"""
import math
import random
from typing import List, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import check, current_stream, get_lib, ptr

# Ds2SpecAugDraws (include/ds2_b200.h), one record per utterance
SPEC_AUG_DRAWS_DTYPE = np.dtype([("idx", "<i4"), ("d", "<i4"), ("f0", "<i4"), ("f", "<i4"), ("t0", "<i4"),
                                 ("t", "<i4"), ("Z", "<f4", (9,)), ("reserved", "<i4")])
assert SPEC_AUG_DRAWS_DTYPE.itemsize == 64
SPEC_AUG_MIN_FRAMES = 11     # random.randrange(5, T - 5) is empty for T <= 10
_SA_W, _SA_F, _SA_T = 5, 27, 70   # spec_augment's defaults: time_warp(W=5), frequency_masking_para, time_masking_para


def spec_augment_draws(frames: Sequence[int], n_freq: int = 161) -> np.ndarray:
    """The random numbers the reference's `spec_augment` draws for each utterance (frame count T, n_freq rows), one
    utterance after another in the order given, from the process-global python `random`, `np.random` and torch CPU
    generators in the reference's order (spec_augment.py:56,60, sparse_image_warp.py:170, spec_augment.py:99,103,
    108,112), so the generators end in the state the reference leaves them in.  T <= 10 raises the ValueError
    `random.randrange` raises there.  -> structured array of SPEC_AUG_DRAWS_DTYPE."""
    n = len(frames)
    out = np.zeros(n, SPEC_AUG_DRAWS_DTYPE)
    cols = {name: [0] * n for name in ("idx", "d", "f0", "f", "t0", "t")}
    Z = []
    for k, T in enumerate(frames):
        T = int(T)
        cols["idx"][k] = random.randrange(_SA_W, T - _SA_W)
        cols["d"][k] = random.randrange(-_SA_W, _SA_W)
        Z.append(torch.randn((1, 3, 3)))     # one call per utterance: a larger call draws a different sequence
        f = int(np.random.uniform(low=0.0, high=_SA_F))
        if n_freq - f >= 0:
            cols["f0"][k], cols["f"][k] = random.randint(0, n_freq - f), f
        t = int(np.random.uniform(low=0.0, high=_SA_T))
        if T - t >= 0:                                   # otherwise the reference skips the mask without a draw
            cols["t0"][k], cols["t"][k] = random.randint(0, T - t), t
    for name, v in cols.items():
        out[name] = v
    if n:
        out["Z"] = (torch.cat(Z) / 1e10).reshape(n, 9).numpy()   # the same fp32 division, elementwise
    return out


def _launch_spec_augment(spec, out, frames_d, draws_d, ws, nws):
    B, _, F, Tmax = spec.shape
    check(get_lib().ds2_spec_augment(B, F, Tmax, ptr(spec), ptr(frames_d), ptr(draws_d), ptr(out), ptr(ws), nws,
                                     current_stream()), "ds2_spec_augment")


def spec_augment_batch(inputs: torch.Tensor, frames: Sequence[int], draws: np.ndarray = None) -> torch.Tensor:
    """SpecAugment on an existing (B, 1, F, Tmax) fp32 CUDA batch whose row b holds an utterance of frames[b] frames
    (zero padded after).  `draws` (SPEC_AUG_DRAWS_DTYPE, one per row) default to `spec_augment_draws(frames, F)`,
    drawn now in row order.  Returns a new tensor; frames t >= frames[b] of it are 0."""
    if not (inputs.is_cuda and inputs.dtype == torch.float32 and inputs.dim() == 4 and inputs.shape[1] == 1):
        raise _lib.Ds2Error("spec_augment_batch: inputs must be a (B, 1, F, Tmax) float32 CUDA tensor")
    B, _, F, Tmax = inputs.shape
    frames = [int(t) for t in frames]
    if len(frames) != B:
        raise _lib.Ds2Error(f"spec_augment_batch: {len(frames)} frame counts for a batch of {B}")
    if draws is None:
        draws = spec_augment_draws(frames, F)
    draws = np.ascontiguousarray(draws, SPEC_AUG_DRAWS_DTYPE)
    if len(draws) != B:
        raise _lib.Ds2Error(f"spec_augment_batch: {len(draws)} draws for a batch of {B}")
    if min(frames) < SPEC_AUG_MIN_FRAMES or max(frames) > Tmax:
        raise _lib.Ds2Error(f"spec_augment_batch: frame counts must lie in [{SPEC_AUG_MIN_FRAMES}, Tmax={Tmax}]")
    dev = inputs.device
    with torch.cuda.device(dev):
        x = inputs.contiguous()
        frames_d = torch.tensor(frames, dtype=torch.int32).to(dev)
        draws_d = torch.from_numpy(draws.view(np.uint8).copy()).to(dev)
        out = torch.empty_like(x)
        nws = get_lib().ds2_spec_augment_workspace_bytes(B)
        ws = torch.empty(nws, dtype=torch.uint8, device=dev)
        _launch_spec_augment(x, out, frames_d, draws_d, ws, nws)
    return out


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


def spect_geometry(spect_cfg):
    """-> (sample_rate, n_fft, hop, window name) of a SpectConfig: n_fft = win_length = sample_rate * window_size,
    hop = sample_rate * window_stride (data_loader.py:78-80)"""
    window = spect_cfg.window.value if hasattr(spect_cfg.window, "value") else str(spect_cfg.window)
    return (int(spect_cfg.sample_rate), int(spect_cfg.sample_rate * spect_cfg.window_size),
            int(spect_cfg.sample_rate * spect_cfg.window_stride), window)


class SpectrogramBatcher:
    """callable: (waves, transcripts) -> (inputs cuda (B,1,F,Tmax), targets int64, input_percentages f32,
    target_sizes int32) — the `_collate_fn` tuple, with `inputs` already on the device.

    `augmentation_conf` mirrors SpectrogramParser's parameter (data_loader.py:132-149): with `spec_augment` set, every
    utterance is augmented as `spec_augment` does it, with the random numbers drawn in the order the waves are given
    (the dataset order: the reference augments in __getitem__, before the collate sorts by length).  Noise
    injection and speed / volume perturbation need sox and are not implemented here: asking for them raises."""

    def __init__(self, spect_cfg, normalize: bool = True, pad_mode: str = "constant", device="cuda",
                 augmentation_conf=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.Ds2Error("SpectrogramBatcher: needs a CUDA device; there is no CPU path")
        self.spec_augment = False
        if augmentation_conf is not None:
            if augmentation_conf.noise_dir:
                raise _lib.Ds2Error("SpectrogramBatcher: noise injection (augmentation.noise_dir) is not implemented "
                                    "on the GPU input pipeline")
            if augmentation_conf.speed_volume_perturb:
                raise _lib.Ds2Error("SpectrogramBatcher: speed / volume perturbation (augmentation."
                                    "speed_volume_perturb) is not implemented on the GPU input pipeline")
            self.spec_augment = bool(augmentation_conf.spec_augment)
        _, self.n_fft, self.hop, wname = spect_geometry(spect_cfg)
        self.window = torch.from_numpy(analysis_window(wname, self.n_fft)).to(self.device)
        if pad_mode not in ("constant", "reflect"):
            raise ValueError("pad_mode must be 'constant' (librosa >= 0.10) or 'reflect' (librosa < 0.10)")
        self.pad_reflect = int(pad_mode == "reflect")
        self.normalize = int(bool(normalize))
        self._stage = None          # pinned PCM staging buffer (grow-only)
        self._meta = None           # pinned int64 offsets + int32 rows
        # recorded after the H2D copies out of _stage / _meta: the next call rewrites that pinned memory only once the
        # copies have run, so a caller that does not synchronise (a training loop) can be at most one batch ahead
        self._staged = None

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
        F = self.n_fft // 2 + 1
        aug = self.spec_augment
        # drawn in the caller's (dataset) order, before the length sort: the reference augments in __getitem__
        draws = spec_augment_draws(frames, F) if aug else None
        total = sum(lens)
        if self._staged is not None:
            self._staged.synchronize()
        if self._stage is None or self._stage.numel() < total:
            self._stage = torch.empty(int(total * 1.25) + 1024, dtype=torch.float32).pin_memory()
        # int64 words: offsets (B + 1) | int32 rows (B) + int32 frames (B) | Ds2SpecAugDraws (8 words each)
        n_meta = 2 * (B + 1) + (8 * B if aug else 0)
        if self._meta is None or self._meta.numel() < n_meta:
            self._meta = torch.empty(max(4 * (B + 1), n_meta), dtype=torch.int64).pin_memory()
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
        if aug:
            self._meta[B + 1:2 * (B + 1)].view(torch.int32)[B:2 * B].copy_(
                torch.tensor([frames[i] for i in order], dtype=torch.int32))
            self._meta[2 * (B + 1):n_meta].numpy().view(SPEC_AUG_DRAWS_DTYPE)[:] = draws[order]
        Tmax = frames[order[0]]
        dev = self.device
        with torch.cuda.device(dev):
            wave_d = self._stage[:total].to(dev, non_blocking=True)
            meta_d = self._meta[:n_meta].to(dev, non_blocking=True)
            if self._staged is None:
                self._staged = torch.cuda.Event()
            self._staged.record()
            offs_d = meta_d[:B + 1]
            rows_d = meta_d[B + 1:2 * (B + 1)].view(torch.int32)[:B]
            out = torch.empty(B, 1, F, Tmax, device=dev)
            spec = torch.empty_like(out) if aug else out
            lib = get_lib()
            nws = lib.ds2_spectrogram_workspace_bytes(B)
            nws_aug = lib.ds2_spec_augment_workspace_bytes(B) if aug else 0
            ws = torch.empty(nws + nws_aug, dtype=torch.uint8, device=dev)
            check(lib.ds2_spectrogram_batch(B, ptr(wave_d), ptr(offs_d), ptr(rows_d), max(lens), self.n_fft, self.hop,
                                            ptr(self.window), self.pad_reflect, self.normalize, ptr(spec), Tmax, ptr(ws),
                                            nws, current_stream()), "ds2_spectrogram_batch")
            if aug:
                frames_d = meta_d[B + 1:2 * (B + 1)].view(torch.int32)[B:2 * B]
                draws_d = meta_d[2 * (B + 1):n_meta]
                _launch_spec_augment(spec, out, frames_d, draws_d, ws[nws:], nws_aug)
        # host-side part of _collate_fn (data_loader.py:256-270), in the sorted order
        input_percentages = torch.tensor([frames[i] / float(Tmax) for i in order], dtype=torch.float32)
        target_sizes = torch.tensor([len(transcripts[i]) for i in order], dtype=torch.int32)
        flat = [int(c) for i in order for c in transcripts[i]]
        targets = torch.tensor(flat, dtype=torch.long)
        self.h2d_bytes = total * 4 + n_meta * 8
        return out, targets, input_percentages, target_sizes
