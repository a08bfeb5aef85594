"""Device time of the GPU input pipeline (`SpectrogramBatcher`) per batch, with and without SpecAugment.

B synthetic utterances of about 10 s each (T ~ 1000 frames, the size of a LibriSpeech training batch) go through
`SpectrogramBatcher` with `augmentation_conf=None` and with `AugmentationConfig(spec_augment=True)`, alternating,
after warm-up.  Per batch it reports the device time between CUDA events recorded around the whole call (PCM
upload, spectrogram, SpecAugment) and, separately, the time of `ds2_spec_augment` alone over back-to-back launches on
a prepared batch, with the bytes it must move (read + write of the (B, 1, 161, Tmax) fp32 batch) over that time.  The
card name and power limit are read in the same run.  Needs a GPU; prints one JSON line.

    python tools/bench_input_pipeline.py [--batch 32] [--seconds 10] [--iters 30]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import deepspeech_pytorch_b200 as ds  # noqa: E402
from deepspeech_pytorch_b200 import input_pipeline as ip  # noqa: E402


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": clk}
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def waves(B, seconds, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(B):
        L = int(16000 * seconds * rng.uniform(0.95, 1.0))
        t = np.arange(L) / 16000.0
        y = 0.3 * np.sin(2 * np.pi * (120 + 17 * i) * t) + 0.05 * rng.standard_normal(L)
        out.append(y.astype(np.float32))
    return out


def time_events(fn, iters):
    """device ms per call: events recorded around each call, median over `iters` calls"""
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_input_pipeline: needs a CUDA device")
    torch.cuda.set_device(0)
    ds.get_lib()
    W = waves(args.batch, args.seconds)
    tr = [[1, 2, 3]] * len(W)
    plain = ip.SpectrogramBatcher(ds.SpectConfig())
    aug = ip.SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=ds.AugmentationConfig(spec_augment=True))
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    for _ in range(args.warmup):
        plain(W, tr)
        aug(W, tr)
    torch.cuda.synchronize()
    res_plain, res_aug = [], []
    for _ in range(3):                                  # alternate the two pipelines
        res_plain.append(time_events(lambda: plain(W, tr), args.iters))
        res_aug.append(time_events(lambda: aug(W, tr), args.iters))
    ms_plain = float(np.median([r[0] for r in res_plain]))
    ms_aug = float(np.median([r[0] for r in res_aug]))

    # the kernel pair alone, back to back on a prepared batch
    x = plain(W, tr)[0]
    B, _, F, Tmax = x.shape
    frames = [1 + len(w) // plain.hop for w in W]
    draws = ip.spec_augment_draws(frames, F)
    frames_d = torch.tensor(frames, dtype=torch.int32, device="cuda")
    draws_d = torch.from_numpy(draws.view(np.uint8).copy()).cuda()
    out = torch.empty_like(x)
    nws = ds.get_lib().ds2_spec_augment_workspace_bytes(B)
    ws = torch.empty(nws, dtype=torch.uint8, device="cuda")
    reps = 50

    def kernels():
        for _ in range(reps):
            ip._launch_spec_augment(x, out, frames_d, draws_d, ws, nws)

    kernels()
    torch.cuda.synchronize()
    k_med, k_min = time_events(kernels, 10)
    us = 1e3 * k_med / reps
    nbytes = 2 * x.numel() * 4
    print(json.dumps({
        "card": card_info(), "batch": B, "F": F, "Tmax": Tmax, "seconds_per_utt": args.seconds,
        "batch_ms_plain": round(ms_plain, 4), "batch_ms_spec_augment": round(ms_aug, 4),
        "added_ms_per_batch": round(ms_aug - ms_plain, 4),
        "spec_augment_kernels_us": round(us, 2), "spec_augment_kernels_us_min": round(1e3 * k_min / reps, 2),
        "spec_augment_bytes": nbytes, "spec_augment_GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
        "runs_plain_ms": [round(r[0], 4) for r in res_plain], "runs_aug_ms": [round(r[0], 4) for r in res_aug],
    }))


if __name__ == "__main__":
    main()
