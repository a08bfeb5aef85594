"""TEST INFRASTRUCTURE — generates tests/golden/spec_augment/spec_augment.npz by EXECUTING THE REFERENCE.

Runs only in the dev container (needs /root/reference).  Imports the reference's unmodified
``deepspeech_pytorch/loader/spec_augment.py`` (with ``sparse_image_warp.py``) and runs its ``spec_augment`` on
normalised spectrograms of synthetic PCM.  Each utterance seeds python ``random``, ``np.random`` and torch with its
own seed and runs once; the fixture keeps its input, the reference's output, the dense x-flow (captured by wrapping
the module's ``sparse_image_warp`` and calling through to the original), the numbers it drew and one probe value from
each generator afterwards.  This pins oracle/spec_augment_oracle.py and the CUDA kernel (csrc/spec_augment.cu).  The
model fixtures written by oracle/make_golden.py are not touched.

To keep the file small the inputs are rounded to multiples of 1/256 (still spectrogram-shaped, normalised values),
and for the T = 1000 utterance the output and flow are kept for a subset of rows only: both ends, the control-point
row and its neighbours, the last two rows (the last one takes alpha_y = 1) and the rows around the frequency mask's
edges.  Every output row depends on its own input row only (on rows 159 and 160 for the last one), so a row subset
checks the same arithmetic.

    python oracle/make_spec_augment_golden.py
"""
import json
import os
import random
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
import spect_oracle  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "spec_augment", "spec_augment.npz")
F = 161
# (T, first seed tried, what the seed search asks of the utterance, keep all rows)
CASES = [(11, 11, "time_mask_skipped", True), (12, 20, None, True), (40, 40, "empty_freq_mask", True),
         (300, 300, "large_flow", True), (1000, 1000, None, False)]


def load_spec_augment():
    """The reference's unmodified ``deepspeech_pytorch.loader.spec_augment`` module.  Its module-level imports of
    librosa / librosa.display / matplotlib / matplotlib.pyplot serve only ``visualization_spectrogram``; inert
    stand-ins satisfy them.  ``spec_augment`` itself runs on numpy, python ``random`` and torch CPU."""
    for name in ("librosa", "librosa.display", "matplotlib", "matplotlib.pyplot"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["librosa"].display = sys.modules["librosa.display"]
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    if not hasattr(sys.modules["matplotlib"], "use"):
        sys.modules["matplotlib"].use = lambda *a, **k: None   # spec_augment.py:42
    if ref_shim.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shim.REFERENCE_ROOT)
    from deepspeech_pytorch.loader import spec_augment as ref_sa
    return ref_sa


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def _wants(want, T, flow, dr):
    if want == "time_mask_skipped":
        return dr["t"] > T
    if want == "empty_freq_mask":
        return dr["f"] == 0
    if want == "large_flow":
        return float(np.abs(flow).max()) >= 1000.0
    return True


def _rows(dr, all_rows):
    if all_rows:
        return np.arange(F)
    rows = {0, 1, 2, F // 2 - 1, F // 2, F // 2 + 1, F - 2, F - 1}
    for r in (dr["f0"] - 1, dr["f0"], dr["f0"] + dr["f"] - 1, dr["f0"] + dr["f"]):
        if 0 <= r < F:
            rows.add(r)
    return np.array(sorted(rows))


def main():
    ref_sa = load_spec_augment()
    orig_warp = ref_sa.sparse_image_warp
    captured = {}

    def capture(img, src, dst, *a, **k):
        warped, flows = orig_warp(img, src, dst, *a, **k)
        captured["flows"] = flows.detach().clone()
        return warped, flows

    ref_sa.sparse_image_warp = capture
    torch.set_num_threads(1)
    blob = {}
    for k, (T, seed, want, all_rows) in enumerate(CASES):
        rng = np.random.default_rng(1000 + k)
        n = (T - 1) * 160 + int(rng.integers(0, 160))          # 1 + n // 160 == T frames
        t = np.arange(n) / 16000.0
        y = 0.3 * np.sin(2 * np.pi * (180 + 41 * k) * t) * (1 + 0.5 * np.sin(2 * np.pi * 1.3 * t))
        y = (y + 0.05 * rng.standard_normal(n)).astype(np.float32)
        x = np.round(spect_oracle.compute_spectrogram(y) * 256.0) / 256.0
        x = x.astype(np.float32)
        assert x.shape == (F, T)
        while True:
            _seed(seed)
            out = ref_sa.spec_augment(torch.from_numpy(x.copy())).numpy()
            probes = np.array([random.random(), np.random.random(), float(torch.rand(1))], np.float64)
            flows = captured["flows"][0].numpy()
            assert np.all(flows[..., 0] == 0.0), "y-flow is not exactly zero"
            # the draws, read back from the generators re-seeded and replayed in spec_augment's order
            _seed(seed)
            idx = random.randrange(5, T - 5)
            d = random.randrange(-5, 5)
            Z = (torch.randn((1, 3, 3)) / 1e10).numpy().reshape(9)
            f = int(np.random.uniform(0.0, 27))
            f0 = random.randint(0, F - f)
            tt = int(np.random.uniform(0.0, 70))
            t0 = random.randint(0, T - tt) if T - tt >= 0 else 0
            dr = dict(idx=idx, d=d, f=f, f0=f0, t=tt, t0=t0)
            if _wants(want, T, flows[..., 1], dr):
                break
            seed += 1
        rows = _rows(dr, all_rows)
        blob[f"x/{k}"] = x
        blob[f"rows/{k}"] = rows.astype(np.int32)
        blob[f"out/{k}"] = out[rows].astype(np.float32)
        blob[f"flow_x/{k}"] = flows[rows, :, 1].astype(np.float32)
        blob[f"max_abs_flow/{k}"] = np.array(float(np.abs(flows[..., 1]).max()), np.float64)
        blob[f"probes/{k}"] = probes
        blob[f"draws/{k}"] = np.array([idx, d, f0, f, t0, tt], np.int64)
        blob[f"Z/{k}"] = Z.astype(np.float32)
        blob[f"seed/{k}"] = np.array(seed, np.int64)
        print(f"spec_augment[{k}]: T={T} seed={seed} draws={dr} rows={len(rows)} "
              f"max|flow|={np.abs(flows[..., 1]).max():.4g}")
    blob["meta"] = np.array(json.dumps(dict(n=len(CASES), F=F, torch=torch.__version__, numpy=np.__version__)))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **blob)
    print(f"-> {OUT}: {os.path.getsize(OUT) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
