"""SpecAugment on the GPU input pipeline.  CPU: the float64 oracle (oracle/spec_augment_oracle.py) against the
reference's own outputs and dense flows (tests/golden/spec_augment/spec_augment.npz, written by
`python oracle/make_spec_augment_golden.py`), and `spec_augment_draws` against the reference's generator states.
-m gpu: `ds2_spec_augment` (csrc/spec_augment.cu) against the fixture and the oracle, through `spec_augment_batch` and
`SpectrogramBatcher(augmentation_conf=...)`."""
import ctypes
import json
import os
import random
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib
from deepspeech_pytorch_b200.input_pipeline import (SPEC_AUG_DRAWS_DTYPE, SpectrogramBatcher, spec_augment_batch,
                                                    spec_augment_draws)
from oracle import spec_augment_oracle as SA
from oracle import spect_oracle as SO

FIXTURE = os.path.join(GOLDEN_DIR, "spec_augment", "spec_augment.npz")


@pytest.fixture(scope="module")
def golden():
    z = np.load(FIXTURE, allow_pickle=False)
    cases = []
    for k in range(json.loads(str(z["meta"]))["n"]):
        idx, d, f0, f, t0, t = (int(v) for v in z[f"draws/{k}"])
        # out / flow hold the rows listed in rows/k (all of them except for the T = 1000 utterance)
        cases.append(dict(x=z[f"x/{k}"], rows=z[f"rows/{k}"], out=z[f"out/{k}"], flow=z[f"flow_x/{k}"],
                          max_flow=float(z[f"max_abs_flow/{k}"]), probes=z[f"probes/{k}"], seed=int(z[f"seed/{k}"]),
                          draw=dict(idx=idx, d=d, f0=f0, f=f, t0=t0, t=t, Z=z[f"Z/{k}"])))
    return cases


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def _probes():
    return np.array([random.random(), np.random.random(), float(torch.rand(1))])


def _mask(shape, dr):
    m = np.zeros(shape, bool)
    m[dr["f0"]:dr["f0"] + dr["f"], :] = True
    m[:, dr["t0"]:dr["t0"] + dr["t"]] = True
    return m


def _out_tol(max_flow):
    return 1e-3 + 4e-6 * max_flow


def _records(draws):
    rec = np.zeros(len(draws), SPEC_AUG_DRAWS_DTYPE)
    for k, dr in enumerate(draws):
        for name in ("idx", "d", "f0", "f", "t0", "t", "Z"):
            rec[k][name] = dr[name]
    return rec


def test_fixture_covers_the_edge_cases(golden):
    Ts = [c["x"].shape[1] for c in golden]
    assert min(Ts) == 11 and 12 in Ts and max(Ts) >= 1000
    assert max(c["max_flow"] for c in golden) >= 1000.0                                    # flow in the thousands
    assert any(c["draw"]["t"] > c["x"].shape[1] or c["draw"]["f"] == 0 for c in golden)   # a skipped / empty mask
    for c in golden:
        assert c["out"].shape == c["flow"].shape == (len(c["rows"]), c["x"].shape[1])
        assert c["max_flow"] == 0.0 or float(np.abs(c["flow"]).max()) > 0.5 * c["max_flow"]
    assert os.path.getsize(FIXTURE) < 1e6


def test_oracle_matches_reference(golden):
    for c in golden:
        x, dr, rows = c["x"], dict(c["draw"]), c["rows"]
        T = x.shape[1]
        if dr["t"] > T:                       # the reference skipped the time mask
            dr["t"] = 0
        out, flow = SA.spec_augment(x, dr)
        ferr = np.abs(flow[rows] - c["flow"]).max()
        assert ferr <= 1e-4 * max(1.0, c["max_flow"]), (T, ferr)
        assert float(np.abs(flow).max()) == pytest.approx(c["max_flow"], rel=1e-4, abs=1e-4)
        err = np.abs(out[rows] - c["out"]).max()
        assert err <= _out_tol(c["max_flow"]), (T, err)
        m = _mask(x.shape, dr)
        assert np.all(c["out"][m[rows]] == 0.0) and np.all(out[m] == 0.0), T      # masks: exact zeros


def test_draws_leave_the_generators_where_the_reference_does(golden):
    for c in golden:
        T = c["x"].shape[1]
        _seed(c["seed"])
        rec = spec_augment_draws([T])[0]
        assert np.array_equal(_probes(), c["probes"]), T
        dr = c["draw"]
        assert (int(rec["idx"]), int(rec["d"]), int(rec["f0"]), int(rec["f"])) == (dr["idx"], dr["d"], dr["f0"], dr["f"])
        assert int(rec["t"]) == (dr["t"] if dr["t"] <= T else 0)
        assert int(rec["t0"]) == (dr["t0"] if dr["t"] <= T else 0)
        assert np.array_equal(rec["Z"], dr["Z"])


def test_draws_match_the_oracle_over_a_batch():
    frames = [11, 12, 640, 47, 1000, 300, 11]
    _seed(7)
    got = spec_augment_draws(frames)
    p_got = _probes()
    _seed(7)
    ref = SA.draws(frames)
    assert np.array_equal(_probes(), p_got)
    assert np.array_equal(got, _records(ref))


@pytest.mark.parametrize("T", [10, 7])
def test_short_utterance_raises_value_error(T):
    with pytest.raises(ValueError):
        spec_augment_draws([40, T])
    with pytest.raises(ValueError):
        SA.draws([T])


@pytest.mark.parametrize("conf", [dict(noise_dir="/data/noise"), dict(speed_volume_perturb=True),
                                  dict(spec_augment=True, noise_dir="/data/noise")])
def test_unsupported_augmentation_raises(conf):
    with pytest.raises(ds.Ds2Error, match="not implemented"):
        SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=ds.AugmentationConfig(**conf))


def test_spec_augment_batch_needs_a_cuda_tensor():
    with pytest.raises(ds.Ds2Error):
        spec_augment_batch(torch.zeros(1, 1, 161, 20), [20])


def test_draws_record_matches_the_c_struct():
    class Draws(ctypes.Structure):            # Ds2SpecAugDraws, include/ds2_b200.h
        _fields_ = [("idx", ctypes.c_int32), ("d", ctypes.c_int32), ("f0", ctypes.c_int32), ("f", ctypes.c_int32),
                    ("t0", ctypes.c_int32), ("t", ctypes.c_int32), ("Z", ctypes.c_float * 9),
                    ("reserved", ctypes.c_int32)]
    assert ctypes.sizeof(Draws) == SPEC_AUG_DRAWS_DTYPE.itemsize
    for name in SPEC_AUG_DRAWS_DTYPE.names:
        assert getattr(Draws, name).offset == SPEC_AUG_DRAWS_DTYPE.fields[name][1], name


def test_kernels_do_not_spill():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    lines = txt.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if "Function" in line and "spec_augment" in line:
            found += 1
            assert "STACK:0 " in lines[i + 1] and "LOCAL:0 " in lines[i + 1], (line, lines[i + 1])
    assert found == 2


# ---------------------------------------------------------------------------------------------------------------- GPU

def _ragged(xs):
    Tmax = max(x.shape[1] for x in xs)
    batch = np.zeros((len(xs), 1, xs[0].shape[0], Tmax), np.float32)
    for b, x in enumerate(xs):
        batch[b, 0, :, :x.shape[1]] = x
    return batch


@pytest.mark.gpu
def test_gpu_kernel_matches_reference_fixture(golden):
    xs = [c["x"] for c in golden]
    frames = [x.shape[1] for x in xs]
    draws = []
    for c, T in zip(golden, frames):
        dr = dict(c["draw"])
        if dr["t"] > T:
            dr["t0"], dr["t"] = 0, 0
        draws.append(dr)
    inp = torch.from_numpy(_ragged(xs)).cuda()
    keep = inp.clone()
    out = spec_augment_batch(inp, frames, _records(draws))
    torch.cuda.synchronize()
    assert torch.equal(inp, keep)                                   # the input is left alone
    got = out.cpu().numpy()
    for b, c in enumerate(golden):
        T = frames[b]
        err = np.abs(got[b, 0, c["rows"], :T] - c["out"]).max()
        print(f"\n[spec_augment] T={T} max|flow|={c['max_flow']:.3g}: max abs err vs reference {err:.2e}")
        assert err <= _out_tol(c["max_flow"]), (T, err)
        # every row (the fixture keeps a subset of rows at T = 1000) against the float64 oracle
        oerr = np.abs(got[b, 0, :, :T] - SA.spec_augment(c["x"], draws[b])[0]).max()
        assert oerr <= _out_tol(c["max_flow"]), (T, oerr)
        m = _mask(c["x"].shape, draws[b])
        assert np.all(got[b, 0, :, :T][m] == 0.0)                   # mask regions exactly 0
        assert np.all(got[b, 0, :, T:] == 0.0)                      # padding exactly 0


def _pcm(n, seed, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi))
        t = np.arange(L) / 16000.0
        y = 0.3 * np.sin(2 * np.pi * (150 + 53 * i) * t) * (1 + 0.4 * np.sin(2 * np.pi * 2.1 * t))
        out.append((y + 0.05 * rng.standard_normal(L)).astype(np.float32))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [3, 302])
def test_gpu_batcher_matches_oracle_in_dataset_order(seed):
    waves = _pcm(7, seed, 1700, 60000) + [_pcm(1, 9, 1600, 1601)[0]]    # ragged, the last one T = 11
    transcripts = [[1 + (i % 27)] * (1 + i) for i in range(len(waves))]
    batcher = SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=ds.AugmentationConfig(spec_augment=True))
    _seed(seed)
    inputs, targets, pct, tsz = batcher(waves, transcripts)
    torch.cuda.synchronize()
    p_gpu = _probes()
    _seed(seed)
    specs = [SO.compute_spectrogram(w).astype(np.float32) for w in waves]
    draws = SA.draws([s.shape[1] for s in specs])
    assert np.array_equal(_probes(), p_gpu)
    aug = [SA.spec_augment(s, dr) for s, dr in zip(specs, draws)]
    r_in, r_t, r_pct, r_tsz = SO.collate([(o, tr) for (o, _), tr in zip(aug, transcripts)])
    assert tuple(inputs.shape) == r_in.shape and targets.tolist() == r_t.tolist()
    assert np.array_equal(pct.numpy(), r_pct) and tsz.tolist() == r_tsz.tolist()
    got = inputs.cpu().numpy()
    order = sorted(range(len(waves)), key=lambda i: specs[i].shape[1], reverse=True)
    for row, i in enumerate(order):
        T = specs[i].shape[1]
        flow = aug[i][1]
        err = np.abs(got[row, 0, :, :T] - r_in[row, 0, :, :T]).max()
        assert err <= 2e-4 + _out_tol(float(np.abs(flow).max())), (i, T, err)
        assert np.all(got[row, 0, :, :T][_mask(specs[i].shape, draws[i])] == 0.0)
        assert np.all(got[row, 0, :, T:] == 0.0)


@pytest.mark.gpu
def test_gpu_same_seed_gives_bit_identical_batches():
    waves = _pcm(6, 4, 3000, 90000)
    transcripts = [[2, 3]] * len(waves)
    conf = ds.AugmentationConfig(spec_augment=True)
    _seed(11)
    a = SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=conf)(waves, transcripts)[0]
    _seed(11)
    b = SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=conf)(waves, transcripts)[0]
    plain = SpectrogramBatcher(ds.SpectConfig())(waves, transcripts)[0]
    off = SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=ds.AugmentationConfig())(waves, transcripts)[0]
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(plain, off)                      # augmentation off: the plain batch, byte for byte
    assert not torch.equal(a, plain)


@pytest.mark.gpu
def test_gpu_spec_augment_batch_rejects_short_utterances():
    x = torch.zeros(2, 1, 161, 40, device="cuda")
    with pytest.raises(ValueError):
        spec_augment_batch(x, [40, 10])
    with pytest.raises(ds.Ds2Error):
        spec_augment_batch(x, [40, 10], spec_augment_draws([40, 40]))


@pytest.mark.gpu
def test_gpu_augmented_batch_feeds_the_train_step():
    from gpu_helpers import make_model
    waves = _pcm(4, 2, 6000, 12000)
    transcripts = [[3, 5, 7], [2, 2, 9, 1], [4], [8, 6]]
    _seed(0)
    batch = SpectrogramBatcher(ds.SpectConfig(), augmentation_conf=ds.AugmentationConfig(spec_augment=True))(
        waves, transcripts)
    ds.set_precision("fp32")
    model = make_model("gru", True, 16, 1).train()
    loss = model.training_step(batch, 0)
    loss.backward()
    assert torch.isfinite(loss) and float(loss) > 0
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
