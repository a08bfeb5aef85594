"""-m gpu: the wgmma forward sweeps with an initial state h0 / c0 (chunked transcription carries each chunk's final
states into the next chunk's forward).

* kernels: `ops.RnnLayer` with random h0 / c0 (|h| < 1) in the fp16 and tf32 modes against the fp32 FFMA path, on
  the split-K state kernel (LSTM / GRU, H in {128, 640, 1024, 1152}, B in {1, 20, 32, 48, 64}) and the 16-unit
  resident kernel (H = 256 / 320, B up to 128), uni- and bidirectional, ragged lengths with zero-length utterances,
  h0 only and c0 only; the kernel that ran is read from the profiler; no fallback, exact zeros at padded steps,
  hn / cn = h0 / c0 bit for bit where len = 0, bit repeatability.  The shapes that still fall back with a state are
  pinned too;
* the reference: tests/golden/chunked/*.npz (oracle/make_chunked_golden.py) holds the reference's own
  `DeepSpeech.forward` over 3 chunks carrying `hs`;
* full size: 5 x bi-LSTM-1024 in precision 16, B = 1, 3 chunks of 500 frames, against the fp32 path."""
import glob
import json
import os

import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib
from gpu_helpers import make_model, rel, rel_l2

pytestmark = pytest.mark.gpu

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3), "tanh": (_lib.RNN_TANH, 1)}
CHUNKED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "chunked")


def _kernels(fn):
    """names of the library's kernels `fn` launches (the profiler can miss a window's kernel records: it is asked
    again until it has some)"""
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.key for e in prof.key_averages() if "ds2::" in e.key}
        if names:
            break
    return names


def _ran(names, kernel):
    return any(kernel in n for n in names)


def _layer(rnn, T, B, In, H, bidir, state, seed):
    code, G = CODES[rnn]
    D = 2 if bidir else 1
    g = torch.Generator().manual_seed(seed)
    lens = sorted([max(0, T - 3 * i) for i in range(B)], reverse=True)
    lens[0] = T
    if B >= 4:
        lens[-2:] = [0, 0]
    lens = torch.tensor(lens, dtype=torch.int32)
    x = torch.randn(T, B, In, generator=g)
    for b in range(B):
        x[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    ws = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda() for s in
          [(G * H, In), (G * H, H), (G * H,), (G * H,)] * D]
    h0 = ((torch.rand(D, B, H, generator=g) * 2 - 1) * 0.9).cuda() if state in ("both", "h0") else None
    c0 = ((torch.rand(D, B, H, generator=g) * 2 - 1) * 0.9).cuda() if rnn == "lstm" and state in ("both", "c0") else None
    x, lens_dev = x.cuda(), lens.cuda()

    def run():
        with torch.no_grad():
            y, hn, cn = ds.ops.RnnLayer.apply(x, lens_dev, code, bidir, False, 0.1, 1e-5, None, None, None, None, h0,
                                              c0, *ws)
        torch.cuda.synchronize()
        return [t.clone() for t in (y, hn, cn) if t is not None]
    return run, lens, h0, c0


def _check(rnn, T, B, In, H, bidir, state, prec, kernel):
    run, lens, h0, c0 = _layer(rnn, T, B, In, H, bidir, state, seed=B * 7 + H)
    ds.set_precision("fp32")
    ref = run()
    ds.set_precision(prec)
    try:
        lib = ds.get_lib()
        lib.ds2_fallback_count(1)
        got = run()
        again = run()
        assert lib.ds2_fallback_count(1) == 0, "a sweep with an initial state fell back to the per-step FFMA kernels"
        names = _kernels(run)
    finally:
        ds.set_precision("fp32")
    for b in range(B):
        L = int(lens[b])
        if L < T:
            assert float(got[0][L:, b].abs().max()) == 0.0, f"padded outputs of utterance {b} are not 0"
        if L == 0:   # hn / cn are the initial state (zeros where it is not given), bit for bit
            assert torch.equal(got[1][:, b], h0[:, b] if h0 is not None else torch.zeros_like(got[1][:, b]))
            if rnn == "lstm":
                assert torch.equal(got[2][:, b], c0[:, b] if c0 is not None else torch.zeros_like(got[2][:, b]))
    for a, r in zip(got, ref):
        assert rel(a, r) < 5e-3, (rel(a, r), rel_l2(a, r))
    for a, b_ in zip(got, again):
        assert torch.equal(a, b_), "not bit-repeatable"
    assert _ran(names, kernel), f"{kernel} did not run: {sorted(names)}"


@pytest.mark.parametrize("prec", ["fp16", "tf32"])
@pytest.mark.parametrize("rnn,B,H,bidir,state", [
    ("lstm", 1, 1024, True, "both"), ("gru", 1, 1024, True, "h0"), ("lstm", 32, 1024, True, "both"),
    ("gru", 64, 1024, False, "h0"), ("lstm", 1, 1024, True, "h0"), ("lstm", 20, 1024, True, "c0"),
    ("lstm", 48, 1024, True, "both"), ("gru", 64, 1024, True, "h0"), ("lstm", 1, 1152, True, "both"),
    ("gru", 20, 1152, True, "h0"), ("lstm", 32, 1152, False, "c0"), ("gru", 20, 640, True, "h0"),
    ("lstm", 64, 640, True, "both"), ("lstm", 1, 640, False, "both"), ("lstm", 48, 128, True, "h0"),
    ("gru", 1, 128, True, "h0")])
def test_split_k_sweep_with_initial_state(rnn, B, H, bidir, state, prec):
    _check(rnn, 29, B, 96, H, bidir, state, prec, "rnn_fwd_splitk_state_kernel")


@pytest.mark.parametrize("prec", ["fp16", "tf32"])
@pytest.mark.parametrize("rnn,B,H,bidir,state", [
    ("tanh", 65, 320, True, "h0"), ("tanh", 100, 320, False, "h0"), ("tanh", 128, 320, True, "h0"),
    ("lstm", 100, 320, True, "both"), ("gru", 128, 320, True, "h0"),
    # split-K shapes whose chunk count has no state kernel (H / 128 = 2)
    ("lstm", 20, 256, True, "h0"), ("lstm", 48, 256, False, "c0"), ("gru", 48, 256, True, "h0")])
def test_16_unit_sweep_with_initial_state(rnn, B, H, bidir, state, prec):
    _check(rnn, 23, B, 64, H, bidir, state, prec, "rnn_fwd_persist_kernel")


@pytest.mark.parametrize("B,H", [(1, 1280), (48, 768), (64, 896)])
def test_shapes_without_a_wgmma_state_sweep_fall_back_loudly(B, H):
    """no state kernel at these H / 128 and the 16-unit kernel does not fit: the FFMA step kernels, counted"""
    run, _, _, _ = _layer("lstm", 9, B, 32, H, False, "both", seed=1)
    ds.set_precision("fp16")
    try:
        lib = ds.get_lib()
        lib.ds2_fallback_count(1)
        run()
        assert lib.ds2_fallback_count(1) == 1
    finally:
        ds.set_precision("fp32")


# ---------------------------------------------------------------------------------------- against the reference
def _chunked_model(meta, z):
    torch.manual_seed(123456)          # the reference's seed: the default initialisation draw for draw
    model = make_model(meta["rnn_type"], meta["bidirectional"], meta["hidden_size"], meta["hidden_layers"],
                       meta["lookahead_context"] or 20, device="cpu")
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for k, v in model.state_dict().items():
            if k.endswith("running_mean"):
                v.copy_(0.05 * torch.randn(v.shape, generator=g))
            elif k.endswith("running_var"):
                v.copy_(1.0 + 0.2 * torch.rand(v.shape, generator=g))
    for k, v in model.state_dict().items():
        s, a = float(v.double().sum()), float(v.double().abs().sum())
        assert abs(s - float(z["psum/" + k])) <= 1e-9 * max(1.0, a) and abs(a - float(z["pabs/" + k])) <= 1e-9 * max(1.0, a), k
    return model.cuda().eval()


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(CHUNKED, "*.npz"))),
                         ids=lambda p: os.path.splitext(os.path.basename(p))[0])
def test_chunked_forward_carrying_hs_matches_the_reference(path, prec):
    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    model = _chunked_model(meta, z)
    lib = ds.get_lib()
    ds.set_precision(prec)
    try:
        lib.ds2_fallback_count(1)
        hs = None
        for c in range(meta["chunks"]):
            with torch.no_grad():
                out, out_sizes, hs = model(torch.from_numpy(z[f"x/{c}"]).cuda(), torch.from_numpy(z[f"sizes/{c}"]), hs)
            assert out_sizes.tolist() == z[f"out_sizes/{c}"].tolist()
            ref_out = torch.from_numpy(z[f"out/{c}"])
            states = [(h if isinstance(h, tuple) else (h,)) for h in hs]
            ref_states = [(torch.from_numpy(z[f"hn/{c}/{i}"]),) +
                          ((torch.from_numpy(z[f"cn/{c}/{i}"]),) if f"cn/{c}/{i}" in z.files else ())
                          for i in range(len(hs))]
            if prec == "fp32":
                assert rel(out, ref_out) < 1e-3, (c, rel(out, ref_out))
                for s, r in zip(states, ref_states):
                    for a, b_ in zip(s, r):
                        assert rel(a, b_) < 1e-3, (c, rel(a, b_))
            else:
                assert rel(out, ref_out) < 2e-2 and rel_l2(out, ref_out) < 1e-2, (c, rel(out, ref_out))
                for s, r in zip(states, ref_states):
                    for a, b_ in zip(s, r):
                        assert rel_l2(a, b_) < 1e-2, (c, rel_l2(a, b_))
        if prec == "fp16":
            assert lib.ds2_fallback_count(1) == 0, "a sweep fell back to the per-step FFMA kernels"
            # the chunks after the first ran the state kernels: H = 128 split-K, H = 64 the 16-unit kernel
            kernel = "rnn_fwd_splitk_state_kernel" if meta["hidden_size"] % 128 == 0 else "rnn_fwd_persist_kernel"
            with torch.no_grad():
                names = _kernels(lambda: model(torch.from_numpy(z["x/1"]).cuda(), torch.from_numpy(z["sizes/1"]), hs))
            assert _ran(names, kernel), f"{kernel} did not run: {sorted(names)}"
    finally:
        ds.set_precision("fp32")


# ---------------------------------------------------------------------------------------- full size
def test_fullsize_bilstm_1024_precision_16_three_chunks_carrying_hs():
    torch.manual_seed(0)
    model = ds.DeepSpeech(ds.LABELS, ds.BiDirectionalConfig(), 16, ds.AdamConfig(), ds.SpectConfig()).cuda().eval()
    g = torch.Generator().manual_seed(3)
    chunks = [torch.randn(1, 1, 161, 1000, generator=g).cuda() for _ in range(3)]   # T' = 500 per chunk
    sizes = torch.tensor([1000], dtype=torch.int32)
    lib = ds.get_lib()

    def run(precision):
        model.precision = precision
        outs, hs = [], None
        with torch.no_grad():
            for x in chunks:
                out, _, hs = model(x, sizes, hs)
                outs.append(out)
        return outs, hs
    ds.set_precision("fp32")
    ref_outs, ref_hs = run(32)
    lib.ds2_fallback_count(1)
    outs, hs = run(16)
    assert lib.ds2_fallback_count(1) == 0, "a chunk's forward fell back to the per-step FFMA kernels"
    for c, (a, r) in enumerate(zip(outs, ref_outs)):
        print(f"chunk {c}: out rel {rel(a, r):.2e} rel-L2 {rel_l2(a, r):.2e}")
        assert rel(a, r) < 2e-2 and rel_l2(a, r) < 1e-2, c
    for i, (s, r) in enumerate(zip(hs, ref_hs)):
        for a, b_ in zip(s, r):
            print(f"layer {i}: state rel-L2 {rel_l2(a, b_):.2e}")
            assert rel_l2(a, b_) < 2e-2, i
