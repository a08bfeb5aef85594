"""-m gpu: which recurrent sweep variant runs for a shape, in the precision-16 mode.

For one layer's training step (forward, then backward) the profiler records the sweep kernels that ran in each pass
and how often, and `ds2_fallback_count` the sweeps that fell back to the per-step FFMA kernels.  EXPECTED pins that
table for the shapes of the benchmark workloads, the shapes at the edges of the selection and each of the switches
of DESIGN §6.1.  Separately: a backward sweep that runs on the forward pass's fp16 W_hh^T makes no fp32 transposes."""
import re

import pytest
import torch
from torch.autograd import DeviceType

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3), "tanh": (_lib.RNN_TANH, 1)}
SWEEP = re.compile(r"ds2::(rnn_(?:fwd|bwd|step)_\w*kernel(?:<[^>]*>)?)")

# case: (rnn, H, B, bidirectional, initial state, switches)
CASES = {
    "bilstm1024_b32": ("lstm", 1024, 32, True, False, {}),
    "unigru1024_b32": ("gru", 1024, 32, False, False, {}),
    "bigru256_b4": ("gru", 256, 4, True, False, {}),
    "bilstm1536_b8": ("lstm", 1536, 8, True, False, {}),
    "bitanh1024_b32": ("tanh", 1024, 32, True, False, {}),
    "bilstm160_b16": ("lstm", 160, 16, True, False, {}),
    "bilstm256_b96": ("lstm", 256, 96, True, False, {}),
    "bilstm1024_b1_state": ("lstm", 1024, 1, True, True, {}),
    "no_resident": ("lstm", 1024, 32, True, False, {"DS2_NO_RESIDENT": "1"}),
    "no_splitk": ("lstm", 1024, 32, True, False, {"DS2_NO_SPLITK": "1"}),
    "fwd_splitk_off": ("lstm", 1024, 32, True, False, {"DS2_FWD_SPLITK": "0"}),
    "splitk_cl4": ("lstm", 1024, 32, True, False, {"DS2_SPLITK_CL": "4"}),
    "xchg_cluster": ("lstm", 1024, 32, True, False, {"DS2_SPLITK_XCHG": "cluster"}),
    "xchg_global": ("lstm", 1024, 32, True, False, {"DS2_SPLITK_XCHG": "global"}),
}

EXPECTED = {   # what runs, as observed on an H100 SXM (132 SMs)
    "bigru256_b4": {"fwd": {"rnn_fwd_splitk_kernel<1, 0>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<1, true, 4, 0, false>": 1}, "fallbacks": 0},
    "bilstm1024_b1_state": {"fwd": {"rnn_fwd_splitk_state_kernel<0, 8>": 1},
     "bwd": {}, "fallbacks": 0},
    "bilstm1024_b32": {"fwd": {"rnn_fwd_splitk_kernel<0, 8>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 16, true>": 1}, "fallbacks": 0},
    "bilstm1536_b8": {"fwd": {"rnn_fwd_persist_kernel<0, false, false>": 2},
     "bwd": {"rnn_bwd_splitk_kernel<0, false, 4, 0, false>": 2}, "fallbacks": 0},
    "bilstm160_b16": {"fwd": {"rnn_fwd_persist_kernel<0, false, false>": 1},
     "bwd": {"rnn_bwd_persist_kernel<0>": 1}, "fallbacks": 0},
    "bilstm256_b96": {"fwd": {"rnn_fwd_persist_kernel<0, true, false>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 0, false>": 1}, "fallbacks": 0},
    "bitanh1024_b32": {"fwd": {"rnn_fwd_persist_kernel<2, true, false>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<2, true, 4, 4, true>": 1}, "fallbacks": 0},
    "fwd_splitk_off": {"fwd": {"rnn_fwd_persist_kernel<0, true, false>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 16, true>": 1}, "fallbacks": 0},
    "no_resident": {"fwd": {"rnn_fwd_persist_kernel<0, false, false>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, false, 4, 0, false>": 2}, "fallbacks": 0},
    "no_splitk": {"fwd": {"rnn_fwd_splitk_kernel<0, 8>": 1},
     "bwd": {"rnn_bwd_persist_kernel<0>": 1}, "fallbacks": 0},
    "splitk_cl4": {"fwd": {"rnn_fwd_splitk_kernel<0, 8>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 16, true>": 1}, "fallbacks": 0},
    "unigru1024_b32": {"fwd": {"rnn_fwd_splitk_kernel<1, 8>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<1, true, 8, 6, false>": 1}, "fallbacks": 0},
    "xchg_cluster": {"fwd": {"rnn_fwd_splitk_kernel<0, 8>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 16, false>": 2}, "fallbacks": 0},
    "xchg_global": {"fwd": {"rnn_fwd_splitk_kernel<0, 8>": 1},
     "bwd": {"rnn_bwd_splitk_kernel<0, true, 4, 16, true>": 1}, "fallbacks": 0},
}


def _sweep_kernels(prof):
    """{sweep kernel name with its template arguments: launches} of one profiled window"""
    out = {}
    for e in prof.key_averages():
        m = SWEEP.search(e.key)
        if m:
            out[m.group(1)] = out.get(m.group(1), 0) + e.count
    return out


def _layer(rnn, H, B, bidir, state, T=24, In=96, seed=5):
    code, G = CODES[rnn]
    D = 2 if bidir else 1
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor(sorted([max(1, T - 2 * i) for i in range(B)], reverse=True), dtype=torch.int32)
    x = torch.randn(T, B, In, generator=g)
    dy = torch.randn(T, B, H, generator=g)
    for b in range(B):
        x[int(lens[b]):, b] = 0
        dy[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    ws = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda().requires_grad_(not state) for s in
          [(G * H, In), (G * H, H), (G * H,), (G * H,)] * D]
    h0 = ((torch.rand(D, B, H, generator=g) * 2 - 1) * 0.9).cuda() if state else None
    x, dy, lens = x.cuda(), dy.cuda(), lens.cuda()

    def forward():
        xx = x.clone().requires_grad_(not state)
        y, _, _ = ds.ops.RnnLayer.apply(xx, lens, code, bidir, not state, 0.1, 1e-5, None, None, None, None, h0, None,
                                        *ws)
        return y
    return forward, dy


def _profiled_step(forward, dy):
    """(forward kernel events, backward kernel events) of one training step, or of one forward when dy is None; the
    profiler can miss a window's kernel records, so the step is repeated until both windows have some"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as pf:
            y = forward()
            torch.cuda.synchronize()
        pb = None
        if dy is not None:
            with profile(activities=[ProfilerActivity.CUDA]) as pb:
                y.backward(dy)
                torch.cuda.synchronize()
        if _sweep_kernels(pf) and (pb is None or _sweep_kernels(pb)):
            break
    return pf, pb


def observe(case, precision="fp16"):
    rnn, H, B, bidir, state, env = CASES[case]
    forward, dy = _layer(rnn, H, B, bidir, state)
    lib = ds.get_lib()
    mp = pytest.MonkeyPatch()
    try:
        for k, v in env.items():
            mp.setenv(k, v)
        ds.set_precision(precision)
        lib.ds2_fallback_count(1)
        if state:
            with torch.no_grad():
                pf, pb = _profiled_step(forward, None)
        else:
            pf, pb = _profiled_step(forward, dy)
        fallbacks = int(lib.ds2_fallback_count(1))
    finally:
        mp.undo()
        ds.set_precision("fp32")
    return {"fwd": _sweep_kernels(pf), "bwd": _sweep_kernels(pb) if pb is not None else {},
            "fallbacks": fallbacks}, pb


@pytest.mark.parametrize("case", sorted(CASES))
def test_sweep_variant_for_shape_and_switches(case):
    got, _ = observe(case)
    assert got == EXPECTED[case]


@pytest.mark.parametrize("precision", ["fp16", "tf32"])
@pytest.mark.parametrize("case", ["bilstm1024_b32", "bigru256_b4"])
def test_backward_on_the_fp16_weights_makes_no_fp32_transposes(case, precision):
    """the forward pass leaves an fp16 W_hh^T for the backward; a sweep that runs on it needs no fp32 transposes.
    (In the tf32 mode the weight-gradient GEMMs transpose operands too, after the sweep.)"""
    got, pb = observe(case, precision)
    assert got["fallbacks"] == 0
    kern = sorted((e.time_range.start, e.name) for e in pb.events() if e.device_type == DeviceType.CUDA)
    sweep_start = min(t for t, n in kern if SWEEP.search(n))
    before = [n for t, n in kern if t < sweep_start and "transpose_strided_kernel" in n]
    assert not before, f"{len(before)} fp32 transposes before the backward sweep"
