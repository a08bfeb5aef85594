"""-m gpu: the resident split-K backward sweep exchanges its partial dh_rec tiles either through distributed shared
memory inside 4-CTA clusters or, when the clusters of both directions do not fit the GPU at once, through L2 between
plain cooperative CTAs.  Both paths run the same MMAs and sum the same tiles in the same order, so every output of a
layer call must be bit-identical between them (DS2_SPLITK_XCHG forces either path)."""
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3), "tanh": (_lib.RNN_TANH, 1)}


def _layer(rnn, T, B, In, H, bidir, lens, seed):
    """one RnnLayer forward + backward on seeded inputs; run() returns y, hn, dx and every weight / bias gradient"""
    code, G = CODES[rnn]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, B, In, generator=g).cuda()
    lens = torch.tensor(lens, dtype=torch.int32)
    dy = torch.randn(T, B, H, generator=g).cuda()
    for b in range(B):
        x[int(lens[b]):, b] = 0
        dy[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    ws = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda().requires_grad_(True) for s in
          [(G * H, In), (G * H, H), (G * H,), (G * H,)] * (2 if bidir else 1)]
    lens_dev = lens.cuda()

    def run():
        for w in ws:
            w.grad = None
        xx = x.clone().requires_grad_(True)
        y, hn, _ = ds.ops.RnnLayer.apply(xx, lens_dev, code, bidir, True, 0.1, 1e-5, None, None, None, None, None,
                                         None, *ws)
        y.backward(dy)
        torch.cuda.synchronize()
        return [y.detach(), hn.detach(), xx.grad.clone()] + [w.grad.clone() for w in ws]
    return run


def _run_with(run, monkeypatch, xchg):
    if xchg is None:
        monkeypatch.delenv("DS2_SPLITK_XCHG", raising=False)
    else:
        monkeypatch.setenv("DS2_SPLITK_XCHG", xchg)
    lib = ds.get_lib()
    lib.ds2_fallback_count(1)
    out = run()
    assert lib.ds2_fallback_count(1) == 0, "a sweep fell back to the per-step FFMA kernels"
    monkeypatch.delenv("DS2_SPLITK_XCHG", raising=False)
    return out


def _assert_identical(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), f"output {i} differs: max |diff| {float((u - v).abs().max())}"


def _ragged(T, B):
    """descending lengths with a long tail, the last two utterances fully masked"""
    lens = sorted([max(0, T - 3 * i) for i in range(B)], reverse=True)
    lens[0] = T
    lens[-2:] = [0, 0]
    return lens


@pytest.mark.parametrize("prec", ["fp16", "tf32"])
@pytest.mark.parametrize("rnn,B,bidir", [("lstm", 32, True), ("lstm", 20, True), ("lstm", 40, True),
                                         ("gru", 32, True), ("tanh", 32, True), ("lstm", 32, False)])
def test_l2_exchange_is_bit_identical_to_the_cluster_exchange(rnn, B, bidir, prec, monkeypatch):
    """H = 256: B = 20 pads the batch columns, B = 40 takes a second column pass of the epilogue; GRU, tanh and a
    unidirectional layer; ragged lengths with fully masked utterances.  DS2_SPLITK_CL=4: at these shapes 8-CTA
    clusters would otherwise take the cluster leg (a different K split, so different sums)."""
    monkeypatch.setenv("DS2_SPLITK_CL", "4")
    ds.set_precision(prec)
    try:
        run = _layer(rnn, T=37, B=B, In=160, H=256, bidir=bidir, lens=_ragged(37, B), seed=21)
        _assert_identical(_run_with(run, monkeypatch, "global"), _run_with(run, monkeypatch, "cluster"))
    finally:
        ds.set_precision("fp32")


def test_full_size_layer_one_backward_launch_bit_identical(monkeypatch):
    """bi-LSTM-1024, T' = 500, B = 32, fp16 mode (the benchmarked layer): the default path gives the same bits as the
    cluster exchange, and its backward sweep is ONE launch of rnn_bwd_splitk_kernel for both directions."""
    from torch.profiler import ProfilerActivity, profile
    ds.set_precision("fp16")
    try:
        T, B, H = 500, 32, 1024
        lens = [T - 4 * i for i in range(B)]
        run = _layer("lstm", T=T, B=B, In=H, H=H, bidir=True, lens=lens, seed=5)
        ref = _run_with(run, monkeypatch, "cluster")
        _run_with(run, monkeypatch, None)                       # warm-up of the default path
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got = _run_with(run, monkeypatch, None)
        _assert_identical(got, ref)
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        bwd = [n for n in names if "rnn_bwd_splitk_kernel" in n]
        assert len(bwd) == 1, f"backward sweep launches: {bwd}"
    finally:
        ds.set_precision("fp32")
