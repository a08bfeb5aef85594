"""-m gpu: the kernels of the step outside the GEMMs, the recurrent sweeps and the conv front-end, against float64 at
the benchmarked shapes and at their edges: sequence-wise BatchNorm (`csrc/bn.cu`, through the fc head and through a
recurrent layer), the fc head's forward and backward, Lookahead, CTC and the greedy decoder.

Kernels that reduce over rows are compared per column (`col_err`): the maximum error over a whole tensor hides a single
wrong feature column.  Where the fp32 rounding floor is not obvious, the same operation runs through ATen in fp32 on
the GPU (TF32 off) as a yardstick, and the kernel must be within 2x the yardstick's error plus a stated floor.

The BatchNorm inputs carry near-constant columns (mean 0.76 .. 10, std 0.01 .. 0.001), which is what saturated LSTM
units feed the next layer: the sum of two directions of h sits near +-2 with a tiny spread.  Statistics formed as
E[x^2] - E[x]^2 from fp32 partial sums cancel there; the kernels must stay within 1e-5 of float64 all the same."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_helpers import rel_l2
from oracle import ds2_oracle as O

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS, MOM = 1e-5, 0.1


@pytest.fixture(autouse=True)
def _fp32():
    ds.set_precision("fp32")
    yield


class _no_tf32:
    """ATen yardstick arithmetic: cuBLAS / cuDNN in plain fp32"""

    def __enter__(self):
        self.saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def col_err(a, b):
    """per column of two (..., F) tensors: max |a - b| / max |b| over the rows of that column (plain max |a - b| where
    the column of b is all zero).  Returns F float64 values."""
    b = torch.as_tensor(b).detach().double()
    a = torch.as_tensor(a).detach().to(b.device).double()
    a, b = a.reshape(-1, a.shape[-1]), b.reshape(-1, b.shape[-1])
    num, den = (a - b).abs().amax(0), b.abs().amax(0)
    return torch.where(den > 0, num / torch.where(den > 0, den, torch.ones_like(den)), num)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    lib = ds.get_lib()
    rc = getattr(lib, name)(*args)
    assert rc == 0, f"{name}: {lib.ds2_last_error().decode(errors='replace')}"


def _report(failures, name, got, yard, floor, extra=0.0):
    """yardstick rule: got <= 2 * yard + floor (+ extra, a per-column allowance where given).  `got` and `extra` may
    be per-column vectors; `yard` is the yardstick's worst column.  Prints both, records a failure."""
    got, extra = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(extra, dtype=torch.float64)
    over = got > 2.0 * yard + floor + extra
    ok = not bool(over.any())
    print(f"  {name:<14} kernel {float(got.max()):.2e}  ATen fp32 {yard:.2e}  floor {floor:.0e}"
          f"{f'  allowance <= {float(extra.max()):.1e}' if float(extra.max()) > 0 else ''}  {'ok' if ok else 'FAIL'}",
          flush=True)
    if not ok:
        failures.append((name, over.nonzero().flatten().tolist()[:8], float(got.max()), yard, floor))


# ---------------------------------------------------------------------------------------------------------------------
# 1. Sequence-wise BatchNorm (fc head, recurrent layers 1-4)
# ---------------------------------------------------------------------------------------------------------------------
OFFSET_COLS = [(0.76, 0.01), (1.9, 0.01), (5.0, 0.01), (10.0, 0.001)]   # (mean, std) of features 1 .. 4
CONST = 2.7                                                           # feature F-2; feature F-1 is all zero


def bn_input(T, B, Fe, seed, lens=None):
    """(T, B, F) fp32: N(0, 1) features, the offset features of OFFSET_COLS, one exactly constant and one all-zero
    feature; rows t >= lens[b] are zero (padding, included in the statistics like the reference's)"""
    x = torch.randn(T, B, Fe, generator=torch.Generator().manual_seed(seed))
    for j, (mu, sd) in enumerate(OFFSET_COLS):
        x[..., 1 + j] = mu + sd * x[..., 1 + j]
    x[..., Fe - 2] = CONST
    x[..., Fe - 1] = 0.0
    if lens is not None:
        for b, n in enumerate(lens):
            x[n:, b] = 0.0
    return x.to(DEV)


def check_stats(tag, x2d, rm, rv, mean=None, invstd=None):
    """per feature, against float64: the running statistics one training forward leaves behind (started at 0, so
    that the unbiased variance is not swamped by 0.9 x 1) and, where the caller has them, the batch statistics (invstd
    within 1e-5 relative, mean within 2^-23 |mean| + 1e-6 std).  Returns a list of failure descriptions."""
    rows, Fe = x2d.shape
    x64 = x2d.double()
    mean64, var64 = x64.mean(0), x64.var(0, unbiased=False)
    std64 = var64.sqrt()
    invstd64 = (var64 + EPS).rsqrt()
    # running statistics: two fp32 roundings (the statistic, the momentum product) -> 2^-22 for the mean
    rm64 = MOM * mean64
    rv64 = MOM * var64 * (rows / (rows - 1) if rows > 1 else 1.0)
    checks = [("running_mean", (rm.double() - rm64).abs() > 2.0 ** -22 * rm64.abs() + 1e-7 * std64),
              ("running_var", (rv.double() - rv64).abs() > 2e-5 * rv64)]
    rv_err = (rv.double() - rv64).abs() / torch.where(rv64 > 0, rv64, torch.ones_like(rv64))
    # the yardstick for the statistics: ATen's own BatchNorm kernel (Welford) on the same fp32 data
    _, _, a_invstd = torch.ops.aten.native_batch_norm(x2d, None, None, None, None, True, MOM, EPS)
    a_inv_err = (a_invstd.double() - invstd64).abs() / invstd64
    if invstd is not None:
        inv_err = (invstd.double() - invstd64).abs() / invstd64
        checks += [("invstd", inv_err > 1e-5),
                   ("mean", (mean.double() - mean64).abs() > 2.0 ** -23 * mean64.abs() + 1e-6 * std64)]
    names = {0: "N(0,1)", Fe - 2: f"const {CONST}", Fe - 1: "zero"}
    names.update({1 + j: f"({mu}, {sd})" for j, (mu, sd) in enumerate(OFFSET_COLS)})
    print(f"\n[bn] {tag}: rows {rows} F {Fe}; relative error per feature: invstd (kernel / ATen fp32), running var",
          flush=True)
    for f, name in sorted(names.items()):
        k = f"{float(inv_err[f]):.1e}" if invstd is not None else "-"
        print(f"  {name:<14} invstd {k} / {float(a_inv_err[f]):.1e}   running var {float(rv_err[f]):.1e}", flush=True)
    bad = []
    for what, mask in checks:
        idx = mask.nonzero().flatten().tolist()
        if idx:
            bad.append(f"{tag} {what}: features {[names.get(f, f) for f in idx[:8]]} ({len(idx)} in all)")
    return bad


def fc_head_fwd(x2d, g, b, rm, rv, w, training, softmax):
    rows, H = x2d.shape
    Cn = w.shape[0]
    logits = torch.empty(rows, Cn, device=DEV)
    xhat = torch.empty(rows, H, device=DEV)
    stats = torch.empty(2 * H, device=DEV)
    ws = torch.empty(ds.get_lib().ds2_fc_head_workspace_bytes(rows, H, Cn), dtype=torch.uint8, device=DEV)
    _call("ds2_fc_head_fwd", rows, H, Cn, _p(x2d), _p(g), _p(b), _p(rm), _p(rv), _p(w), int(training), MOM, EPS,
          int(softmax), _p(logits), _p(xhat), _p(stats), _p(ws), ws.numel(), _stream())
    return logits, xhat, stats


def fc_head_bwd(g, b, w, xhat, stats, dlogits):
    rows, H = xhat.shape
    Cn = w.shape[0]
    dx = torch.empty(rows, H, device=DEV)
    dg, db, dw = torch.empty(H, device=DEV), torch.empty(H, device=DEV), torch.empty(Cn, H, device=DEV)
    ws = torch.empty(ds.get_lib().ds2_fc_head_workspace_bytes(rows, H, Cn), dtype=torch.uint8, device=DEV)
    _call("ds2_fc_head_bwd", rows, H, Cn, _p(g), _p(b), _p(w), _p(xhat), _p(stats), _p(dlogits), _p(dx), _p(dg),
          _p(db), _p(dw), _p(ws), ws.numel(), _stream())
    return dx, dg, db, dw


def bn_linear(x2d, g, b, w, dlogits, dtype):
    """BN (batch statistics) -> Linear, forward and autograd backward, in `dtype` (float64: the reference; float32 on
    the GPU: the ATen yardstick).  ATen's native BatchNorm kernel, whatever cuDNN would do."""
    x, g, b, w = (t.detach().to(dtype).requires_grad_(True) for t in (x2d, g, b, w))
    with _no_tf32():
        y = torch.ops.aten.native_batch_norm(x, g, b, None, None, True, 0.0, EPS)[0]
        logits = y @ w.t()
        logits.backward(dlogits.to(dtype))
    return logits.detach(), x.grad, g.grad, b.grad, w.grad


def sum_err(a, b, scale):
    """per-feature error of a row sum (dgamma, dbeta) in units of the l2 norm of its summands (plain |a - b| where
    every summand is zero)"""
    d = (a.double().to(b.device) - b.double()).abs()
    return torch.where(scale > 0, d / torch.where(scale > 0, scale, torch.ones_like(scale)), d)


BN_SHAPES = [  # id, T', B, F, C, ragged
    ("rows16000_F1024", 500, 32, 1024, 29, False),      # fc head and recurrent layers 1-4 at the benchmark
    ("ragged_F1000", 120, 8, 1000, 29, True),           # F not a multiple of 32, zero padded rows
    ("F29", 300, 4, 29, 29, False),                     # fewer features than one 32-wide block
    ("rows7", 7, 1, 1024, 29, False),                   # < 256 rows: one row chunk, idle row lanes
]


@pytest.mark.parametrize("tag,T,B,Fe,Cn,ragged", BN_SHAPES, ids=[s[0] for s in BN_SHAPES])
def test_fc_head_batchnorm_and_gradients_per_feature(tag, T, B, Fe, Cn, ragged):
    """`ds2_fc_head_fwd/bwd` (BatchNorm1d over all T*B rows -> Linear): per feature, the batch statistics (invstd
    within 1e-5 relative of float64, mean within 2^-23 |mean| + 1e-6 std) and the running statistics; per output
    column, the logits of a training forward, the softmax of an eval forward on running statistics, and dx, dgamma,
    dbeta, dW against float64 autograd, each within 2x the ATen fp32 yardstick + a floor.

    The constant and the all-zero feature have an exact answer: xhat = 0, hence dgamma = 0.  The kernels must
    produce it exactly.

    No fp32 mean of a (10, 0.001) feature is closer to the float64 one than about u = 2^-24 |mean| / std of its std,
    whatever computes it, and xhat carries that error (6e-4 there).  So the yardstick's worst column is taken over
    the features with u < 1e-6, and the kernel is allowed 4 u on top per feature (dx, dgamma, dW) and, through W, per
    class of the logits: both the ATen arm and the kernels round the mean, and which one lands closer is luck."""
    lens = [max(1, T - (T // 2) * i // max(1, B - 1)) for i in range(B)] if ragged else None
    x2d = bn_input(T, B, Fe, seed=Fe + T, lens=lens).reshape(T * B, Fe)
    rows = T * B
    g_ = torch.Generator().manual_seed(7)
    gamma = (1.0 + 0.1 * torch.rand(Fe, generator=g_)).to(DEV)
    beta = (0.1 * torch.randn(Fe, generator=g_)).to(DEV)
    w = ((torch.rand(Cn, Fe, generator=g_) * 2 - 1) / Fe ** 0.5).to(DEV)
    dlogits = torch.randn(rows, Cn, generator=g_).to(DEV)
    rm, rv = torch.zeros(Fe, device=DEV), torch.zeros(Fe, device=DEV)

    logits, xhat, stats = fc_head_fwd(x2d, gamma, beta, rm, rv, w, training=True, softmax=False)
    dx, dg, db, dw = fc_head_bwd(gamma, beta, w, xhat, stats, dlogits)
    torch.cuda.synchronize()
    bad = check_stats(tag, x2d, rm, rv, mean=stats[:Fe], invstd=stats[Fe:])

    ref = bn_linear(x2d, gamma, beta, w, dlogits, torch.float64)
    yard = bn_linear(x2d, gamma, beta, w, dlogits, torch.float32)
    x64 = x2d.double()
    mean64, std64 = x64.mean(0), x64.std(0, unbiased=False)
    xhat64 = (x64 - mean64) * (std64 ** 2 + EPS).rsqrt()
    dy64 = dlogits.double() @ w.double()
    scale_g, scale_b = (dy64 * xhat64).norm(dim=0), dy64.norm(dim=0)
    u = torch.where(std64 > 0, 2.0 ** -24 * mean64.abs() / torch.where(std64 > 0, std64, torch.ones_like(std64)),
                    torch.zeros_like(std64))
    well = u < 1e-6
    exact = [Fe - 1] if ragged else [Fe - 2, Fe - 1]           # the all-zero and (unless padded) constant feature
    well[exact] = False
    if not torch.equal(xhat[:, exact], torch.zeros_like(xhat[:, exact])) or not bool((dg[exact] == 0).all()):
        bad.append(f"{tag}: xhat / dgamma of the constant and the zero feature are not exactly 0")
    # the allowance through W for the logits of class c: sum_f gamma_f u_f |W[c, f]| over the class's scale
    extra_logits = 2.0 * (gamma.double() * u) @ w.double().abs().t() / ref[0].abs().amax(0)
    fails = []
    print(f"[fc head] {tag}: worst per-column error against float64", flush=True)
    _report(fails, "logits", col_err(logits, ref[0]), float(col_err(yard[0], ref[0]).max()), 5e-6, extra_logits)
    _report(fails, "dx", col_err(dx, ref[1]), float(col_err(yard[1], ref[1])[well].max()), 1e-6, 4 * u)
    _report(fails, "dgamma", sum_err(dg, ref[2], scale_g), float(sum_err(yard[2], ref[2], scale_g)[well].max()),
            1e-6, 4 * u)
    _report(fails, "dbeta", sum_err(db, ref[3], scale_b), float(sum_err(yard[3], ref[3], scale_b).max()), 1e-6)
    _report(fails, "dW", col_err(dw, ref[4]), float(col_err(yard[4], ref[4])[well].max()), 1e-5, 4 * u)

    # eval forward (running statistics, InferenceBatchSoftmax): realistic running statistics, the float64 batch ones
    rm_e, rv_e = x64.mean(0).float(), x64.var(0).float()
    probs, _, _ = fc_head_fwd(x2d, gamma, beta, rm_e.clone(), rv_e.clone(), w, training=False, softmax=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        p64 = torch.softmax(torch.ops.aten.native_batch_norm(x64, gamma.double(), beta.double(), rm_e.double(),
                                                              rv_e.double(), False, 0.0, EPS)[0] @ w.double().t(), -1)
        with _no_tf32():
            p32 = torch.softmax(torch.ops.aten.native_batch_norm(x2d, gamma, beta, rm_e, rv_e, False, 0.0, EPS)[0] @
                                w.t(), -1)
    _report(fails, "eval softmax", col_err(probs, p64), float(col_err(p32, p64).max()), 5e-6)
    assert not bad and not fails, (bad, fails)


def test_recurrent_layer_batchnorm_per_feature():
    """`RnnLayer` with BatchNorm (layers 1-4 of the benchmark: bi-LSTM, T' = 500, B = 32, In = 1024; H = 64 keeps the
    float64 reference fast): the running statistics per input feature, and the layer output per hidden unit against
    a float64 BN -> bi-LSTM, within 2x the ATen fp32 (cuDNN) yardstick + 1e-5 + the fp32-mean allowance."""
    T, B, In, H = 500, 32, 1024, 64
    x = bn_input(T, B, In, seed=31)
    lens = torch.full((B,), T, dtype=torch.int32)
    g_ = torch.Generator().manual_seed(8)
    pre = "rnns.0."
    P = {pre + "batch_norm.module.weight": 1.0 + 0.1 * torch.rand(In, generator=g_),
         pre + "batch_norm.module.bias": 0.1 * torch.randn(In, generator=g_),
         pre + "batch_norm.module.running_mean": torch.zeros(In),
         pre + "batch_norm.module.running_var": torch.zeros(In)}
    k = 1.0 / H ** 0.5
    wnames = []
    for sfx in ("", "_reverse"):
        for n, s in (("weight_ih_l0", (4 * H, In)), ("weight_hh_l0", (4 * H, H)), ("bias_ih_l0", (4 * H,)),
                     ("bias_hh_l0", (4 * H,))):
            P[pre + "rnn." + n + sfx] = (torch.rand(s, generator=g_) * 2 - 1) * k
            wnames.append(pre + "rnn." + n + sfx)
    P = {n: v.to(DEV) for n, v in P.items()}
    bn = [P[pre + "batch_norm.module." + n] for n in ("weight", "bias", "running_mean", "running_var")]
    rm, rv = bn[2].clone(), bn[3].clone()
    y, _, _ = ds.ops.RnnLayer.apply(x, lens.to(DEV), _lib.RNN_LSTM, True, True, MOM, EPS, bn[0], bn[1], rm, rv, None,
                                    None, *[P[n] for n in wnames])
    torch.cuda.synchronize()
    # the layer keeps its batch statistics to itself: its running statistics carry them
    bad = check_stats("recurrent layer", x.reshape(T * B, In), rm, rv)

    cfg = O.OracleConfig(rnn_type="lstm", hidden_size=H, hidden_layers=1, bidirectional=True)
    with torch.no_grad():
        P64 = {n: v.double() for n, v in P.items()}
        y64, _ = O.batch_rnn(x.double(), lens.to(DEV), P64, pre, cfg, batch_norm=True, training=True, new_buffers={})
        with _no_tf32():
            y32, _ = O.batch_rnn_aten(x, lens, {n: v.clone() for n, v in P.items()}, pre, cfg, batch_norm=True,
                                      training=True, new_buffers={})
    # allowance for the fp32 mean of the offset features (see the fc head test): u_f in units of std, carried
    # through gamma and W_ih into the gate pre-activations, 4x that per hidden unit's scale
    x64 = x.reshape(T * B, In).double()
    m64, s64 = x64.mean(0), x64.std(0, unbiased=False)
    u = torch.where(s64 > 0, 2.0 ** -24 * m64.abs() / torch.where(s64 > 0, s64, torch.ones_like(s64)),
                    torch.zeros_like(s64))
    w_max = torch.stack([P[pre + "rnn.weight_ih_l0" + s].abs().amax(0) for s in ("", "_reverse")]).amax(0).double()
    pre_shift = float((bn[0].double() * u * w_max).sum())
    fails = []
    print("[recurrent layer] output, worst per-hidden-unit error against float64", flush=True)
    _report(fails, "y", col_err(y, y64), float(col_err(y32, y64).max()), 1e-5,
            4 * pre_shift / y64.reshape(-1, H).abs().amax(0))
    assert not bad and not fails, (bad, fails)


# ---------------------------------------------------------------------------------------------------------------------
# 2. Lookahead (+ Hardtanh(0, 20))
# ---------------------------------------------------------------------------------------------------------------------
def lookahead_cuda(x, w, dy):
    T, B, H = x.shape
    ctx = w.shape[-1]
    y, dz, dx = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    dw = torch.empty(H, ctx, device=DEV)
    _call("ds2_lookahead_fwd", T, B, H, ctx, _p(x), _p(w), _p(y), _stream())
    _call("ds2_lookahead_bwd", T, B, H, ctx, _p(x), _p(w), _p(dy), _p(dz), _p(dx), _p(dw), _stream())
    torch.cuda.synchronize()
    return y, dz, dx, dw


def lookahead_ref(x, w, dy, dtype):
    """the reference module's arithmetic: F.pad + depthwise conv1d, then Hardtanh(0, 20); returns y, the
    pre-activation, dx, dw"""
    T, B, H = x.shape
    ctx = w.shape[-1]
    x, w = x.detach().to(dtype).requires_grad_(True), w.detach().to(dtype).reshape(H, 1, ctx).requires_grad_(True)
    with _no_tf32():
        z = F.conv1d(F.pad(x.permute(1, 2, 0), (0, ctx - 1)), w, groups=H).permute(2, 0, 1)
        y = F.hardtanh(z, 0.0, 20.0)
        y.backward(dy.to(dtype))
    return y.detach(), z.detach(), x.grad, w.grad.reshape(H, ctx)


LOOKAHEAD_CASES = [  # id, T', B, H, ctx
    ("T500_B32_H1024_ctx20", 500, 32, 1024, 20),        # the streaming uni-GRU configuration of the benchmark suite
    ("T7_lt_ctx20", 7, 3, 64, 20),                      # every frame's window runs past the end
    ("H40", 50, 5, 40, 20),                             # H not a multiple of 32
]


@pytest.mark.parametrize("tag,T,B,H,ctx", LOOKAHEAD_CASES, ids=[c[0] for c in LOOKAHEAD_CASES])
def test_lookahead_vs_float64(tag, T, B, H, ctx):
    """y and dx per channel within 2x the ATen fp32 yardstick + 1e-6; dw (float atomics) in relative L2 within 2x
    the yardstick + 1e-5.  dy is zeroed where the float64 pre-activation lies within 1e-4 of a clip point, so that
    rounding does not decide the clip mask (the exact-edge test does that)."""
    g = torch.Generator().manual_seed(T + H)
    x = torch.randn(T, B, H, generator=g).to(DEV)
    w = ((torch.rand(H, ctx, generator=g) * 2 - 1) / ctx ** 0.5).to(DEV)
    dy = torch.randn(T, B, H, generator=g).to(DEV)
    z64 = lookahead_ref(x, w, dy, torch.float64)[1]
    dy[(z64.abs() < 1e-4) | ((z64 - 20.0).abs() < 1e-4)] = 0.0
    y, _, dx, dw = lookahead_cuda(x, w, dy)
    ref = lookahead_ref(x, w, dy, torch.float64)
    yard = lookahead_ref(x, w, dy, torch.float32)
    fails = []
    print(f"\n[lookahead] {tag}: worst per-channel error against float64 (dw: rel-L2)", flush=True)
    _report(fails, "y", float(col_err(y, ref[0]).max()), float(col_err(yard[0], ref[0]).max()), 1e-6)
    _report(fails, "dx", float(col_err(dx, ref[2]).max()), float(col_err(yard[2], ref[2]).max()), 1e-6)
    _report(fails, "dw", rel_l2(dw, ref[3]), rel_l2(yard[3], ref[3]), 1e-5)
    assert not fails, fails


def test_lookahead_pre_activations_exactly_on_the_clip_points():
    """small integers everywhere, so every sum is exact in fp32: pre-activations land exactly on 0 and on 20, where
    torch's hardtanh_backward passes no gradient (strict inequalities).  y, dz, dx and dw must equal float64 exactly."""
    T, B, H, ctx = 64, 4, 40, 5
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 6, (T, B, H), generator=g).float().to(DEV)
    w = torch.randint(-1, 3, (H, ctx), generator=g).float().to(DEV)
    dy = torch.randint(-3, 4, (T, B, H), generator=g).float().to(DEV)
    y, dz, dx, dw = lookahead_cuda(x, w, dy)
    y64, z64, dx64, dw64 = lookahead_ref(x, w, dy, torch.float64)
    n0, n20 = int((z64 == 0).sum()), int((z64 == 20).sum())
    assert n0 > 20 and n20 > 20, (n0, n20)                  # the data does reach both clip points
    assert torch.equal(dz.double(), torch.where((z64 > 0) & (z64 < 20), dy.double(), torch.zeros_like(z64)))
    assert torch.equal(y.double(), y64)
    assert torch.equal(dx.double(), dx64)
    assert torch.equal(dw.double(), dw64)


# ---------------------------------------------------------------------------------------------------------------------
# 3. CTC
# ---------------------------------------------------------------------------------------------------------------------
def ctc_cuda(logits, targets, in_len, tgt_len, blank):
    T, B, Cn = logits.shape
    lg = logits.to(DEV).contiguous()
    tg = targets.to(DEV, torch.int64).contiguous()
    il, tl = in_len.to(DEV, torch.int32), tgt_len.to(DEV, torch.int32)
    max_l = int(tgt_len.max())
    ws = torch.empty(ds.get_lib().ds2_ctc_workspace_bytes(T, B, Cn, max_l), dtype=torch.uint8, device=DEV)
    nll, grad = torch.empty(B, device=DEV), torch.empty_like(lg)
    _call("ds2_ctc_loss_fwd_bwd", T, B, Cn, _p(lg), _p(tg), _p(il), _p(tl), max_l, blank, _p(nll), _p(grad), _p(ws),
          ws.numel(), _stream())
    torch.cuda.synchronize()
    return nll.cpu(), grad.cpu()


def _labels(n, Cn, blank, g):
    """n labels drawn from the classes other than blank"""
    lab = torch.randint(0, Cn - 1, (n,), generator=g)
    return lab + (lab >= blank).long()


# an utterance of 20 labels with exactly 5 adjacent repeats needs 25 frames: given exactly that many
EXACT = [1, 1, 2, 3, 3, 4, 5, 5, 6, 7, 7, 8, 9, 9, 10, 11, 12, 13, 14, 15]

CTC_CASES = [  # id, C, blank, logit scale, [(T'_b, L_b or a fixed label list)], gradient bound
    # 2L+1 > 1024 (several states per thread) next to L = 511 (2L+1 = 1023, the last one-state case) in one launch
    ("long_T1750_L700", 29, 0, 2.0, [(1750, 700), (1750, 512), (1600, 511), (900, 40)], 5e-4),
    ("edges", 29, 0, 2.0, [(6, 0), (1, 0), (1, 1), (25, EXACT), (3, [2, 2, 3]), (6, 2)], 1e-4),
    ("blank_last", 29, 28, 2.0, [(200, 60), (150, 40), (90, 1)], 1e-4),
    ("blank5", 29, 5, 2.0, [(200, 60), (150, 40), (90, 1)], 1e-4),
    ("C40", 40, 0, 2.0, [(180, 50), (120, 30), (40, 3)], 1e-4),
    ("C40_blank_last", 40, 39, 2.0, [(180, 50), (120, 30), (40, 3)], 1e-4),
    ("peaked_x30", 29, 0, 30.0, [(300, 100), (250, 80), (120, 30)], 5e-4),
]


@pytest.mark.parametrize("tag,Cn,blank,scale,utts,grad_tol", CTC_CASES, ids=[c[0] for c in CTC_CASES])
def test_ctc_vs_float64(tag, Cn, blank, scale, utts, grad_tol):
    """per utterance: NLL within 1e-5 relative of the float64 lattice (`O.ctc_loss_and_grad`) and of float64
    `F.ctc_loss`; the gradient within 1e-4 absolute (two cases: 5e-4, below); gradient rows t >= T'_b, and
    everything of an infeasible utterance (zero_infinity), exactly zero.

    The fp32 lattice accumulates rounding along the time axis, and the posterior exp(alpha + beta - ll) turns an
    absolute error of the log values into a relative one.  Long blank runs (T' = 900 with L = 40, T' = 1750) and
    x30 logits take the gradient error to 2-3e-4: a float32 replay of the same recursion on the same data, with
    correctly rounded exp / log, gives 2.3e-4 and 2.4e-4 on those two cases (the kernel on an H100: 3.0e-4 and
    2.4e-4), and rescaling every step instead of every 8 does not change that.  Those two cases are held to 5e-4;
    ATen's own fp32 CTC, which does not rescale at all, is printed beside them."""
    g = torch.Generator().manual_seed(len(tag) * 1000 + Cn)
    in_len = torch.tensor([u[0] for u in utts], dtype=torch.int32)
    tgts = [torch.tensor(u[1], dtype=torch.int64) if isinstance(u[1], list) else _labels(u[1], Cn, blank, g)
            for u in utts]
    tgt_len = torch.tensor([len(t) for t in tgts], dtype=torch.int32)
    targets = torch.cat(tgts)
    T, B = int(in_len.max()), len(utts)
    logits = torch.randn(T, B, Cn, generator=g) * scale
    nll, grad = ctc_cuda(logits, targets, in_len, tgt_len, blank)
    nll64, grad64 = O.ctc_loss_and_grad(logits.numpy(), targets.numpy(), in_len.numpy(), tgt_len.numpy(), blank=blank)
    aten = F.ctc_loss(logits.double().log_softmax(-1), targets, in_len.long(), tgt_len.long(), blank=blank,
                      reduction="none", zero_infinity=True)
    print(f"\n[ctc] {tag}: NLL {[round(float(v), 2) for v in nll64]}", flush=True)
    for b in range(B):
        ref = float(nll64[b])
        assert abs(ref - float(aten[b])) <= 1e-9 * max(1.0, abs(ref)), (b, ref, float(aten[b]))
        assert abs(float(nll[b]) - ref) <= 1e-5 * max(1.0, abs(ref)), (b, float(nll[b]), ref)
        assert abs(float(nll[b]) - float(aten[b])) <= 1e-5 * max(1.0, abs(float(aten[b]))), b
        Tb = int(in_len[b])
        if Tb < T:
            assert float(grad[Tb:, b].abs().max()) == 0.0, b
        if ref == 0.0 and int(tgt_len[b]) > 0:                      # infeasible: zero_infinity
            assert float(nll[b]) == 0.0 and float(grad[:, b].abs().max()) == 0.0, b
    err = float((grad.double() - torch.from_numpy(grad64)).abs().max())
    lg = logits.to(DEV).requires_grad_(True)
    F.ctc_loss(lg.log_softmax(-1), targets.to(DEV), in_len.long(), tgt_len.long(), blank=blank, reduction="sum",
               zero_infinity=True).backward()
    yard = float((lg.grad.double().cpu() - torch.from_numpy(grad64)).abs().max())
    nll_err = max(abs(float(nll[b]) - float(nll64[b])) / max(1.0, abs(float(nll64[b]))) for b in range(B))
    print(f"  NLL rel. error {nll_err:.1e}; grad max abs error {err:.2e} (bound {grad_tol:.0e}; ATen fp32 {yard:.2e})",
          flush=True)
    assert err < grad_tol


def test_ctc_edge_case_preconditions():
    """the edge utterances are what they claim to be: the exact-length one is feasible with no frame to spare, the
    short repeated one is infeasible (so its zero loss comes from zero_infinity)"""
    lp = np.zeros((25, 1, 29))
    nll, _ = O.ctc_loss_and_grad(lp, np.array(EXACT), np.array([25]), np.array([20]))
    assert np.isfinite(nll[0]) and nll[0] > 0
    nll, _ = O.ctc_loss_and_grad(lp[:24], np.array(EXACT), np.array([24]), np.array([20]), zero_infinity=False)
    assert nll[0] == np.inf
    nll, _ = O.ctc_loss_and_grad(lp[:3], np.array([2, 2, 3]), np.array([3]), np.array([3]), zero_infinity=False)
    assert nll[0] == np.inf


# ---------------------------------------------------------------------------------------------------------------------
# 4. Greedy decode
# ---------------------------------------------------------------------------------------------------------------------
def tie_free_probs(B, T, Cn, blank, seed):
    """softmax rows whose argmax follows runs of repeated labels and blanks (so the collapse has work to do), with a
    margin that rules out ties"""
    rng = np.random.default_rng(seed)
    lab = np.empty((B, T), np.int64)
    for b in range(B):
        t = 0
        while t < T:
            c = blank if rng.random() < 0.3 else int(rng.integers(0, Cn))
            n = int(rng.integers(1, 5))
            lab[b, t:t + n] = c
            t += n
    noise = torch.from_numpy(rng.standard_normal((B, T, Cn))).float() * 0.5
    probs = torch.softmax(noise + 6.0 * F.one_hot(torch.from_numpy(lab), Cn).float(), -1)
    top2 = probs.topk(2, -1).values
    assert bool((top2[..., 0] > top2[..., 1]).all())
    return probs


GREEDY_CASES = [  # id, B, T, C, blank, sizes
    ("T20000", 3, 20000, 29, 0, [20000, 13001, 0]),      # 80 KB of dynamic shared memory (opt-in); out_len = 0
    ("blank_last", 4, 300, 29, 28, [300, 255, 1, 0]),
    ("blank5_no_sizes", 2, 200, 40, 5, None),
]


@pytest.mark.parametrize("tag,B,T,Cn,blank,sizes", GREEDY_CASES, ids=[c[0] for c in GREEDY_CASES])
def test_greedy_decode_bit_exact(tag, B, T, Cn, blank, sizes):
    """labels, frame offsets and counts equal `O.greedy_path` exactly"""
    probs = tie_free_probs(B, T, Cn, blank, seed=T + blank)
    dec = ds.GreedyDecoder(ds.LABELS, blank_index=blank)
    labels, offsets, counts = dec.decode_indices(probs.to(DEV), None if sizes is None else torch.tensor(sizes))
    ref = O.greedy_path(probs, sizes, blank=blank)
    assert sum(len(r[0]) for r in ref) > 0
    for b, (lab, offs) in enumerate(ref):
        n = int(counts[b])
        assert n == len(lab), (b, n, len(lab))
        assert labels[b, :n].tolist() == lab, b
        assert offsets[b, :n].tolist() == offs, b
