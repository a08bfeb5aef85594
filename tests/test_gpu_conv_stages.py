"""The conv front-end one stage at a time against float64 (tests/conv_stage_reference.py), every stage fed with the
kernels' own input to it, at the shapes where its kernels have edges: 54-output time tiles with a 10-position halo,
32-step K chunks of the weight gradients, T' below one 32-step box, T' % 4 (tensor-core or FFMA weight gradients),
ragged lengths at tile edges, batches that leave weight-gradient slices empty, input that is not zero beyond the
lengths, eval mode, precision modes, the side-stream conv2 weight gradient, and BatchNorm2d channels with a large
offset.

Bounds follow from the arithmetic of each stage (see the reference module's metric functions); the worst figure
measured on an H100 80GB HBM3 is given with each check."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import conv_stage_reference as R
import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200._lib import check, get_lib, ptr

pytestmark = pytest.mark.gpu

MOM, EPS = 0.1, 1e-5
U = R.U32


# ---- running the kernels ---------------------------------------------------------------------------------------------
def _params(seed, w2_nonneg=False):
    g = torch.Generator().manual_seed(seed)

    def rn(*s):
        return torch.randn(*s, generator=g)

    P = dict(w1=rn(32, 1, 41, 11) * 0.05, b1=rn(32) * 0.1, g1=1 + 0.2 * rn(32), be1=0.5 + 0.2 * rn(32),
             rm1=0.1 * rn(32), rv1=1 + 0.1 * rn(32).abs(), w2=rn(32, 32, 21, 11) * 0.01, b2=rn(32) * 0.1,
             g2=1 + 0.2 * rn(32), be2=0.5 + 0.2 * rn(32), rm2=0.1 * rn(32), rv2=1 + 0.1 * rn(32).abs())
    if w2_nonneg:
        P["w2"] = P["w2"].abs()
    return {k: v.cuda() for k, v in P.items()}


def _inputs(B, T, out_len, seed, pad_noise=False):
    """x (B, 1, 161, T): zero beyond 2 * out_len[b] input frames, or noise there with pad_noise"""
    g = torch.Generator().manual_seed(seed + 1000)
    x = torch.randn(B, 1, 161, T, generator=g)
    if not pad_noise:
        for b, l in enumerate(out_len):
            x[b, :, :, 2 * l:] = 0
    return x.cuda(), torch.tensor(out_len, dtype=torch.int32).cuda()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ws(B, T):
    return ds.ops.workspace(get_lib().ds2_conv_frontend_workspace_bytes(B, T), torch.device("cuda"))


def _fwd(x, out_len, P, training=True):
    """ds2_conv_frontend_fwd: y, z1, a1, z2, stats (mean1, invstd1, mean2, invstd2) and the running statistics after"""
    lib = get_lib()
    B, _, _, T = x.shape
    Tp = R.out_frames(T)
    o = dict(y=torch.empty(Tp, B, 1312, device="cuda"), z1=torch.empty(B, 32, 81, Tp, device="cuda"),
             a1=torch.empty(B, 32, 81, Tp, device="cuda"), z2=torch.empty(B, 32, 41, Tp, device="cuda"),
             stats=torch.empty(128, device="cuda"))
    run = {k: P[k].clone() for k in ("rm1", "rv1", "rm2", "rv2")}
    ws = _ws(B, T)
    check(lib.ds2_conv_frontend_fwd(B, T, ptr(x), ptr(out_len), ptr(P["w1"]), ptr(P["b1"]), ptr(P["g1"]),
                                    ptr(P["be1"]), ptr(run["rm1"]), ptr(run["rv1"]), ptr(P["w2"]), ptr(P["b2"]),
                                    ptr(P["g2"]), ptr(P["be2"]), ptr(run["rm2"]), ptr(run["rv2"]), int(training), MOM,
                                    EPS, ptr(o["y"]), ptr(o["z1"]), ptr(o["a1"]), ptr(o["z2"]), ptr(o["stats"]),
                                    ptr(ws), ws.numel(), _stream()), "ds2_conv_frontend_fwd")
    o.update(run)
    return o


GRADS = ("dw1", "db1", "dg1", "dbe1", "dw2", "db2", "dg2", "dbe2")


def _bwd(x, out_len, P, f, dy):
    lib = get_lib()
    B, _, _, T = x.shape
    shapes = dict(dw1=P["w1"], dw2=P["w2"])
    o = {k: torch.empty_like(shapes.get(k, P["b1"])) for k in GRADS}
    ws = _ws(B, T)
    check(lib.ds2_conv_frontend_bwd(B, T, ptr(x), ptr(out_len), ptr(P["w1"]), ptr(P["g1"]), ptr(P["be1"]),
                                    ptr(P["w2"]), ptr(P["g2"]), ptr(P["be2"]), ptr(f["z1"]), ptr(f["a1"]),
                                    ptr(f["z2"]), ptr(f["stats"]), ptr(dy), *[ptr(o[k]) for k in GRADS], ptr(ws),
                                    ws.numel(), _stream()), "ds2_conv_frontend_bwd")
    return o


def _dy(f, P, out_len, seed):
    """seeded output gradient, zero where BN2 + Hardtanh's u lies within rounding of a clip point"""
    st = f["stats"]
    amb = R.ambiguous(f["z2"], st[64:96], st[96:128], P["g2"], P["be2"])
    dy = torch.randn(f["y"].shape, generator=torch.Generator().manual_seed(seed)).cuda()
    return dy * (~R.time_major(amb)).float()


# ---- the checks ------------------------------------------------------------------------------------------------------
def _stats_check(z, mean_k, invstd_k, rm_k, rv_k, rm0, rv0):
    """per channel against float64 of the kernel's own z, with fp32 ATen batch_norm on the same z as the yardstick:
    the kernel may be off by 4x ATen's worst channel, or by the rounding of its own float32 results (the mean
    rounded to float: U32 of |mean|; invstd through rsqrtf, 2 ulp, and the variance rounded to float; the running
    statistics' three float operations).  Errors: mean relative to the channel's std, the rest relative."""
    ref = R.bn_stats(z, rm0, rv0, MOM, EPS)
    _, am, ainv = torch.ops.aten.native_batch_norm(z, None, None, None, None, True, MOM, EPS)
    arm, arv = rm0.clone(), rv0.clone()
    F.batch_norm(z, arm, arv, None, None, True, MOM, EPS)
    sd = 1.0 / ref["invstd"]

    def errs(m, inv, rm, rv):
        return dict(mean=(m.double() - ref["mean"]).abs() / sd, invstd=(inv.double() / ref["invstd"] - 1).abs(),
                    rmean=(rm.double() - ref["rmean"]).abs() / (MOM * sd), rvar=(rv.double() / ref["rvar"] - 1).abs())

    ek, ea = errs(mean_k, invstd_k, rm_k, rv_k), errs(am, ainv, arm, arv)
    floor = dict(mean=2 * U * (ref["mean"].abs() / sd + 1), invstd=torch.full_like(sd, 8 * U),
                 rmean=4 * U * (ref["rmean"].abs() / (MOM * sd) + 1), rvar=torch.full_like(sd, 6 * U))
    worst = {}
    for k in ek:
        bound = torch.maximum(4 * ea[k].max(), floor[k])
        worst[k] = (float(ek[k].max()), float(ea[k].max()))
        assert bool((ek[k] <= bound).all()), (k, ek[k].tolist(), bound.tolist())
    return worst


def _forward_checks(x, out_len, P, f, tf32, training=True):
    """each forward stage from the kernel's own input; returns the worst ratios (error / bound)"""
    st = f["stats"]
    r = {}
    z1, mag = R.conv1(x, P["w1"], P["b1"], out_len)
    r["z1"] = R.elementwise_ratio(f["z1"], z1, mag, R.z1_c())
    a1, mag = R.bn_act(f["z1"], st[0:32], st[32:64], P["g1"], P["be1"], out_len)
    r["a1"] = R.elementwise_ratio(f["a1"], a1, mag, R.bn_act_c())
    z2, mag = R.conv2(f["a1"], P["w2"], P["b2"], out_len)
    r["z2"] = R.elementwise_ratio(f["z2"], z2, mag, R.z2_c(tf32))
    a2, mag = R.bn_act(f["z2"], st[64:96], st[96:128], P["g2"], P["be2"], out_len)
    r["y"] = R.elementwise_ratio(f["y"], R.time_major(a2), R.time_major(mag), R.bn_act_c())
    for k, v in r.items():
        assert v <= 1.0, (k, r)
    if training:
        r["stats1"] = _stats_check(f["z1"], st[0:32], st[32:64], f["rm1"], f["rv1"], P["rm1"], P["rv1"])
        r["stats2"] = _stats_check(f["z2"], st[64:96], st[96:128], f["rm2"], f["rv2"], P["rm2"], P["rv2"])
    else:
        # eval mode: the running statistics as given, invstd = rsqrtf(var + eps) within 2 ulp + the rounding of the add
        for i, (rm, rv) in enumerate(((P["rm1"], P["rv1"]), (P["rm2"], P["rv2"]))):
            assert torch.equal(st[64 * i:64 * i + 32], rm)
            inv = 1.0 / torch.sqrt(rv.double() + EPS)
            assert float((st[64 * i + 32:64 * i + 64].double() / inv - 1).abs().max()) <= 6 * U
            assert torch.equal(f[f"rm{i + 1}"], rm) and torch.equal(f[f"rv{i + 1}"], rv)
    return r


def _backward_checks(x, out_len, P, f, g, dy, tc_wgrad, tf32):
    """the backward from the kernel's saved z1, a1, z2 and stats, with the clip masks decided on u computed as the
    kernels compute it; returns the worst ratios (error / bound) and stage 1's rel_l2 figures"""
    st = f["stats"]
    B, _, _, Tp = f["z2"].shape
    r = {}
    u2 = R.u_kernel(f["z2"], st[64:96], st[96:128], P["g2"], P["be2"])
    s2 = R.bn_act_backward(f["z2"], st[64:96], st[96:128], P["g2"], R.clip_mask(u2, out_len),
                           R.batch_major(dy, R.D2), out_len)
    # stage 2 sums: one product (dgamma) and at most 12 fp32 adds (warp trees over 32 time lanes and over the rows
    # of a channel, at most 2 partial sums a thread) before the double atomics: 12 U32 of the sum of |terms|, +2 U32
    # for zh = (z - mean) * invstd
    r["dbe2"] = float(((g["dbe2"].double() - s2["dbeta"]).abs() / (12 * U * s2["s_du"]).clamp_min(1e-300)).max())
    r["dg2"] = float(((g["dg2"].double() - s2["dgamma"]).abs() / (14 * U * s2["s_duzh"]).clamp_min(1e-300)).max())
    # conv bias gradients (about 0): each dz within 8 U32 of dz_mag, then at most 32 fp32 adds (warp tree, 8 warps
    # in sequence, the ordered sum's strided per-thread sums and tree): 40 U32 of sum dz_mag
    r["db2"] = float(((g["db2"].double() - s2["dbias"]).abs()
                      / (40 * U * s2["dz_mag"].sum((0, 2, 3))).clamp_min(1e-300)).max())
    dw2 = R.conv2_wgrad(s2["dz"], f["a1"])
    r["dw2"] = R.wgrad_ratio(g["dw2"], dw2, s2["dz"], s2["dz_mag"], f["a1"], R.conv2_wgrad, B * R.D2 * Tp,
                             tc_wgrad)
    # stage 1: the clip masks from the kernel's own z1 and stats, ambiguous positions counted (they get the kernel's
    # data gradient either way and stay out of no check but are rare: u within 8 U32 of 0 or 20)
    amb1 = R.ambiguous(f["z1"], st[0:32], st[32:64], P["g1"], P["be1"]) & (R.keep(out_len, Tp, "cuda") > 0)
    assert int(amb1.sum()) <= max(2, amb1.numel() // 100000), int(amb1.sum())
    u1 = R.u_kernel(f["z1"], st[0:32], st[32:64], P["g1"], P["be1"])
    da1 = R.conv2_dgrad(s2["dz"], P["w2"])
    s1 = R.bn_act_backward(f["z1"], st[0:32], st[32:64], P["g1"], R.clip_mask(u1, out_len), da1, out_len)
    dw1 = R.conv1_wgrad(s1["dz"], x)
    # d(a1) comes from a TF32 GEMM (dz2 and w2 rounded) and dw1 from another (dz1 and x rounded): every term of a
    # stage-1 gradient carries four TF32 operand roundings, at most 4 UTF32 ~ 2e-3 relative together; the rounding
    # errors of different terms are independent and partly cancel, so rel_l2 stays below 2e-3.  In fp32 mode the
    # same sums run on FFMA, off by at most K U32 relative per term, K = 3872 products per d(a1) entry: 2.3e-4
    lim = 4 * R.UTF32 if tf32 else 3872 * U
    for k, ref in (("dw1", dw1), ("dg1", s1["dgamma"]), ("dbe1", s1["dbeta"])):
        r[k] = R.rel_l2(g[k], ref) / lim
    # db1 = k (dbeta (1 - Nv/N) - dgamma sum_valid(zh) / N) with Nv the valid count: d(a1)'s error (the same 4 UTF32
    # relative per term as above) reaches it only through those two factors; plus the fp32 rounding as for db2
    nv = R.keep(out_len, Tp, "cuda").sum() * R.D1
    zs = (s1["zh"] * R.keep(out_len, Tp, "cuda")).sum((0, 2, 3))
    lim_db1 = (40 * U * s1["dz_mag"].sum((0, 2, 3)) + lim * s1["k"].abs().flatten()
               * (s1["s_du"] * (1 - nv / s1["n"]) + s1["s_duzh"] * zs.abs() / s1["n"]))
    r["db1"] = float(((g["db1"].double() - s1["dbias"]).abs() / lim_db1.clamp_min(1e-300)).max())
    for k, v in r.items():
        assert v <= 1.0, (k, r)
    return r


def _run_case(T, B, out_len, prec="tf32", seed=0, pad_noise=False, training=True, P=None, backward=True):
    ds.set_precision(prec)
    try:
        P = P if P is not None else _params(seed)
        x, ol = _inputs(B, T, out_len, seed, pad_noise)
        f = _fwd(x, ol, P, training)
        tf32 = prec != "fp32"
        Tp = R.out_frames(T)
        r = _forward_checks(x, ol, P, f, tf32, training)
        if backward:
            dy = _dy(f, P, ol, seed + 7)
            g = _bwd(x, ol, P, f, dy)
            torch.cuda.synchronize()
            r.update(_backward_checks(x, ol, P, f, g, dy, tf32 and Tp % 4 == 0, tf32))
        print(f"T={T} B={B} {prec}: " + ", ".join(f"{k} {v}" for k, v in r.items()))
        return r
    finally:
        ds.set_precision("tf32")


# ---- cases -------------------------------------------------------------------------------------------------------------
def _ragged(Tp, B):
    return sorted([max(1, Tp - (Tp // (B + 1)) * i) for i in range(B)], reverse=True)


@pytest.mark.parametrize("ragged", [False, True])
def test_stages_benchmark_shape(ragged):
    """B = 32, T = 1000 (T' = 500): every stage at the benchmarked shape, full length and ragged.
    Worst measured (error / bound): z1 0.015, a1 0.61, z2 0.032, y 0.58, dbeta2 1.0e-3, dgamma2 9.3e-4, db2 5.2e-3,
    dw2 0.053, db1 3.7e-3; rel_l2 of dw1 4.2e-4, dgamma1 2.3e-4, dbeta1 4.3e-4 (bound 2e-3).  Statistics (kernel /
    ATen on the same z, worst channel): invstd 8.8e-8 / 1.2e-6, mean 7.1e-8 / 3.2e-7 of the std."""
    _run_case(1000, 32, _ragged(500, 32) if ragged else [500] * 32)


@pytest.mark.parametrize("T,B", [(1, 2), (2, 3), (7, 2), (8, 3)])
def test_stages_tiny(T, B):
    """T' = 1 (T = 1, 2) and T' = 4 (T = 7, 8): below one 32-step box of the weight gradients' TMA loads and one
    64-position tile; T' = 4 takes the tensor-core weight gradients.  Out lengths T' and 1.
    Worst measured (error / bound): z2 0.065, y 0.44, dbeta2 0.042, dgamma2 0.067, dw2 0.60 (T' = 4), db1 0.028;
    rel_l2 of dw1 4.3e-4."""
    Tp = R.out_frames(T)
    _run_case(T, B, [Tp] + [1] * (B - 1))


@pytest.mark.parametrize("Tp", [32, 36, 52, 54, 55, 56, 108])
def test_stages_tile_and_chunk_edges(Tp):
    """T' at the 32-step K-chunk edges (32, 36) and the 54-output tile edges (52, 54, 55, 56, 108), both parities
    of T (T = 2T' - 1 for odd T', 2T' for even), with lengths at the edges: one full-length utterance, out_len 54 and
    55, a fully masked last tile (out_len <= 54 at T' = 108) and out_len 1.  T' % 4 != 0 (55) takes the FFMA weight
    gradients.  Worst measured (error / bound): z2 0.052, y 0.61, dw2 0.59 (T' = 32; 6.1e-3 on FFMA at T' = 55),
    db1 5.0e-3; rel_l2 of dw1 4.1e-4, dbeta1 4.9e-4."""
    T = 2 * Tp - (Tp % 2)
    lens = [Tp, min(Tp, 54), min(Tp, 55), 1, max(1, Tp - 33)]
    _run_case(T, len(lens), lens, seed=Tp)


@pytest.mark.parametrize("B,Tp", [(1, 56), (3, 56), (33, 100)])
def test_stages_batch_sizes(B, Tp):
    """B = 1 and 3 leave slices of the weight gradients' (12 for conv2, 24 for conv1) (b, row) pairs empty, whose
    tiles are stored as zeros; B = 33 is one past the benchmark.  Worst measured (error / bound): dw2 0.65 (B = 1),
    0.54 (B = 3), 0.15 (B = 33); z2 0.031; rel_l2 of dw1 4.1e-4."""
    _run_case(2 * Tp, B, _ragged(Tp, B), seed=B)


def test_stages_nonzero_padding():
    """x holds noise beyond each length: conv1's last valid outputs and the conv1 weight gradient read it, as the
    reference does.  Worst measured (error / bound): z1 0.014, z2 0.038, dw2 0.53; rel_l2 of dw1 4.1e-4."""
    _run_case(216, 4, [108, 80, 54, 3], pad_noise=True, seed=5)


def test_stages_eval_mode():
    """training = False: the running statistics normalise, on the tensor-core conv2.  Worst measured (error / bound):
    z2 0.032, y 0.55."""
    _run_case(400, 6, _ragged(200, 6), training=False, backward=False, seed=6)


@pytest.mark.parametrize("T,B", [(216, 4), (111, 3)])
def test_stages_fp32_mode(T, B):
    """fp32 mode: every convolution on FFMA, bounds at fp32 level.  Worst measured (error / bound): z2 7.9e-4, dw2
    8.7e-3, dbeta1 8.9e-3 (rel_l2 2.0e-6 against 2.3e-4), dw1 5.1e-3."""
    _run_case(T, B, _ragged(R.out_frames(T), B), prec="fp32", seed=T)


def test_fp16_frontend_equals_tf32_bitwise():
    """precision-16 runs the front-end as in tf32 mode: outputs and gradients bit-identical"""
    out = {}
    for prec in ("tf32", "fp16"):
        ds.set_precision(prec)
        try:
            P = _params(11)
            x, ol = _inputs(5, 216, _ragged(108, 5), 11)
            f = _fwd(x, ol, P)
            g = _bwd(x, ol, P, f, _dy(f, P, ol, 12))
            torch.cuda.synchronize()
            out[prec] = (f, g)
        finally:
            ds.set_precision("tf32")
    for k in ("y", "z1", "a1", "z2", "stats", "rm1", "rv1", "rm2", "rv2"):
        assert torch.equal(out["tf32"][0][k], out["fp16"][0][k]), k
    for k in GRADS:
        assert torch.equal(out["tf32"][1][k], out["fp16"][1][k]), k


def test_side_stream_weight_grad_equals_main_stream_bitwise():
    """with deferred weight gradients the conv2 weight gradient runs on the side stream (T' % 4 == 0) and hands its
    staging buffer to the conv1 weight gradient and to the next call: two back-to-back forward + backward calls on
    different inputs give the same bits as without a side stream"""
    ds.set_precision("tf32")
    P = _params(21)
    cases = [_inputs(8, 400, _ragged(200, 8), s) for s in (22, 23)]

    def run():
        res = []
        for x, ol in cases:
            f = _fwd(x, ol, P)
            res.append((f, _bwd(x, ol, P, f, _dy(f, P, ol, 24))))
        ds.ops.join_deferred()
        torch.cuda.synchronize()
        return res

    base = run()
    ds.ops.enable_deferred_weight_grads()
    try:
        side = run()
    finally:
        ds.ops.enable_deferred_weight_grads(enable=False)
    for (f0, g0), (f1, g1) in zip(base, side):
        for k in ("y", "z1", "a1", "z2", "stats"):
            assert torch.equal(f0[k], f1[k]), k
        for k in GRADS:
            assert torch.equal(g0[k], g1[k]), k


def test_conv2_tf32_rounds_to_nearest_on_same_sign_data():
    """w2 >= 0 and a1 >= 0: all of conv2's products have one sign, so a truncating TF32 conversion would show as a
    bias of about -7e-4 in the mean signed relative error of z2 (conv part); rounding to nearest gives about 0.
    Bound 1e-4.  Measured: -2.1e-6."""
    ds.set_precision("tf32")
    P = _params(31, w2_nonneg=True)
    x, ol = _inputs(4, 400, [200, 180, 150, 120], 31)
    f = _fwd(x, ol, P)
    z2, _ = R.conv2(f["a1"], P["w2"], P["b2"], ol)
    bias = R.same_sign_bias(f["z2"], z2, P["b2"], ol)
    print(f"same-sign mean signed relative error {bias:.3e}")
    assert abs(bias) <= 1e-4, bias


@pytest.mark.parametrize("B,T,offset", [(1, 16, 30.0), (1, 16, 300.0), (2, 110, 300.0), (32, 1000, 300.0)])
def test_bn2d_statistics_with_large_channel_offsets(B, T, offset):
    """channels 0 and 1 of both convolutions get a bias of offset x and offset / 10 x the std of their output,
    so their mean is large against their spread; every channel's mean, invstd and running statistics must stay
    within 4x the error of fp32 ATen batch_norm on the same z.  Few statistics partials at B = 1, short T'; many at
    the benchmark shape.  Before the bias pivot (raw sums only) the 300x channel's invstd was 5.0e-5 off at B = 1,
    T = 16, against a bound of 1.4e-6: every case here failed.  Worst measured with it (kernel / ATen): invstd 9.8e-8 /
    6.7e-7, running var 1.2e-7 / 1.2e-7, mean 1.1e-5 / 3.9e-5 of the std (the float rounding of a mean 300 std
    large)."""
    ds.set_precision("tf32")
    P = _params(41)
    Tp = R.out_frames(T)
    lens = [Tp] * B
    x, ol = _inputs(B, T, lens, 41)
    # the std of each conv's output without its bias, from a first forward
    f = _fwd(x, ol, P)
    sd1 = (f["z1"] - P["b1"][None, :, None, None]).double().std((0, 2, 3))
    P["b1"][0] = offset * sd1[0]
    P["b1"][1] = offset / 10 * sd1[1]
    f = _fwd(x, ol, P)
    sd2 = (f["z2"] - P["b2"][None, :, None, None]).double().std((0, 2, 3))
    P["b2"][0] = offset * sd2[0]
    P["b2"][1] = offset / 10 * sd2[1]
    r = _run_case(T, B, lens, seed=41, P=P, backward=False)
    print(f"offset {offset} B={B} T={T}: {r['stats1']} {r['stats2']}")
