"""The float64 stage references of the conv front-end (tests/conv_stage_reference.py) without a GPU: chained together
they equal float64 autograd through the oracle's conv front-end, and the GPU tests' metrics, fed with planted defects
of the kinds a kernel change can make, exceed their bounds by at least 3x at the GPU tests' edge shapes."""
import pytest
import torch

import conv_stage_reference as R
from oracle import ds2_oracle as O

MOM, EPS = 0.1, 1e-5


def _setup(B, T, lens, seed=0):
    g = torch.Generator().manual_seed(seed)

    def rn(*s):
        return torch.randn(*s, generator=g, dtype=torch.float64)

    P = dict(w1=rn(32, 1, 41, 11) * 0.05, b1=rn(32) * 0.1, g1=1 + 0.2 * rn(32), be1=0.5 + 0.2 * rn(32),
             rm1=0.1 * rn(32), rv1=1 + 0.1 * rn(32).abs(), w2=rn(32, 32, 21, 11) * 0.01, b2=rn(32) * 0.1,
             g2=1 + 0.2 * rn(32), be2=0.5 + 0.2 * rn(32), rm2=0.1 * rn(32), rv2=1 + 0.1 * rn(32).abs())
    x = rn(B, 1, 161, T)
    for b, l in enumerate(lens):
        x[b, :, :, 2 * l:] = 0
    ol = torch.tensor(lens, dtype=torch.int32)
    f = R.frontend_forward(x, ol, P, MOM, EPS)
    dy = rn(*f["y"].shape)
    return P, x, ol, f, dy


def test_stage_references_equal_float64_autograd_through_the_oracle():
    P, x, ol, f, dy = _setup(2, 60, [30, 17])
    names = {"0.weight": "w1", "0.bias": "b1", "1.weight": "g1", "1.bias": "be1", "1.running_mean": "rm1",
             "1.running_var": "rv1", "3.weight": "w2", "3.bias": "b2", "4.weight": "g2", "4.bias": "be2",
             "4.running_mean": "rm2", "4.running_var": "rv2"}
    OP = {"conv.seq_module." + k: P[v].clone() for k, v in names.items()}
    leaves = ["0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias", "4.weight", "4.bias"]
    for k in leaves:
        OP["conv.seq_module." + k].requires_grad_(True)
    nb = {}
    z = O.conv_frontend(x, ol, OP, True, nb)
    y = R.time_major(z)
    assert float((y.detach() - f["y"]).abs().max()) < 1e-12
    for k, s in (("1.", "s1"), ("4.", "s2")):
        assert torch.allclose(nb["conv.seq_module." + k + "running_mean"], f[s]["rmean"], rtol=0, atol=1e-12)
        assert torch.allclose(nb["conv.seq_module." + k + "running_var"], f[s]["rvar"], rtol=1e-12, atol=0)
    # no activation near a clip point, so the masks agree whichever way they are decided
    for zk, s, gk, bk in (("z1", "s1", "g1", "be1"), ("z2", "s2", "g2", "be2")):
        u = (f[zk] - f[s]["mean"][None, :, None, None]) * f[s]["invstd"][None, :, None, None] \
            * P[gk][None, :, None, None] + P[bk][None, :, None, None]
        assert float(torch.minimum(u.abs(), (u - 20).abs()).min()) > 1e-9
    (y * dy).sum().backward()
    b = R.frontend_backward(x, ol, P, f["z1"], f["a1"], f["z2"], f["s1"], f["s2"], dy)
    for k, ours in zip(leaves, ("dw1", "db1", "dg1", "dbe1", "dw2", "db2", "dg2", "dbe2")):
        ref = OP["conv.seq_module." + k].grad
        assert float((b[ours] - ref).abs().max()) <= 1e-10 * max(1.0, float(ref.abs().max())), k


# ---- planted defects: each must push the GPU test's metric to at least 3x its bound -----------------------------------
def _stage2(P, x, ol, f, dy):
    s2 = R.bn_act_backward(f["z2"], f["s2"]["mean"], f["s2"]["invstd"], P["g2"],
                           R.clip_mask((f["z2"] - f["s2"]["mean"][None, :, None, None])
                                       * f["s2"]["invstd"][None, :, None, None] * P["g2"][None, :, None, None]
                                       + P["be2"][None, :, None, None], ol), R.batch_major(dy, R.D2), ol)
    return s2


def _dw2_ratio(P, f, s2, dw2_got, B, Tp):
    dw2 = R.conv2_wgrad(s2["dz"], f["a1"])
    return R.wgrad_ratio(dw2_got, dw2, s2["dz"], s2["dz_mag"], f["a1"], R.conv2_wgrad, B * R.D2 * Tp, True)


@pytest.mark.parametrize("B,Tp,lens", [(1, 56, [56]), (3, 56, [56, 54, 1]), (4, 108, [108, 55, 54, 1])])
def test_dropped_last_frame_of_dz2_fails_the_dw2_check(B, Tp, lens):
    P, x, ol, f, dy = _setup(B, 2 * Tp, lens, seed=Tp + B)
    s2 = _stage2(P, x, ol, f, dy)
    assert _dw2_ratio(P, f, s2, R.conv2_wgrad(s2["dz"], f["a1"]), B, Tp) < 1e-3   # the float64 value passes
    b = max(range(B), key=lambda i: lens[i] > 1)   # an utterance longer than one frame
    dz = s2["dz"].clone()
    dz[b, :, :, lens[b] - 1] = 0
    assert _dw2_ratio(P, f, s2, R.conv2_wgrad(dz, f["a1"]), B, Tp) >= 3


@pytest.mark.parametrize("B,Tp", [(1, 64), (3, 64)])
def test_missing_k_chunk_of_one_row_fails_the_dw2_check(B, Tp):
    """one 32-step K chunk (output time 32..63) of one (b, input row r) pair left out of dw2"""
    P, x, ol, f, dy = _setup(B, 2 * Tp, [Tp] * B, seed=B)
    s2 = _stage2(P, x, ol, f, dy)
    dz_chunk = torch.zeros_like(s2["dz"])
    dz_chunk[B - 1, :, :, 32:64] = s2["dz"][B - 1, :, :, 32:64]
    a_row = torch.zeros_like(f["a1"])
    a_row[B - 1, :, 40] = f["a1"][B - 1, :, 40]
    dw2 = R.conv2_wgrad(s2["dz"], f["a1"]) - R.conv2_wgrad(dz_chunk, a_row)
    assert _dw2_ratio(P, f, s2, dw2, B, Tp) >= 3


@pytest.mark.parametrize("B,Tp,lens", [(3, 4, [4, 1, 2]), (4, 108, [108, 55, 54, 1])])
def test_stage1_mask_off_by_one_fails_the_z1_check(B, Tp, lens):
    P, x, ol, f, dy = _setup(B, 2 * Tp, lens, seed=Tp)
    z1, mag = R.conv1(x, P["w1"], P["b1"], ol)
    assert R.elementwise_ratio(z1.float(), z1, mag, R.z1_c()) <= 1
    bad, _ = R.conv1(x, P["w1"], P["b1"], ol + 1)      # t <= len kept
    bad = bad[..., :Tp]
    assert R.elementwise_ratio(bad, z1, mag, R.z1_c()) >= 3


@pytest.mark.parametrize("B,Tp", [(1, 56), (3, 56)])
def test_missing_last_conv2_row_fails_the_z2_check(B, Tp):
    P, x, ol, f, dy = _setup(B, 2 * Tp, [Tp] * B)
    a1 = f["a1"].float()
    z2, mag = R.conv2(a1, P["w2"], P["b2"], ol)
    got = R.conv2(R.round_tf32(a1), R.round_tf32(P["w2"]), P["b2"], ol)[0]
    assert R.elementwise_ratio(got, z2, mag, R.z2_c(True)) <= 1     # TF32 operands pass
    got[:, :, 40] = P["b2"][None, :, None]
    assert R.elementwise_ratio(got, z2, mag, R.z2_c(True)) >= 3


def _stage1_ratios(P, x, ol, f, s2, da1):
    """the GPU test's stage-1 metrics (rel_l2 / 4 UTF32) of dw1, dgamma1, dbeta1 from a given d(a1)"""
    s1, u1 = f["s1"], None
    u1 = (f["z1"] - s1["mean"][None, :, None, None]) * s1["invstd"][None, :, None, None] \
        * P["g1"][None, :, None, None] + P["be1"][None, :, None, None]
    m1 = R.clip_mask(u1, ol)
    ref = R.bn_act_backward(f["z1"], s1["mean"], s1["invstd"], P["g1"], m1, R.conv2_dgrad(s2["dz"], P["w2"]), ol)
    got = R.bn_act_backward(f["z1"], s1["mean"], s1["invstd"], P["g1"], m1, da1, ol)
    lim = 4 * R.UTF32
    return {k: R.rel_l2(a, b) / lim for k, a, b in (
        ("dw1", R.conv1_wgrad(got["dz"], x), R.conv1_wgrad(ref["dz"], x)), ("dg1", got["dgamma"], ref["dgamma"]),
        ("dbe1", got["dbeta"], ref["dbeta"]))}


@pytest.mark.parametrize("B,Tp,kw", [(1, 56, 0), (1, 108, 10), (3, 56, 5)])
def test_missing_tap_column_in_one_data_gradient_tile_fails_the_stage1_checks(B, Tp, kw):
    """one kw tap column left out of d(a1) in one 54-output tile (outputs 0..53 of the even rows of utterance 0)"""
    P, x, ol, f, dy = _setup(B, 2 * Tp, [Tp] * B, seed=kw)
    s2 = _stage2(P, x, ol, f, dy)
    da1 = R.conv2_dgrad(s2["dz"], P["w2"])
    w_bad = P["w2"].clone()
    w_bad[..., kw] = 0
    da1_bad = da1.clone()
    da1_bad[0, :, 0::2, :54] = R.conv2_dgrad(s2["dz"], w_bad)[0, :, 0::2, :54]
    assert max(_stage1_ratios(P, x, ol, f, s2, da1).values()) < 1e-6
    assert max(_stage1_ratios(P, x, ol, f, s2, da1_bad).values()) >= 3


@pytest.mark.parametrize("B,Tp", [(1, 56), (3, 108)])
def test_missing_first_odd_data_gradient_row_fails_the_stage1_checks(B, Tp):
    P, x, ol, f, dy = _setup(B, 2 * Tp, [Tp] * B, seed=B)
    s2 = _stage2(P, x, ol, f, dy)
    da1 = R.conv2_dgrad(s2["dz"], P["w2"])
    da1[:, :, 1] = 0
    assert max(_stage1_ratios(P, x, ol, f, s2, da1).values()) >= 3


def test_tf32_truncation_fails_the_same_sign_check():
    P, x, ol, f, dy = _setup(2, 200, [100, 80])
    w2 = P["w2"].abs()
    a1 = f["a1"].float()
    z2, _ = R.conv2(a1, w2, P["b2"], ol)
    near = R.conv2(R.round_tf32(a1), R.round_tf32(w2), P["b2"], ol)[0]
    trunc = R.conv2(R.round_tf32(a1, truncate=True), R.round_tf32(w2, truncate=True), P["b2"], ol)[0]
    assert abs(R.same_sign_bias(near, z2, P["b2"], ol)) <= 1e-4 / 3
    assert R.same_sign_bias(trunc, z2, P["b2"], ol) <= -3e-4
