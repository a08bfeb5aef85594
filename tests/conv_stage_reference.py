"""Float64 references of the conv front-end (model.py:157-164 under MaskConv, and its backward), one stage at a time.

Every stage takes the kernel's own input to that stage ("teacher forcing"), so the rounding of one stage never reaches
the check of the next, and a check can be as tight as the arithmetic of its own stage allows.  Besides each reference
value, a stage returns the magnitudes its error bound is made of: the absolute-value convolution |w| * |input| for a
sum of products (at most `u` relative per product and per add), and the sum of squared products for the bounds that
model rounding errors as independent and zero-mean (round to nearest).

Plain torch, device-agnostic (the GPU tests run it on the GPU in float64); no GPU needed to import it.
"""
import math

import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

D1, D2, NF, C = 81, 41, 161, 32
ST1, PD1 = (2, 2), (20, 5)          # conv1: 1 -> 32, 41 x 11 taps
ST2, PD2 = (2, 1), (10, 5)          # conv2: 32 -> 32, 21 x 11 taps
K1, K2 = 41 * 11, 32 * 21 * 11      # products per conv1 / conv2 output
U32 = 2.0 ** -24                    # unit roundoff of fp32
UTF32 = 2.0 ** -11                  # unit roundoff of a TF32 operand (10 stored mantissa bits, round to nearest)
# standard deviation of the relative error of a product of two TF32-rounded operands, each error uniform in
# [-UTF32, UTF32] (variance UTF32^2 / 3) and independent
SIG_TF32 = UTF32 * math.sqrt(2.0 / 3.0)
NSIG = 6.0                          # bounds built from standard deviations sit this many of them out


def out_frames(T):
    return (T - 1) // 2 + 1


def keep(out_len, Tp, device=None):
    """(B, 1, 1, Tp) float64: 1 where t < out_len[b]"""
    ol = torch.as_tensor(out_len).to(device=device, dtype=torch.int64)
    return (torch.arange(Tp, device=ol.device)[None, :] < ol[:, None]).double()[:, None, None, :]


# ---- forward -------------------------------------------------------------------------------------------------------
def conv1(x, w1, b1, out_len):
    """z1 = mask(conv1(x) + b1) and |w1| * |x| + |b1| (masked)"""
    x, w1, b1 = x.double(), w1.double(), b1.double()
    m = keep(out_len, out_frames(x.shape[-1]), x.device)
    z = F.conv2d(x, w1, b1, stride=ST1, padding=PD1) * m
    mag = F.conv2d(x.abs(), w1.abs(), b1.abs(), stride=ST1, padding=PD1) * m
    return z, mag


def conv2(a1, w2, b2, out_len):
    """z2 = mask(conv2(a1) + b2) and |w2| * |a1| + |b2| (masked)"""
    a1, w2, b2 = a1.double(), w2.double(), b2.double()
    m = keep(out_len, a1.shape[-1], a1.device)
    z = F.conv2d(a1, w2, b2, stride=ST2, padding=PD2) * m
    mag = F.conv2d(a1.abs(), w2.abs(), b2.abs(), stride=ST2, padding=PD2) * m
    return z, mag


def bn_stats(z, rmean, rvar, momentum, eps):
    """BatchNorm2d training statistics of z (B, C, D, T), masked zeros included (count B*D*T): mean, biased var,
    invstd = 1/sqrt(var + eps), and the running statistics after the update (unbiased var)"""
    z = z.double()
    n = z.numel() // z.shape[1]
    mean = z.mean((0, 2, 3))
    var = ((z - mean[None, :, None, None]) ** 2).mean((0, 2, 3))
    unb = var * n / (n - 1) if n > 1 else var
    rm = (1 - momentum) * rmean.double() + momentum * mean
    rv = (1 - momentum) * rvar.double() + momentum * unb
    return dict(mean=mean, var=var, invstd=1.0 / torch.sqrt(var + eps), rmean=rm, rvar=rv, n=n)


def _ch(v):
    return v.double()[None, :, None, None]


def bn_act(z, mean, invstd, g, be, out_len):
    """a = mask(clamp(g * (z - mean) * invstd + be, 0, 20)) in float64 from the given statistics, and the magnitude
    |z - mean| * invstd * |g| + |be| of its terms"""
    z = z.double()
    m = keep(out_len, z.shape[-1], z.device)
    zh = (z - _ch(mean)) * _ch(invstd)
    u = zh * _ch(g) + _ch(be)
    return torch.clamp(u, 0.0, 20.0) * m, (zh.abs() * _ch(g).abs() + _ch(be).abs() + _ch(mean).abs() * _ch(invstd)
                                          * _ch(g).abs()) * m


def u_kernel(z, mean, invstd, g, be):
    """u = fmaf((z - mean) * invstd, g, be) evaluated as the kernels do, in float32 (the product of two floats is exact
    in float64, so the fma's single rounding is the float64 sum's rounding to float32, up to a double rounding)"""
    z = z.float()
    zh = (z - mean.float()[None, :, None, None]) * invstd.float()[None, :, None, None]
    return (zh.double() * _ch(g.float()) + _ch(be.float())).float()


def ambiguous(z, mean, invstd, g, be):
    """positions where u lies within rounding of a clip point (0 or 20): there the kernel's and any emulation's
    Hardtanh decisions may differ"""
    z = z.float()
    zh = (z - mean.float()[None, :, None, None]) * invstd.float()[None, :, None, None]
    u = zh.double() * _ch(g.float()) + _ch(be.float())
    tol = 8 * U32 * (zh.double().abs() * _ch(g).abs() + _ch(be).abs() + (_ch(mean).abs() + z.double().abs())
                     * _ch(invstd).abs() * _ch(g).abs())
    return (u.abs() <= tol) | ((u - 20.0).abs() <= tol)


def time_major(a):
    """(B, C, D, T) -> (T, B, C*D), feature c*D + d"""
    B, Cc, D, T = a.shape
    return a.reshape(B, Cc * D, T).permute(2, 0, 1)


def batch_major(y, D):
    """(T, B, C*D) -> (B, C, D, T)"""
    T, B, CD = y.shape
    return y.permute(1, 2, 0).reshape(B, CD // D, D, T)


# ---- backward ------------------------------------------------------------------------------------------------------
def clip_mask(u, out_len):
    """1[t < len] * 1[0 < u < 20] in float64"""
    return keep(out_len, u.shape[-1], u.device) * ((u > 0) & (u < 20)).double()


def bn_act_backward(z, mean, invstd, g, mask, dout, out_len):
    """BatchNorm (batch statistics) + Hardtanh + mask backward with the clip mask given:
    du = dout * mask, dbeta = sum du, dgamma = sum du * zh, dz = 1[t<len] * g * invstd * (du - dbeta/N - zh dgamma/N),
    db (bias of the producing conv) = sum dz.  Also |k| (|du| + sum|du|/N + |zh| sum|du zh|/N), which bounds the
    magnitude of dz's terms and of the rounding of dbeta and dgamma as the kernel sums them."""
    z, dout = z.double(), dout.double()
    n = z.numel() // z.shape[1]
    zh = (z - _ch(mean)) * _ch(invstd)
    du = dout * mask
    dbe = du.sum((0, 2, 3))
    dg = (du * zh).sum((0, 2, 3))
    k = _ch(g) * _ch(invstd)
    m = keep(out_len, z.shape[-1], z.device)
    dz = m * k * (du - _ch(dbe) / n - zh * _ch(dg) / n)
    s_du, s_duzh = du.abs().sum((0, 2, 3)), (du * zh).abs().sum((0, 2, 3))
    mag = m * k.abs() * (du.abs() + _ch(s_du) / n + zh.abs() * _ch(s_duzh) / n)
    return dict(du=du, dz=dz, dz_mag=mag, zh=zh, k=k, dbeta=dbe, dgamma=dg, dbias=dz.sum((0, 2, 3)), n=n, s_du=s_du,
                s_duzh=s_duzh)


def conv2_wgrad(dz2, a1):
    """dw2 = sum_{b,d,t} dz2[b,co,d,t] a1[b,ci,2d+kh-10,t+kw-5]"""
    return conv2d_weight(a1.double(), (C, C, 21, 11), dz2.double(), stride=ST2, padding=PD2)


def conv2_dgrad(dz2, w2):
    """d(a1) = conv2's data gradient (B, 32, 81, T')"""
    B, _, _, Tp = dz2.shape
    return conv2d_input((B, C, D1, Tp), w2.double(), dz2.double(), stride=ST2, padding=PD2)


def conv1_wgrad(dz1, x):
    """dw1 = sum_{b,d,t} dz1[b,co,d,t] x[b,0,2d+kh-20,2t+kw-5]"""
    return conv2d_weight(x.double(), (C, 1, 41, 11), dz1.double(), stride=ST1, padding=PD1)


def tc_sum_sigma(s_sq, s_abs, k_terms, tf32=True):
    """standard deviation of the error of a sum of k_terms products on the tensor cores (both operands rounded to
    TF32 when tf32, fp32 accumulation): sqrt(sum of the products' variances + the adds' variances), the adds' error
    at most U32 of a partial sum no larger than s_abs, uniform"""
    a = SIG_TF32 * s_sq if tf32 else 0.0
    return torch.sqrt(a ** 2 + (U32 * s_abs) ** 2 * k_terms / 3.0)


def frontend_forward(x, out_len, P, momentum=0.1, eps=1e-5):
    """the whole forward in float64 without teacher forcing (used by the host tests): a dict with every stage's
    value, as the GPU stages are checked"""
    z1, _ = conv1(x, P["w1"], P["b1"], out_len)
    s1 = bn_stats(z1, P["rm1"], P["rv1"], momentum, eps)
    a1, _ = bn_act(z1, s1["mean"], s1["invstd"], P["g1"], P["be1"], out_len)
    z2, _ = conv2(a1, P["w2"], P["b2"], out_len)
    s2 = bn_stats(z2, P["rm2"], P["rv2"], momentum, eps)
    a2, _ = bn_act(z2, s2["mean"], s2["invstd"], P["g2"], P["be2"], out_len)
    return dict(z1=z1, s1=s1, a1=a1, z2=z2, s2=s2, y=time_major(a2))


def frontend_backward(x, out_len, P, z1, a1, z2, s1, s2, dy, m1=None, m2=None):
    """the backward from the given forward tensors and statistics (s1 / s2: dicts with mean, invstd) and the clip
    masks m1 / m2 (default: decided in float64 on u)"""
    if m2 is None:
        u2 = (z2.double() - _ch(s2["mean"])) * _ch(s2["invstd"]) * _ch(P["g2"]) + _ch(P["be2"])
        m2 = clip_mask(u2, out_len)
    if m1 is None:
        u1 = (z1.double() - _ch(s1["mean"])) * _ch(s1["invstd"]) * _ch(P["g1"]) + _ch(P["be1"])
        m1 = clip_mask(u1, out_len)
    b2 = bn_act_backward(z2, s2["mean"], s2["invstd"], P["g2"], m2, batch_major(dy.double(), D2), out_len)
    dw2 = conv2_wgrad(b2["dz"], a1)
    da1 = conv2_dgrad(b2["dz"], P["w2"])
    b1 = bn_act_backward(z1, s1["mean"], s1["invstd"], P["g1"], m1, da1, out_len)
    dw1 = conv1_wgrad(b1["dz"], x)
    return dict(st2=b2, st1=b1, da1=da1, dw2=dw2, dw1=dw1, db2=b2["dbias"], db1=b1["dbias"], dg2=b2["dgamma"],
                dbe2=b2["dbeta"], dg1=b1["dgamma"], dbe1=b1["dbeta"])


# ---- the checks' metrics: each returns (worst error) / (its bound), so a check passes at <= 1 ----------------------
def elementwise_ratio(got, ref, mag, c):
    """max |got - ref| / (c * mag); where mag is 0 (masked positions) the outputs must agree exactly"""
    d = (got.double() - ref.double()).abs()
    bound = c * mag.double()
    if bool((d[bound == 0] > 0).any()):
        return math.inf
    return float((d / bound.clamp_min(1e-300)).max())


def z1_c():
    """conv1 forward (FFMA): 451 fused multiply-adds in sequence and the bias add, then the store; each rounding is
    at most U32 of a partial sum bounded by |w1| * |x| + |b1|: gamma_453"""
    return (K1 + 2) * U32


def z2_c(tf32):
    """conv2 forward: 7392 products and the bias.  FFMA: gamma_7394 as for conv1.  Tensor cores: both operands
    rounded to TF32 (at most UTF32 each, 2 UTF32 + UTF32^2 per product) plus the fp32 accumulation's gamma_7394"""
    return (2 * UTF32 + UTF32 ** 2 if tf32 else 0.0) + (K2 + 2) * U32


def bn_act_c():
    """BN + Hardtanh from given statistics: z - mean, times invstd, one fma with gamma and beta: three roundings, each
    within U32 of a term of the magnitude bn_act returns (the clamp is 1-Lipschitz)"""
    return 4 * U32


def wgrad_ratio(got, ref, dz, dz_mag, inp, wgrad, k_terms, tf32):
    """per-entry check of a weight gradient whose input `inp` is the kernel's own (exact here) and whose output
    gradient dz the reference recomputed in float64 (the kernel's dz is off by at most 8 U32 dz_mag per element):
    |got - ref| <= NSIG * sigma + 8 U32 (dz_mag * |inp|), sigma from tc_sum_sigma with the sums of |products| and of
    squared products (each weight entry sums products of distinct element pairs: their roundings are independent)"""
    s_abs = wgrad(dz.abs(), inp.abs())
    s_sq = torch.sqrt(wgrad(dz * dz, inp.double() * inp.double()).clamp_min(0))
    bound = NSIG * tc_sum_sigma(s_sq, s_abs, k_terms, tf32) + 8 * U32 * wgrad(dz_mag, inp.abs())
    return elementwise_ratio(got, ref, bound, 1.0)


def rel_l2(got, ref):
    d = float(ref.double().norm())
    return float((got.double() - ref.double()).norm()) / (d if d > 0 else 1.0)


def round_tf32(t, truncate=False):
    """t rounded to TF32 (10 mantissa bits): to nearest even, or by truncation"""
    i = t.float().contiguous().view(torch.int32).to(torch.int64)
    if not truncate:
        i = i + 0xFFF + ((i >> 13) & 1)
    return (i & ~0x1FFF).to(torch.int32).view(torch.float32)


def same_sign_bias(z2, ref, b2, out_len):
    """mean signed relative error of conv2 without its bias over the valid positions: sum(got - ref) / sum(ref - b2)
    (all terms >= 0 when w2 >= 0, a1 >= 0).  Rounding to nearest has no bias (about 0 +- UTF32 / sqrt(count));
    truncating both operands to TF32 loses about half an ulp of each: about -7e-4"""
    m = keep(out_len, z2.shape[-1], z2.device)
    num = ((z2.double() - ref.double()) * m).sum()
    den = ((ref.double() - _ch(b2)) * m).sum()
    return float(num / den)
