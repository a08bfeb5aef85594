"""TEST INFRASTRUCTURE — CPU restatement (numpy float64) of the reference's SpecAugment, as
`SpectrogramParser.parse_audio` applies it to one normalised (F, T) utterance (reference
deepspeech_pytorch/loader/data_loader.py:161-163).  Not product code.

  reference deepspeech_pytorch/loader/spec_augment.py
    :48-65    time_warp            -> the control point (draws 1-2) and `warp`
    :68-115   spec_augment         -> `draws` (the generator order) and `spec_augment`
  reference deepspeech_pytorch/loader/sparse_image_warp.py
    :141-184  solve_interpolation  -> `solve` (order 2, the 4x4 system, the tiny randn block)
    :187-205  cross_squared_distance_matrix (sums x^2 over ALL query points) -> `dense_flow_x`
    :236-266  apply_interpolation  -> `dense_flow_x`
    :269-410  dense_image_warp / interpolate_bilinear -> `warp`

What is kept in fp32 on purpose, because the reference's semantics depend on it: the control point
c = (F//2, fp32(p + d)) and its x-flow fx = fp32(c1 - p), with p the fp32 spectrogram value at
(F//2, idx).  Everything downstream is float64.  tests/test_spec_augment.py pins this file against
tests/golden/spec_augment/spec_augment.npz, written by running the reference itself.
"""
import random

import numpy as np
import torch

W = 5                    # time_warp's own default (spec_augment.py:48); time_warping_para=40 is never passed on
FREQ_MASK_PARA = 27      # spec_augment.py:68 defaults, one mask each
TIME_MASK_PARA = 70


def draws(frames, F=161):
    """the random numbers spec_augment draws for each utterance, one utterance after another, from the
    process-global `random`, `np.random` and torch CPU generators in the reference's order"""
    out = []
    for T in frames:
        T = int(T)
        idx = random.randrange(W, T - W)                       # spec_augment.py:56 (raises for T <= 10)
        d = random.randrange(-W, W)                            # :60
        Z = (torch.randn((1, 3, 3)) / 1e10).numpy().reshape(9)  # sparse_image_warp.py:170
        f = int(np.random.uniform(low=0.0, high=FREQ_MASK_PARA))  # spec_augment.py:99-100
        if F - f < 0:                                          # :101-103
            f, f0 = 0, 0
        else:
            f0 = random.randint(0, F - f)
        t = int(np.random.uniform(low=0.0, high=TIME_MASK_PARA))  # :108-109
        if T - t < 0:                                          # :110-111: skipped, no randint drawn
            t, t0 = 0, 0
        else:
            t0 = random.randint(0, T - t)
        out.append(dict(idx=idx, d=d, Z=Z.astype(np.float32), f0=f0, f=f, t0=t0, t=t))
    return out


def control_point(spect, dr):
    """(c0, c1, fx): c = (F//2, fp32(p + d)), fx = fp32(c1 - p) with p = spect[F//2, idx] (fp32)"""
    F = spect.shape[0]
    p = np.float32(spect[F // 2, dr["idx"]])
    c1 = np.float32(p + np.float32(dr["d"]))
    fx = np.float32(c1 - p)
    return float(F // 2), float(c1), float(fx)


def solve(c0, c1, fx, Z):
    """order-2 polyharmonic fit through one control point (sparse_image_warp.py:141-184), float64:
    [[A, b^T], [b, Z]] [w; v] = [fx; 0], b = (c0, c1, 1), A = phi(|c - c|^2) = 0.  -> (w, v0, v1, v2)"""
    b = np.array([c0, c1, 1.0])
    M = np.zeros((4, 4))
    M[0, 1:] = b
    M[1:, 0] = b
    M[1:, 1:] = np.asarray(Z, np.float64).reshape(3, 3)
    x = np.linalg.solve(M, np.array([fx, 0.0, 0.0, 0.0]))
    return x[0], x[1], x[2], x[3]


def phi(r):
    return 0.5 * r * np.log(np.maximum(r, 1e-10))


def dense_flow_x(F, T, c0, c1, w, v0, v1, v2):
    """the x (time) component of the dense flow on the (F, T) grid (sparse_image_warp.py:236-266).  The squared
    distance uses the reference's sum of x^2 over ALL grid points (cross_squared_distance_matrix, :197), not the
    per-point norm.  The y component is exactly 0: its right-hand side is zero."""
    j = np.arange(F, dtype=np.float64)[:, None]
    i = np.arange(T, dtype=np.float64)[None, :]
    grid_sum = float(T * np.sum(np.arange(F, dtype=np.float64) ** 2) + F * np.sum(np.arange(T, dtype=np.float64) ** 2))
    r = grid_sum - 2.0 * (j * c0 + i * c1) + (c0 * c0 + c1 * c1)
    return phi(r) * w + (j * v0 + i * v1 + v2)


def warp(spect, flow_x):
    """dense_image_warp with a zero y-flow (:269-410): output (j, i) bilinearly samples (j, i - flow_x) with the
    floor clamped to [0, size - 2] and alpha to [0, 1] in each dimension; the last row takes alpha_y = 1."""
    s = np.asarray(spect, np.float64)
    F, T = s.shape
    j = np.arange(F)[:, None]
    q = np.arange(T, dtype=np.float64)[None, :] - flow_x
    fl = np.minimum(np.maximum(0.0, np.floor(q)), T - 2)
    ax = np.clip(q - fl, 0.0, 1.0)
    fx = fl.astype(np.int64)
    fy = np.minimum(j, F - 2) + np.zeros_like(fx)
    ay = np.clip(j - np.minimum(j, F - 2), 0.0, 1.0)
    tl, tr = s[fy, fx], s[fy, fx + 1]
    bl, br = s[fy + 1, fx], s[fy + 1, fx + 1]
    top = tl + ax * (tr - tl)
    bot = bl + ax * (br - bl)
    return top + ay * (bot - top)


def spec_augment(spect, dr):
    """one utterance: time warp, then the frequency mask, then the time mask.  -> (out float64 (F, T),
    flow_x float64 (F, T))"""
    spect = np.asarray(spect, np.float32)
    F, T = spect.shape
    c0, c1, fx = control_point(spect, dr)
    w, v0, v1, v2 = solve(c0, c1, fx, dr["Z"])
    flow = dense_flow_x(F, T, c0, c1, w, v0, v1, v2)
    out = warp(spect, flow)
    out[dr["f0"]:dr["f0"] + dr["f"], :] = 0.0
    out[:, dr["t0"]:dr["t0"] + dr["t"]] = 0.0
    return out, flow
