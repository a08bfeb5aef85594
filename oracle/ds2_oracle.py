"""TEST INFRASTRUCTURE — the parity oracle.  Not product code, never imported by the package.

A CPU restatement (torch CPU tensors for the dense algebra + autograd, plain numpy float64
for the CTC lattice) of the DeepSpeech2 train-step path of SeanNaren/deepspeech.pytorch:

    reference deepspeech_pytorch/model.py
      :53-69    MaskConv.forward        -> mask_time / conv_frontend
      :94-102   BatchRNN.forward        -> batch_rnn (explicit per-timestep cells, length masking
                                           instead of pack/pad; proven equal, tests/test_oracle.py)
      :115-130  Lookahead.forward       -> lookahead
      :195-201  fc (BN1d + Linear)      -> fc_head
      :214-239  DeepSpeech.forward      -> forward
      :241-249  DeepSpeech.training_step-> train_step (+ ctc_loss_and_grad for torch CTCLoss :203)
      :299-310  DeepSpeech.get_seq_lens -> get_seq_lens

The arithmetic of the reference lives in third-party PyTorch (unpinned in the reference's
requirements.txt:14; torch 2.11.0 here).  Gate orders / CTC recursion are restated from
PyTorch's documented semantics:  LSTM rows [i,f,g,o], GRU rows [r,z,n] with
n = tanh(W_in x + b_in + r*(W_hn h + b_hn)), CTC = Graves 2006 in log space with
`zero_infinity`.

PINNING: the reference ships no golden vectors and no numeric tests ("parity unpinned" by its
own test-suite, SURVEY.md §8c).  This oracle is instead pinned against outputs of the reference
itself: `oracle/make_golden.py` executes the unmodified reference model.py (via
`oracle/ref_shim.py`) in the dev container and commits logits / loss / every parameter gradient /
running statistics to `tests/golden/*.npz`; `tests/test_oracle.py` checks this file against those
fixtures on every run (CPU, no reference needed).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
BN_MOMENTUM = 0.1
NUM_FREQ = 161


@dataclass
class OracleConfig:
    rnn_type: str = "lstm"          # "lstm" | "gru" | "rnn"   (reference enums.py:18-21)
    hidden_size: int = 1024         # reference train_config.py:48-50
    hidden_layers: int = 5
    bidirectional: bool = True
    lookahead_context: int = 20     # only when not bidirectional (train_config.py:55)
    num_classes: int = 29           # labels.json
    blank: int = 0


GATES = {"lstm": 4, "gru": 3, "rnn": 1}


# ----------------------------------------------------------------------------- lengths
def get_seq_lens(lengths: torch.Tensor) -> torch.Tensor:
    """reference model.py:299-310 — time axis of the two Conv2d: k=11,p=5,d=1, strides 2 then 1."""
    L = lengths.to(torch.int64)
    for (k, p, d, s) in ((11, 5, 1, 2), (11, 5, 1, 1)):
        L = torch.div(L + 2 * p - d * (k - 1) - 1, s, rounding_mode="floor") + 1
    return L.int()


def input_sizes_from_percentages(input_percentages: torch.Tensor, t_max: int) -> torch.Tensor:
    """reference model.py:243 — float32 multiply then truncation (kept bit-for-bit: may lose a frame)."""
    return input_percentages.clone().mul_(int(t_max)).int()


def mask_time(x: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """reference model.py:59-68 — zero positions t >= length[b] on the last axis of (B,C,D,T)."""
    T = x.size(-1)
    keep = (torch.arange(T, device=x.device)[None, :] < lengths.to(device=x.device, dtype=torch.int64)[:, None])  # (B,T)
    return x * keep[:, None, None, :].to(x.dtype)


# ----------------------------------------------------------------------------- blocks
def _bn_train(x2d_or_4d, weight, bias, running_mean, running_var, training, new_buffers, prefix):
    """torch BatchNorm semantics (biased var to normalise, unbiased var into running stats)."""
    if training:
        rm = running_mean.clone()
        rv = running_var.clone()
        y = F.batch_norm(x2d_or_4d, rm, rv, weight, bias, True, BN_MOMENTUM, BN_EPS)
        new_buffers[prefix + "running_mean"] = rm
        new_buffers[prefix + "running_var"] = rv
        return y
    return F.batch_norm(x2d_or_4d, running_mean, running_var, weight, bias, False, BN_MOMENTUM, BN_EPS)


def conv_frontend(x, out_lens, P, training, new_buffers):
    """reference model.py:157-164 wrapped by MaskConv :53-69: mask after EVERY sub-module."""
    pre = "conv.seq_module."
    x = F.conv2d(x, P[pre + "0.weight"], P[pre + "0.bias"], stride=(2, 2), padding=(20, 5))
    x = mask_time(x, out_lens)
    x = _bn_train(x, P[pre + "1.weight"], P[pre + "1.bias"], P[pre + "1.running_mean"], P[pre + "1.running_var"],
                  training, new_buffers, pre + "1.")
    x = mask_time(x, out_lens)
    x = mask_time(torch.clamp(x, 0.0, 20.0), out_lens)
    x = F.conv2d(x, P[pre + "3.weight"], P[pre + "3.bias"], stride=(2, 1), padding=(10, 5))
    x = mask_time(x, out_lens)
    x = _bn_train(x, P[pre + "4.weight"], P[pre + "4.bias"], P[pre + "4.running_mean"], P[pre + "4.running_var"],
                  training, new_buffers, pre + "4.")
    x = mask_time(x, out_lens)
    x = mask_time(torch.clamp(x, 0.0, 20.0), out_lens)
    return x


def _cell(rnn_type, gx, h, c, w_hh, b_hh):
    """One time step.  gx already holds x W_ih^T + b_ih."""
    gh = h @ w_hh.t() + b_hh
    if rnn_type == "lstm":
        i, f, g, o = (gx + gh).chunk(4, dim=-1)
        c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h2 = torch.sigmoid(o) * torch.tanh(c2)
        return h2, c2
    if rnn_type == "gru":
        xr, xz, xn = gx.chunk(3, dim=-1)
        hr, hz, hn = gh.chunk(3, dim=-1)
        r = torch.sigmoid(xr + hr)
        z = torch.sigmoid(xz + hz)
        n = torch.tanh(xn + r * hn)
        return (1.0 - z) * n + z * h, c
    return torch.tanh(gx + gh), c


def _run_direction(rnn_type, x, lens, w_ih, w_hh, b_ih, b_hh, h0, c0, reverse):
    T, B, _ = x.shape
    gx_all = x @ w_ih.t() + b_ih
    h, c = h0, c0
    outs = [None] * T
    order = range(T - 1, -1, -1) if reverse else range(T)
    for t in order:
        m = (lens > t).to(x.dtype)[:, None]
        h2, c2 = _cell(rnn_type, gx_all[t], h, c, w_hh, b_hh)
        h = m * h2 + (1.0 - m) * h
        if rnn_type == "lstm":
            c = m * c2 + (1.0 - m) * c
        outs[t] = m * h2
    return torch.stack(outs, 0), h, c


def batch_rnn(x, out_lens, P, prefix, cfg: OracleConfig, batch_norm, training, new_buffers, h0=None):
    """reference model.py:94-102.  x (T,B,In) already truncated to T = max(out_lens)."""
    T, B, _ = x.shape
    if batch_norm:
        bp = prefix + "batch_norm.module."
        x = _bn_train(x.reshape(T * B, -1), P[bp + "weight"], P[bp + "bias"], P[bp + "running_mean"],
                      P[bp + "running_var"], training, new_buffers, bp).reshape(T, B, -1)
    H = cfg.hidden_size
    dirs = 2 if cfg.bidirectional else 1
    lens = out_lens.to(torch.int64)
    ys, hns, cns = [], [], []
    for d in range(dirs):
        sfx = "_reverse" if d == 1 else ""
        if h0 is None:
            h_init = x.new_zeros(B, H)
            c_init = x.new_zeros(B, H)
        elif cfg.rnn_type == "lstm":
            h_init, c_init = h0[0][d], h0[1][d]
        else:
            h_init, c_init = h0[d], x.new_zeros(B, H)
        y, hn, cn = _run_direction(cfg.rnn_type, x, lens,
                                   P[prefix + "rnn.weight_ih_l0" + sfx], P[prefix + "rnn.weight_hh_l0" + sfx],
                                   P[prefix + "rnn.bias_ih_l0" + sfx], P[prefix + "rnn.bias_hh_l0" + sfx],
                                   h_init, c_init, reverse=(d == 1))
        ys.append(y), hns.append(hn), cns.append(cn)
    y = ys[0] + ys[1] if dirs == 2 else ys[0]  # model.py:100-101 sum of directions
    hn = torch.stack(hns, 0)
    if cfg.rnn_type == "lstm":
        return y, (hn, torch.stack(cns, 0))
    return y, hn


def batch_rnn_aten(x, out_lens, P, prefix, cfg: OracleConfig, batch_norm, training, new_buffers, h0=None):
    """Same layer through the ATen calls the reference itself makes (pack -> _VF.lstm/gru -> pad);
    used for the timed CPU baseline and to cross-check `batch_rnn`."""
    from torch import _VF
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    T, B, _ = x.shape
    if batch_norm:
        bp = prefix + "batch_norm.module."
        x = _bn_train(x.reshape(T * B, -1), P[bp + "weight"], P[bp + "bias"], P[bp + "running_mean"],
                      P[bp + "running_var"], training, new_buffers, bp).reshape(T, B, -1)
    dirs = 2 if cfg.bidirectional else 1
    flat = []
    for d in range(dirs):
        sfx = "_reverse" if d == 1 else ""
        flat += [P[prefix + "rnn.weight_ih_l0" + sfx], P[prefix + "rnn.weight_hh_l0" + sfx],
                 P[prefix + "rnn.bias_ih_l0" + sfx], P[prefix + "rnn.bias_hh_l0" + sfx]]
    packed = pack_padded_sequence(x, out_lens.cpu())
    H = cfg.hidden_size
    if h0 is None:
        z = x.new_zeros(dirs, B, H)
        h0 = (z, z.clone()) if cfg.rnn_type == "lstm" else z
    if cfg.rnn_type == "lstm":
        out, hn, cn = _VF.lstm(packed.data, packed.batch_sizes, h0, flat, True, 1, 0.0, training, cfg.bidirectional)
        h = (hn, cn)
    elif cfg.rnn_type == "gru":
        out, h = _VF.gru(packed.data, packed.batch_sizes, h0, flat, True, 1, 0.0, training, cfg.bidirectional)
    else:
        out, h = _VF.rnn_tanh(packed.data, packed.batch_sizes, h0, flat, True, 1, 0.0, training, cfg.bidirectional)
    packed_out = torch.nn.utils.rnn.PackedSequence(out, packed.batch_sizes, None, None)
    y, _ = pad_packed_sequence(packed_out)
    if dirs == 2:
        y = y.view(y.size(0), y.size(1), 2, -1).sum(2)
    return y, h


def lookahead(x, w):
    """reference model.py:125-130:  y[t,b,c] = sum_k w[c,0,k] * x[t+k,b,c], zero beyond T."""
    T, B, H = x.shape
    ctx = w.shape[-1]
    xp = torch.cat([x, x.new_zeros(ctx - 1, B, H)], 0)
    y = x.new_zeros(T, B, H)
    for k in range(ctx):
        y = y + xp[k:k + T] * w[:, 0, k][None, None, :]
    return y


def fc_head(x, P, training, new_buffers):
    """reference model.py:195-201 — BatchNorm1d(H) over all T*B rows then Linear(H->C, no bias)."""
    T, B, H = x.shape
    bp = "fc.0.module.0."
    z = _bn_train(x.reshape(T * B, H), P[bp + "weight"], P[bp + "bias"], P[bp + "running_mean"],
                  P[bp + "running_var"], training, new_buffers, bp)
    return (z @ P["fc.0.module.1.weight"].t()).reshape(T, B, -1)


def forward(x, lengths, P: Dict[str, torch.Tensor], cfg: OracleConfig, training: bool,
            hs: Optional[list] = None, use_aten_rnn: bool = False, taps: Optional[dict] = None):
    """reference model.py:214-239.  Returns (out (B,T_out,C), output_lengths i32, new_hs, new_buffers)."""
    new_buffers: Dict[str, torch.Tensor] = {}
    lengths = lengths.cpu().int()
    out_lens = get_seq_lens(lengths)
    y = conv_frontend(x, out_lens, P, training, new_buffers)
    if taps is not None:
        taps["conv"] = y
    B, C, D, Tp = y.shape
    y = y.reshape(B, C * D, Tp).permute(2, 0, 1).contiguous()          # (T',B,C*D), feature = c*41+d
    t_out = int(out_lens.max())
    y = y[:t_out]                                                      # pad_packed_sequence truncation
    if hs is None:
        hs = [None] * cfg.hidden_layers
    new_hs = []
    layer = batch_rnn_aten if use_aten_rnn else batch_rnn
    for i in range(cfg.hidden_layers):
        y, h = layer(y, out_lens, P, f"rnns.{i}.", cfg, batch_norm=(i > 0), training=training,
                     new_buffers=new_buffers, h0=hs[i])
        new_hs.append(h)
        if taps is not None:
            taps[f"rnn{i}"] = y
    if not cfg.bidirectional:
        y = torch.clamp(lookahead(y, P["lookahead.0.conv.weight"]), 0.0, 20.0)
        if taps is not None:
            taps["lookahead"] = y
    y = fc_head(y, P, training, new_buffers)
    out = y.transpose(0, 1)
    if not training:
        out = F.softmax(out, dim=-1)                                   # model.py:72-77
    return out, out_lens, new_hs, new_buffers


# ----------------------------------------------------------------------------- CTC (numpy, float64)
def _lse(*xs):
    m = np.maximum.reduce(xs)
    m_safe = np.where(np.isfinite(m), m, 0.0)
    s = sum(np.exp(x - m_safe) for x in xs)
    with np.errstate(divide="ignore"):
        return np.where(np.isfinite(m), m_safe + np.log(s), -np.inf)


def ctc_loss_and_grad(logits: np.ndarray, targets: np.ndarray, input_lengths, target_lengths,
                      blank: int = 0, zero_infinity: bool = True) -> Tuple[np.ndarray, np.ndarray]:
    """torch.nn.CTCLoss(blank, reduction='sum', zero_infinity) on log_softmax(logits) — the per-utterance
    negative log likelihoods and d(sum loss)/d(logits) = softmax - posterior (0 for t >= input_length,
    0 everywhere for an infeasible utterance).   logits (T,B,C); targets 1-D concatenated int64."""
    T, B, C = logits.shape
    x = logits.astype(np.float64)
    mx = x.max(-1, keepdims=True)
    lp = x - mx - np.log(np.exp(x - mx).sum(-1, keepdims=True))
    nll = np.zeros(B, np.float64)
    grad = np.zeros((T, B, C), np.float64)
    off = 0
    for b in range(B):
        Tb, Lb = int(input_lengths[b]), int(target_lengths[b])
        tg = np.asarray(targets[off:off + Lb], dtype=np.int64)
        off += Lb
        S = 2 * Lb + 1
        ext = np.full(S, blank, np.int64)
        ext[1::2] = tg
        can_skip = np.zeros(S, bool)                 # transition s-2 -> s allowed
        can_skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
        if Tb == 0:
            nll[b] = 0.0 if Lb == 0 else np.inf
        else:
            la = np.full((Tb, S), -np.inf)
            la[0, 0] = lp[0, b, blank]
            if S > 1:
                la[0, 1] = lp[0, b, ext[1]]
            for t in range(1, Tb):
                a0 = la[t - 1]
                a1 = np.concatenate(([-np.inf], a0[:-1]))
                a2 = np.where(can_skip, np.concatenate(([-np.inf, -np.inf], a0))[:S], -np.inf)   # [:S]: also S = 1
                la[t] = _lse(a0, a1, a2) + lp[t, b, ext]
            ll = _lse(la[Tb - 1, S - 1], la[Tb - 1, S - 2] if S > 1 else np.float64(-np.inf))
            nll[b] = -float(ll)
        if not np.isfinite(nll[b]):
            if zero_infinity:
                nll[b] = 0.0
            continue
        if Tb == 0:
            continue
        lb = np.full((Tb, S), -np.inf)
        lb[Tb - 1, S - 1] = lp[Tb - 1, b, blank]
        if S > 1:
            lb[Tb - 1, S - 2] = lp[Tb - 1, b, ext[S - 2]]
        skip_fwd = np.zeros(S, bool)                 # transition s -> s+2 allowed
        skip_fwd[:-2] = can_skip[2:]
        for t in range(Tb - 2, -1, -1):
            b0 = lb[t + 1]
            b1 = np.concatenate((b0[1:], [-np.inf]))
            b2 = np.where(skip_fwd, np.concatenate((b0[2:], [-np.inf, -np.inf]))[:S], -np.inf)
            lb[t] = _lse(b0, b1, b2) + lp[t, b, ext]
        # posterior[t,c] = sum_{s: ext[s]=c} exp(la+lb - lp[t,c] + nll)
        lab = la + lb
        post = np.zeros((Tb, C))
        m = lab + nll[b] - lp[:Tb, b][:, ext]
        e = np.exp(m)
        for s in range(S):
            post[:, ext[s]] += e[:, s]
        grad[:Tb, b] = np.exp(lp[:Tb, b]) - post
    return nll, grad


# ----------------------------------------------------------------------------- whole step
def train_step(inputs, targets, input_percentages, target_sizes, P, cfg: OracleConfig,
               use_aten_rnn: bool = False, use_aten_ctc: bool = False):
    """reference model.py:241-249 followed by loss.backward().
    Returns dict(loss, logits (B,T_out,C), output_sizes, grads {name: tensor}, new_buffers)."""
    P = {k: (v.detach().clone().requires_grad_(True) if v.dtype.is_floating_point and "running_" not in k else v)
         for k, v in P.items()}
    input_sizes = input_sizes_from_percentages(input_percentages, inputs.size(3))
    out, output_sizes, _, new_buffers = forward(inputs, input_sizes, P, cfg, training=True,
                                                use_aten_rnn=use_aten_rnn)
    logits_tbc = out.transpose(0, 1)
    if use_aten_ctc:
        loss = F.ctc_loss(logits_tbc.log_softmax(-1), targets, output_sizes, target_sizes, blank=cfg.blank,
                          reduction="sum", zero_infinity=True)
        loss.backward()
        loss_val = float(loss.detach())
    else:
        nll, g = ctc_loss_and_grad(logits_tbc.detach().numpy(), targets.numpy(), output_sizes.numpy(),
                                   target_sizes.numpy(), blank=cfg.blank)
        loss_val = float(nll.sum())
        logits_tbc.backward(torch.from_numpy(g).to(logits_tbc.dtype))
    grads = {k: v.grad.detach() for k, v in P.items() if isinstance(v, torch.Tensor) and v.requires_grad
             and v.grad is not None}
    return dict(loss=loss_val, logits=out.detach(), output_sizes=output_sizes, grads=grads,
                new_buffers=new_buffers)


# ----------------------------------------------------------------------------- greedy decode (N2)
def greedy_path(probs: torch.Tensor, sizes, blank: int = 0) -> List[Tuple[List[int], List[int]]]:
    """reference decoder.py:144-181 as integers: argmax -> drop blank -> collapse repeats;
    returns per utterance (label indices, frame offsets)."""
    am = probs.argmax(2)
    res = []
    for b in range(am.size(0)):
        n = int(sizes[b]) if sizes is not None else am.size(1)
        lab, offs = [], []
        for i in range(n):
            c = int(am[b, i])
            if c != blank and not (i != 0 and c == int(am[b, i - 1])):
                lab.append(c), offs.append(i)
        res.append((lab, offs))
    return res


# ----------------------------------------------------------------------------- parameters
def init_params(cfg: OracleConfig, seed: int = 123456) -> Dict[str, torch.Tensor]:
    """Random parameters with the reference's state_dict keys and shapes (SURVEY.md §8a) and
    torch-like init scales.  Used for synthetic tests/bench (not bit-identical to torch's init)."""
    g = torch.Generator().manual_seed(seed)

    def U(shape, bound):
        return (torch.rand(shape, generator=g) * 2 - 1) * bound

    P: Dict[str, torch.Tensor] = {}
    pre = "conv.seq_module."
    for idx, (co, ci, kh, kw) in (("0", (32, 1, 41, 11)), ("3", (32, 32, 21, 11))):
        bound = 1.0 / math.sqrt(ci * kh * kw)
        P[pre + idx + ".weight"] = U((co, ci, kh, kw), bound)
        P[pre + idx + ".bias"] = U((co,), bound)

    def bn(prefix, n):
        P[prefix + "weight"] = 1.0 + 0.1 * U((n,), 1.0)
        P[prefix + "bias"] = 0.1 * U((n,), 1.0)
        P[prefix + "running_mean"] = torch.zeros(n)
        P[prefix + "running_var"] = torch.ones(n)
        P[prefix + "num_batches_tracked"] = torch.zeros((), dtype=torch.int64)

    bn(pre + "1.", 32)
    bn(pre + "4.", 32)
    H, G = cfg.hidden_size, GATES[cfg.rnn_type]
    k = 1.0 / math.sqrt(H)
    in0 = 32 * 41
    for i in range(cfg.hidden_layers):
        In = in0 if i == 0 else H
        if i > 0:
            bn(f"rnns.{i}.batch_norm.module.", H)
        for sfx in (["", "_reverse"] if cfg.bidirectional else [""]):
            P[f"rnns.{i}.rnn.weight_ih_l0{sfx}"] = U((G * H, In), k)
            P[f"rnns.{i}.rnn.weight_hh_l0{sfx}"] = U((G * H, H), k)
            P[f"rnns.{i}.rnn.bias_ih_l0{sfx}"] = U((G * H,), k)
            P[f"rnns.{i}.rnn.bias_hh_l0{sfx}"] = U((G * H,), k)
    if not cfg.bidirectional:
        P["lookahead.0.conv.weight"] = U((H, 1, cfg.lookahead_context), 1.0 / math.sqrt(cfg.lookahead_context))
    bn("fc.0.module.0.", H)
    P["fc.0.module.1.weight"] = U((cfg.num_classes, H), k)
    return P


def synth_batch(B: int, T: int, seed: int = 1234, ragged: bool = True, lmin: int = 150, lmax: int = 200,
                num_classes: int = 29):
    """SURVEY.md §8d synthetic inputs: N(0,1) spectrograms, lengths descending, labels 1..C-1."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, NUM_FREQ, T, generator=g)
    if ragged and B > 1:
        lens = [int(round(T * (1 - 0.4 * i / (B - 1)))) for i in range(B)]
    else:
        lens = [T] * B
    for b, l in enumerate(lens):
        x[b, :, :, l:] = 0
    pct = torch.tensor([l / float(T) for l in lens], dtype=torch.float32)
    tp = [int(get_seq_lens(torch.tensor([l]))[0]) for l in lens]
    tl = []
    for b in range(B):
        hi = max(1, min(lmax, tp[b] // 2 - 1))
        lo = max(1, min(lmin, hi))
        tl.append(int(torch.randint(lo, hi + 1, (1,), generator=g)))
    target_sizes = torch.tensor(tl, dtype=torch.int32)
    targets = torch.randint(1, num_classes, (int(sum(tl)),), generator=g, dtype=torch.int64)
    return x, targets, pct, target_sizes
