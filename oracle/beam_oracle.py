"""Prefix beam search for CTC without a language model (row N5), in float64 Python/numpy.

The reference builds its beam decoder in deepspeech_pytorch/decoder.py:56-118 (BeamCTCDecoder) as a wrapper around
the external C++ `ctcdecode.CTCBeamDecoder`, which runs PaddlePaddle's `ctc_beam_search_decoder` on a path trie.
That library is not part of the reference checkout, so parity with it is UNPINNED.  What this module computes is
defined by the rules below (ctcdecode's algorithm with `ext_scorer == nullptr`; it deviates only where ctcdecode's
behaviour is order-dependent or degenerate, marked (!)).  The same rules head csrc/beam_decode.cu and DESIGN.md §5.7.

Inputs: probs (B, T, C) fp32 probabilities (the model's eval output, InferenceBatchSoftmax); sizes (B), optional:
frames t >= sizes[b] are ignored; blank, beam_width W, cutoff_top_n, cutoff_prob.

All path arithmetic is in float64 log space, with lp[c] = log((double) p[c]) and log 0 = -inf.  lse(a, b) is a
log-sum-exp that returns -inf when both arguments are -inf, and never NaN.  (!) ctcdecode keeps path probabilities
in fp32; fp64 here makes GPU and oracle agree to rounding of the last bits, so list order can be tested exactly.

1. State.  There is an ordered list of at most W prefixes.  Each prefix has log_b, log_nb and
   score = lse(log_b, log_nb).  Before frame 0 the list is {empty prefix: log_b = 0, log_nb = -inf}.
2. Prefix identity is by content.  The same label sequence is never in the list twice.
   - A prefix that falls out of the list and is produced again later is the same prefix.  Its probabilities restart
     from the new contributions, but it keeps its timestep record (rule 7).  This is ctcdecode's trie node coming
     back with `exists_ = true`.
   - A prefix's parent is its sequence minus the last label.
3. Character pruning per frame.
   - If cutoff_prob < 1 or cutoff_top_n < C: order the characters by (p desc, index asc).
   - With cutoff_prob < 1, take characters in that order, accumulating p in fp64, until the cumulative sum is
     >= cutoff_prob or cutoff_top_n characters are taken.
   - Otherwise take the first cutoff_top_n characters.
   - In all other cases the kept set K is every character.
   - The blank can be pruned.  It then contributes nothing that frame.
4. Candidates at frame t.  For each listed prefix j, with last label l_j, and its parent pi if the parent is in the
   list, the stay candidate is:
   - b' = lp[blank] + score_j if blank in K, else -inf.
   - nb' = lse(lp[l_j] + nb_j, lp[l_j] + (b_pi if l_pi = l_j else score_pi)).
   - Each term is present only if l_j in K, and the second only if pi is listed.  The empty prefix has no nb terms.
   For each listed prefix i and each c in K with c != blank, where i + c is not in the list, the new candidate is:
   - b' = -inf.
   - nb' = lp[c] + (b_i if c = l_i else score_i).
5. Selection.
   - Drop candidates whose score is -inf.  (!) ctcdecode can return -inf prefixes when fewer than W finite ones exist.
   - Order the rest by (score desc, origin asc).  The origin is (j, -1) for the stay candidate of list position j
     and (i, c) for a new candidate.  (!) This is a total order, so ties are defined.
   - The first W candidates become the new list, in that order.
6. Output.
   - Per utterance, the final list in its order, with each prefix's labels and per-label timesteps.  Its reported
     score is the negated final score, i.e. -lse(log_b, log_nb).  That is ctcdecode's sign: a negative
     log-likelihood, lower is better.
   - n_beams[b] <= W.  Unused slots have length 0 and score +inf.
   - sizes[b] = 0 gives one empty beam with score 0.
7. Timesteps.  A label's timestep is the frame at which its prefix was first created, with best = that frame's lp.
   It moves to a later frame t when, at t, the listed parent is extended by the same label with a strictly larger lp
   than the recorded best.  This is ctcdecode's `get_path_trie` rule as we read it; it is not verifiable here.

How the rules are read where they leave room:
- "Created" is the frame at which the prefix first enters the list.  The move of rule 7 is checked for listed
  prefixes whose parent is listed and whose last label is in K (the stay candidate's second nb term), whether or not
  the stay candidate survives selection; a prefix that returns to the list keeps its record unchanged.
- The timesteps reported for a prefix are the records of its ancestors (and its own) at the end of the utterance,
  as ctcdecode's `get_path_vec` walks the trie: a record that moved after a child was created shows in the child.
- A NaN score counts as -inf (dropped).  Scores of +0 and -0 are the same score.

`beam_search` also returns the smallest decision margin it met: the score gap between neighbours in the selection
order over the first min(W + 1, #candidates) candidates (every comparison that decided membership or order), and
|cumulative p - cutoff_prob| at every threshold comparison of rule 3.  A test whose margin is far above the rounding
of fp64 may demand exact equality of the list from any fp64 implementation.
"""
import math
from typing import List, Optional, Tuple

import numpy as np

NEG = -math.inf


def lse(a: float, b: float) -> float:
    m = max(a, b)
    if m == NEG:
        return NEG
    return m + math.log1p(math.exp(-abs(a - b)))


def _lse_vec(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    m = np.maximum(a, b)
    out = np.full_like(m, NEG)
    f = m > NEG
    out[f] = m[f] + np.log1p(np.exp(-np.abs(a[f] - b[f])))
    return out


def kept_chars(p: np.ndarray, cutoff_top_n: int, cutoff_prob: float) -> Tuple[List[int], float]:
    """rule 3: the kept set K (ascending index) and the smallest |cum - cutoff_prob| compared"""
    C = p.shape[0]
    margin = math.inf
    thr = float(np.float32(cutoff_prob))                  # the C-ABI takes cutoff_prob as fp32
    if not (thr < 1.0 or cutoff_top_n < C):
        return list(range(C)), margin
    order = sorted(range(C), key=lambda c: (-float(p[c]), c))
    if thr < 1.0:
        cum, K = 0.0, []
        for c in order:
            cum += float(p[c])
            K.append(c)
            margin = min(margin, abs(cum - thr))
            if cum >= thr or len(K) >= cutoff_top_n:
                break
    else:
        K = order[:cutoff_top_n]
    return sorted(K), margin


def beam_search(probs: np.ndarray, size: Optional[int], blank: int, beam_width: int, cutoff_top_n: int,
                cutoff_prob: float, trace: Optional[list] = None):
    """probs (T, C) fp32 -> (beams [(labels, timesteps, score)] in list order, decision margin).
    `trace`, if given, receives the list after every frame as [(prefix, log_b, log_nb)]."""
    probs = np.asarray(probs, dtype=np.float32)
    T, C = probs.shape
    n = T if size is None else max(0, min(int(size), T))
    W = beam_width
    rec = {}                                   # prefix -> [timestep, best lp]   (the node pool; by content)
    pre = [()]                                 # list: prefixes, log_b, log_nb
    lb = np.array([0.0])
    lnb = np.array([NEG])
    margin = math.inf
    for t in range(n):
        p = probs[t].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            lp = np.log(p)
        K, m3 = kept_chars(probs[t], cutoff_top_n, cutoff_prob)
        margin = min(margin, m3)
        inK = np.zeros(C, dtype=bool)
        inK[K] = True
        Knb = np.array([c for c in K if c != blank], dtype=np.int64)
        L = len(pre)
        sc = _lse_vec(lb, lnb)
        slot = {pr: j for j, pr in enumerate(pre)}
        last = np.array([pr[-1] if pr else -1 for pr in pre], dtype=np.int64)
        # stay candidates (rule 4, first half) and the timestep move (rule 7)
        sb = np.full(L, NEG)
        snb = np.full(L, NEG)
        listed_child = np.zeros((L, C), dtype=bool)
        for j, pr in enumerate(pre):
            if inK[blank]:
                sb[j] = lp[blank] + sc[j]
            if not pr:
                continue
            l = pr[-1]
            pi = slot.get(pr[:-1])
            if pi is not None:
                listed_child[pi, l] = True
            if not inK[l]:
                continue
            v = lp[l] + lnb[j]
            if pi is not None:
                v = lse(v, lp[l] + (lb[pi] if last[pi] == l else sc[pi]))
                r = rec[pr]
                if lp[l] > r[1]:
                    rec[pr] = [t, lp[l]]
            snb[j] = v
        stay = _lse_vec(sb, snb)
        # new candidates (rule 4, second half)
        if len(Knb):
            base = np.where(Knb[None, :] == last[:, None], lb[:, None], sc[:, None])
            new = lp[Knb][None, :] + base
            new[listed_child[:, Knb]] = NEG
        else:
            new = np.zeros((L, 0))
        # selection (rule 5): score desc, origin asc; origin (j, -1) / (i, c)
        s_all = np.concatenate([stay, new.reshape(-1)])
        oi = np.concatenate([np.arange(L), np.repeat(np.arange(L), len(Knb))])
        oc = np.concatenate([np.full(L, -1), np.tile(Knb, L)])
        s_all = s_all + 0.0                                        # -0 -> +0
        ok = s_all > NEG                                           # drops -inf and NaN
        s_all, oi, oc = s_all[ok], oi[ok], oc[ok]
        order = np.lexsort((oc, oi, -s_all))
        head = s_all[order[:W + 1]]
        if len(head) > 1:
            margin = min(margin, float(np.min(head[:-1] - head[1:])))
        keep = order[:W]
        npre, nlb, nlnb = [], np.empty(len(keep)), np.empty(len(keep))
        for r, k in enumerate(keep):
            i, c = int(oi[k]), int(oc[k])
            if c < 0:
                npre.append(pre[i])
                nlb[r], nlnb[r] = sb[i], snb[i]
            else:
                pr = pre[i] + (c,)
                if pr not in rec:
                    rec[pr] = [t, lp[c]]
                npre.append(pr)
                nlb[r], nlnb[r] = NEG, s_all[k]
        pre, lb, lnb = npre, nlb, nlnb
        if trace is not None:
            trace.append([(pr, float(lb[j]), float(lnb[j])) for j, pr in enumerate(pre)])
    sc = _lse_vec(lb, lnb)
    beams = []
    for j, pr in enumerate(pre):
        ts = [rec[pr[:k + 1]][0] for k in range(len(pr))]
        beams.append((list(pr), ts, -sc[j] + 0.0))
    return beams, margin


def beam_decode(probs, sizes, blank: int = 0, beam_width: int = 100, cutoff_top_n: int = 40,
                cutoff_prob: float = 1.0):
    """(B, T, C) -> dict of arrays in the C-ABI's layout (labels/timesteps (B, W, T), lengths/scores (B, W),
    n_beams (B)) plus the smallest decision margin over the batch"""
    probs = np.asarray(probs.detach().cpu().numpy() if hasattr(probs, "detach") else probs, dtype=np.float32)
    B, T, C = probs.shape
    W = beam_width
    labels = np.zeros((B, W, T), np.int32)
    timesteps = np.zeros((B, W, T), np.int32)
    lengths = np.zeros((B, W), np.int32)
    scores = np.full((B, W), math.inf)
    n_beams = np.zeros(B, np.int32)
    margin = math.inf
    for b in range(B):
        size = None if sizes is None else int(sizes[b])
        beams, m = beam_search(probs[b], size, blank, W, cutoff_top_n, cutoff_prob)
        margin = min(margin, m)
        n_beams[b] = len(beams)
        for r, (lab, ts, s) in enumerate(beams):
            lengths[b, r] = len(lab)
            labels[b, r, :len(lab)] = lab
            timesteps[b, r, :len(lab)] = ts
            scores[b, r] = s
    return dict(labels=labels, timesteps=timesteps, lengths=lengths, scores=scores, n_beams=n_beams, margin=margin)
