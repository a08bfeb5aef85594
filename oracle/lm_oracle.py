"""Prefix beam search for CTC with an ARPA n-gram language model (row N6), in float64 Python/numpy.

The reference decodes with a KenLM model through ctcdecode's `Scorer` (PaddlePaddle's `ctc_beam_search_decoder` with
`ext_scorer` set, `fill_dictionary(true)`, `OOV_SCORE = -1000`).  Neither ctcdecode nor KenLM is part of the
reference checkout, so parity with them is UNPINNED.  What this module computes is rules 1-7 of
`oracle/beam_oracle.py` plus the rules below; the same text heads csrc/beam_decode.cu and DESIGN.md §5.7.  (!) marks
a deviation, used only where ctcdecode is order-dependent or degenerate.

L0. Model.
   - The model is an ARPA text file, plain or gzip'd.  Values are parsed to fp32, as KenLM stores them.  A backoff
     that is not written is 0.  Word ids follow the unigram order of the file.
   - Refused (deepspeech.pytorch_b200/lm.py, with a message containing "language-model scoring"): a missing file; a
     file that is not ARPA (a KenLM binary); counts that do not match the \\data\\ header; duplicate n-grams;
     order > 5 or >= 2^24 words; no <s> unigram; labels without ' '; a character-based model (every word one
     character); a model of which no word can be spelled with the labels.
L1. Vocabulary V and dictionary constraint.
   - V is the set of unigrams other than <s>, </s> and <unk> whose every character is a label other than the blank's
     and the space's.  (!) ctcdecode would also map the blank's character.
   - A prefix splits at spaces into its completed words and its partial word, the run after the last space (maybe
     empty).
   - A new candidate (i, c), c != blank, exists only if c != space and partial(i)+c is a prefix of some word in V, or
     c = space and partial(i) is in V.  Leading and double spaces are therefore impossible.
   - (!) ctcdecode's FST matcher rejects the first character after a space in the frame in which it resets its
     state.  Which character that hits depends on the visiting order, so that rejection is not reproduced.
L2. LM value.
   - lm(w | u_1..u_k) is the ARPA conditional log10 probability of w.  Its context is the last N-1 items of
     (<s>^(N-1), u_1, ..., u_k): the longest listed n-gram, plus the backoffs of the longer unlisted contexts, with a
     backoff of 0 for a context that is not listed.  The fp32 values are summed in fp64, from the longest context
     down.
   - A word outside the ARPA vocabulary gets lm = -1000 (LM_OOV), before alpha multiplies it.
   - a(w) = alpha * lm + beta.
   - (!) Units: the value is used in log10, unconverted (LM_SCALE = 1).  That is how we read ctcdecode's
     `get_log_cond_prob`; it is not verifiable here, and it decides whether alpha values tuned with the reference
     carry over.
L3. Where a(w) enters: on the path from "...w" to "...w ".
   - The new candidate (i, space): nb' = lp[space] + score_i + a(partial(i) | ctx(i)).
   - A listed prefix that ends in a space and whose parent pi is listed: the second nb term of its stay candidate.
   - The first nb term (the space repeated) gets no LM term.  Prefix scores carry every LM term from then on.
L4. Full-beam filter (ctcdecode's min_cutoff), when the list holds W prefixes at the start of frame t.
   - m = score of the last listed prefix + log p[blank] - max(0, beta), p[blank] unpruned.
   - Every contribution from a prefix x through a character c with lp[c] + score_x < m is dropped: the blank term of
     a stay (x = j), both nb terms of a stay (x = j, then x = pi, with c = l_j), a new candidate (x = i).
   - A dropped contribution does not move a timestep under rule 7.
L5. End of utterance.
   - Each listed prefix that is non-empty and does not end in a space gets score += a(partial | ctx); a partial word
     not in V scores lm = -1000.
   - The list is reordered by (score desc, list position asc) and -score is reported.
   - (!) ctcdecode orders by this score but reports an "approx_ctc" that subtracts beta once per character and alpha
     times a sentence probability including </s>, a term the search never added.  Here the reported score is the one
     the beams are ordered by.
   - sizes[b] = 0 still gives one empty beam with score 0.

`beam_search_lm` returns the smallest decision margin as `beam_oracle.beam_search` does, and also |lp[c] + score_x - m|
at every L4 comparison and the score gaps of the L5 reorder.
"""
import gzip
import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle import beam_oracle as BO

NEG = -math.inf
LM_OOV = -1000.0
LM_SCALE = 1.0          # log10 values used as written (rule L2); ln 10 if ctcdecode converts to natural log
SPECIAL = ("<s>", "</s>", "<unk>")


class ArpaLM:
    """an ARPA model in float64 dicts: prob[(w1..wn)] = log10 p, bo[(w1..wn)] = log10 backoff (fp32 values)"""

    def __init__(self, order: int, words: List[str], prob: Dict[tuple, float], bo: Dict[tuple, float]):
        self.order, self.words, self.prob, self.bo = order, words, prob, bo
        self.vocab = set(words)

    def lm(self, w: str, ctx: Tuple[str, ...]) -> float:
        """rule L2: lm(w | ctx), ctx the N-1 context words (already <s>-padded), oldest first"""
        if w not in self.vocab:
            return LM_OOV
        N = self.order
        acc = 0.0
        for n in range(N, 0, -1):
            h = tuple(ctx[len(ctx) - (n - 1):]) if n > 1 else ()
            g = h + (w,)
            if g in self.prob:
                return LM_SCALE * (acc + self.prob[g])
            if n > 1:
                acc = acc + self.bo.get(h, 0.0)
        return LM_OOV

    def context(self, words: Tuple[str, ...]) -> Tuple[str, ...]:
        """the last N-1 items of (<s>^(N-1), words...)"""
        k = self.order - 1
        if k == 0:
            return ()
        full = ("<s>",) * k + tuple(words)
        return full[len(full) - k:]


def _f32(s: str) -> float:
    return float(np.float32(float(s)))


def read_arpa(path) -> ArpaLM:
    """a plain line-by-line ARPA reader (no refusals beyond what it cannot read)"""
    op = gzip.open if open(path, "rb").read(2) == b"\x1f\x8b" else open
    with op(path, "rt", encoding="utf-8") as f:
        lines = f.read().split("\n")
    order, n, words, prob, bo = 0, 0, [], {}, {}
    for line in lines:
        s = line.strip()
        if not s:
            continue
        if s.startswith("ngram "):
            order = max(order, int(s[6:].split("=")[0]))
            continue
        if s.startswith("\\"):
            n = int(s[1:s.index("-")]) if s.endswith("-grams:") else 0
            continue
        if n == 0:
            continue
        f = s.split()
        g = tuple(f[1:1 + n])
        prob[g] = _f32(f[0])
        if len(f) == n + 2:
            bo[g] = _f32(f[n + 1])
        if n == 1:
            words.append(f[1])
    return ArpaLM(order, words, prob, bo)


class Dictionary:
    """rule L1 over label tuples: V, the set of prefixes of V's words, and the word string of each"""

    def __init__(self, lm: ArpaLM, labels, blank: int):
        labels = list(labels)
        self.space = labels.index(' ')
        idx = {ch: i for i, ch in enumerate(labels) if i not in (blank, self.space)}
        self.word_of: Dict[tuple, str] = {}
        for w in lm.words:
            if w in SPECIAL or not w or any(ch not in idx for ch in w):
                continue
            self.word_of[tuple(idx[ch] for ch in w)] = w
        self.prefixes = {s[:k] for s in self.word_of for k in range(len(s) + 1)}
        self.labels = labels

    def split(self, pr: tuple) -> Tuple[Tuple[str, ...], tuple]:
        """completed words (as strings) and the partial word (label tuple) of a prefix"""
        sp = [k for k, c in enumerate(pr) if c == self.space]
        start, words = 0, []
        for k in sp:
            words.append(''.join(self.labels[c] for c in pr[start:k]))
            start = k + 1
        return tuple(words), tuple(pr[start:])

    def allowed(self, partial: tuple, c: int) -> bool:
        if c == self.space:
            return partial in self.word_of
        return partial + (c,) in self.prefixes


def beam_search_lm(probs: np.ndarray, size: Optional[int], blank: int, beam_width: int, cutoff_top_n: int,
                   cutoff_prob: float, labels, lm: ArpaLM, alpha: float, beta: float, trace: Optional[list] = None,
                   stats: Optional[dict] = None):
    """probs (T, C) fp32 -> (beams [(labels, timesteps, score)] best first, decision margin); rules 1-7, L1-L5.
    `trace`, if given, receives the list after every frame as [(prefix, log_b, log_nb)]; `stats`, if given, counts
    the contributions L4 dropped under "l4_drops".  The blank term of the last listed prefix is exactly m (beta <= 0)
    or above it whatever the rounding, so it is not a decision and not part of the margin."""
    stats = {} if stats is None else stats
    stats.setdefault("l4_drops", 0)
    probs = np.asarray(probs, dtype=np.float32)
    T, C = probs.shape
    n = T if size is None else max(0, min(int(size), T))
    W = beam_width
    alpha, beta = float(alpha), float(beta)
    D = Dictionary(lm, labels, blank)
    space = D.space
    info = {}

    def lmv(pr):
        """lm value of the prefix's partial word given its context, None if the partial word is not in V"""
        if pr not in info:
            words, part = D.split(pr)
            info[pr] = (lm.lm(D.word_of[part], lm.context(words)) if part in D.word_of else None, part)
        return info[pr]

    def a(v):
        return alpha * v + beta

    rec = {}
    pre = [()]
    lb = np.array([0.0])
    lnb = np.array([NEG])
    margin = math.inf

    def note(x, m):
        nonlocal margin
        d = abs(x - m)
        if d == d:
            margin = min(margin, d)

    for t in range(n):
        p = probs[t].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            lp = np.log(p)
        K, m3 = BO.kept_chars(probs[t], cutoff_top_n, cutoff_prob)
        margin = min(margin, m3)
        inK = np.zeros(C, dtype=bool)
        inK[K] = True
        Knb = np.array([c for c in K if c != blank], dtype=np.int64)
        L = len(pre)
        sc = BO._lse_vec(lb, lnb)
        full = L == W
        m = float(sc[L - 1] + lp[blank] - max(0.0, beta)) if full else NEG
        slot = {pr: j for j, pr in enumerate(pre)}
        last = np.array([pr[-1] if pr else -1 for pr in pre], dtype=np.int64)
        sb = np.full(L, NEG)
        snb = np.full(L, NEG)
        listed_child = np.zeros((L, C), dtype=bool)
        for j, pr in enumerate(pre):
            if inK[blank]:
                v = lp[blank] + sc[j]
                if full and j != L - 1:
                    note(v, m)
                stats["l4_drops"] += bool(v < m)
                sb[j] = NEG if v < m else v
            if not pr:
                continue
            l = pr[-1]
            pi = slot.get(pr[:-1])
            if pi is not None:
                listed_child[pi, l] = True
            if not inK[l]:
                continue
            v = lp[l] + lnb[j]
            if full:
                note(lp[l] + sc[j], m)
            if lp[l] + sc[j] < m:
                v = NEG
                stats["l4_drops"] += 1
            if pi is not None:
                if full:
                    note(lp[l] + sc[pi], m)
                stats["l4_drops"] += bool(lp[l] + sc[pi] < m)
                if not (lp[l] + sc[pi] < m):
                    v2 = lp[l] + (lb[pi] if last[pi] == l else sc[pi])
                    if l == space:
                        v2 = v2 + a(lmv(pre[pi])[0])
                    v = BO.lse(v, v2)
                    r = rec[pr]
                    if lp[l] > r[1]:
                        rec[pr] = [t, lp[l]]
            snb[j] = v
        stay = BO._lse_vec(sb, snb)
        if len(Knb):
            base = np.where(Knb[None, :] == last[:, None], lb[:, None], sc[:, None])
            new = lp[Knb][None, :] + base
            ok = ~listed_child[:, Knb]
            for j, pr in enumerate(pre):
                part = lmv(pr)[1]
                for k, c in enumerate(Knb):
                    if ok[j, k] and not D.allowed(part, int(c)):
                        ok[j, k] = False
            cut = lp[Knb][None, :] + sc[:, None]
            if full:
                for d in np.abs(cut[ok] - m):
                    note(float(d), 0.0)
            stats["l4_drops"] += int(np.count_nonzero(ok & (cut < m)))
            ok &= ~(cut < m)
            ks = np.nonzero(Knb == space)[0]
            for k in ks:
                for j, pr in enumerate(pre):
                    if ok[j, k]:
                        new[j, k] = new[j, k] + a(lmv(pr)[0])
            new[~ok] = NEG
        else:
            new = np.zeros((L, 0))
        s_all = np.concatenate([stay, new.reshape(-1)])
        oi = np.concatenate([np.arange(L), np.repeat(np.arange(L), len(Knb))])
        oc = np.concatenate([np.full(L, -1), np.tile(Knb, L)])
        s_all = s_all + 0.0
        keep_ok = s_all > NEG
        s_all, oi, oc = s_all[keep_ok], oi[keep_ok], oc[keep_ok]
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
    sc = BO._lse_vec(lb, lnb)
    final = []
    for j, pr in enumerate(pre):
        f = float(sc[j])
        if pr and pr[-1] != space:
            v = lmv(pr)[0]
            f = f + a(LM_OOV if v is None else v)
        final.append(f)
    order = sorted(range(len(pre)), key=lambda j: (-final[j], j))
    fs = [final[j] for j in order]
    if len(fs) > 1:
        margin = min(margin, min(x - y for x, y in zip(fs[:-1], fs[1:])))
    beams = []
    for j in order:
        pr = pre[j]
        ts = [rec[pr[:k + 1]][0] for k in range(len(pr))]
        beams.append((list(pr), ts, -final[j] + 0.0))
    return beams, margin


def beam_decode_lm(probs, sizes, labels, lm: ArpaLM, alpha: float, beta: float, blank: int = 0,
                   beam_width: int = 100, cutoff_top_n: int = 40, cutoff_prob: float = 1.0,
                   stats: Optional[dict] = None):
    """(B, T, C) -> dict of arrays in the C-ABI's layout plus the smallest decision margin (beam_oracle.beam_decode
    with the language model)"""
    probs = np.asarray(probs.detach().cpu().numpy() if hasattr(probs, "detach") else probs, dtype=np.float32)
    B, T, C = probs.shape
    W = beam_width
    out = dict(labels=np.zeros((B, W, T), np.int32), timesteps=np.zeros((B, W, T), np.int32),
               lengths=np.zeros((B, W), np.int32), scores=np.full((B, W), math.inf), n_beams=np.zeros(B, np.int32))
    margin = math.inf
    for b in range(B):
        size = None if sizes is None else int(sizes[b])
        beams, m = beam_search_lm(probs[b], size, blank, W, cutoff_top_n, cutoff_prob, labels, lm, alpha, beta,
                                  stats=stats)
        margin = min(margin, m)
        out["n_beams"][b] = len(beams)
        for r, (lab, ts, s) in enumerate(beams):
            out["lengths"][b, r] = len(lab)
            out["labels"][b, r, :len(lab)] = lab
            out["timesteps"][b, r, :len(lab)] = ts
            out["scores"][b, r] = s
    out["margin"] = margin
    return out


def synthetic_arpa(path, n_words: int, order: int, counts: List[int], seed: int, alphabet: str = "ABCDEFGHIJKLMNOP",
                   max_len: int = 8, words: Optional[List[str]] = None, gz: bool = False) -> List[str]:
    """write a seeded random ARPA file: `words` (or n_words random distinct words over `alphabet`) plus <s>, </s>,
    <unk> as unigrams, counts[k] random distinct (k+2)-grams, Zipf-weighted, log10 p in [-5, -0.3], backoffs in
    [-1.5, 0] on every order but the last (every fifth one left unwritten).  Returns the unigram list in file order."""
    rng = np.random.default_rng(seed)
    if words is None:
        got, out = set(), []
        while len(out) < n_words:
            k = int(rng.integers(1, max_len + 1))
            w = ''.join(alphabet[int(x)] for x in rng.integers(0, len(alphabet), k))
            if w not in got:
                got.add(w)
                out.append(w)
        words = out
    uni = ["<s>", "</s>", "<unk>"] + list(words)
    V = len(uni)
    grams = [np.arange(V, dtype=np.int64)[:, None]]
    zipf = 1.0 / np.arange(1, V - 2) ** 0.9
    zipf /= zipf.sum()
    for k, cnt in enumerate(counts[:order - 1]):
        n = k + 2
        assert float(V) ** n < 2 ** 62
        draw = rng.choice(np.arange(3, V), size=(int(cnt * 1.3) + 16, n), p=zipf)
        draw[:, 0] = np.where(rng.random(len(draw)) < 0.1, 0, draw[:, 0])          # some n-grams start with <s>
        code = np.zeros(len(draw), np.int64)
        for q in range(n):
            code = code * V + draw[:, q]
        _, first = np.unique(code, return_index=True)
        first = np.sort(first)[:cnt]
        grams.append(draw[first])
    lines = ["", "\\data\\"] + [f"ngram {n + 1}={len(g)}" for n, g in enumerate(grams)]
    for n, g in enumerate(grams):
        lines += ["", f"\\{n + 1}-grams:"]
        lp = rng.uniform(-5.0, -0.3, len(g))
        bo = rng.uniform(-1.5, 0.0, len(g))
        has_bo = (n + 1 < order) & (rng.random(len(g)) >= 0.2)
        if n == 0:
            lp[0] = -99.0
        strs = [' '.join(uni[i] for i in row) for row in g.tolist()]
        for s, p, b, h in zip(strs, lp.tolist(), bo.tolist(), has_bo.tolist()):
            lines.append(f"{p:.6f}\t{s}\t{b:.6f}" if h else f"{p:.6f}\t{s}")
    lines += ["", "\\end\\", ""]
    data = '\n'.join(lines).encode()
    with open(path, "wb") as f:
        f.write(gzip.compress(data) if gz else data)
    return uni
