"""CTC forced alignment in NumPy float64: the Viterbi recursion `ds2_ctc_align` (include/ds2_b200.h) is specified by.

Extended sequence of S = 2L+1 states (blank, y1, blank, ..., yL, blank).  Scores are float64:
    score_t(s) = max(score_{t-1}(s), score_{t-1}(s-1), score_{t-1}(s-2)) + float64(lp[t][ext[s]])
where s-2 counts only if ext[s] != blank and ext[s] != ext[s-2].  At t = 0 only states 0 and 1 are live.  Ties
prefer s, then s-1, then s-2.  The path ends in S-1 if score(S-1) >= score(S-2), otherwise in S-2.  The same
operations in the same order as the kernel, so the two agree bit for bit on the same fp32 log-probs."""
import numpy as np

NEG_INF = -np.inf


def ctc_align(lp, target, blank=0):
    """lp (T, C) log-probs of one utterance (only its own frames), target: sequence of label ids.
    -> dict(labels (T,) int64, frame_log_probs (T,) float64, spans (L, 2) int64 [start, end), score float,
            final (score(S-1), score(S-2)) as floats).
    An utterance without a finite path gets score -inf, labels -1 and spans -1; T = 0 gives score 0 for an empty
    target and -inf otherwise."""
    lp = np.asarray(lp)
    T = lp.shape[0]
    target = [int(c) for c in target]
    L = len(target)
    S = 2 * L + 1
    ext = np.full(S, blank, dtype=np.int64)
    ext[1::2] = target
    skip = np.zeros(S, dtype=bool)
    if S > 2:
        skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])

    def infeasible(score=NEG_INF):
        return dict(labels=np.full(T, -1, np.int64), frame_log_probs=np.zeros(T), spans=np.full((L, 2), -1, np.int64),
                    score=float(score), final=(NEG_INF, NEG_INF))

    if T == 0:
        return infeasible(0.0 if L == 0 else NEG_INF)
    bp = np.zeros((T, S), dtype=np.int8)
    cur = np.full(S, NEG_INF)
    cur[:2] = lp[0, ext[:2]].astype(np.float64)
    for t in range(1, T):
        prev = np.concatenate([[NEG_INF, NEG_INF], cur])
        best = prev[2:].copy()
        d = np.zeros(S, dtype=np.int8)
        c1 = prev[1:-1]
        m = c1 > best
        best[m], d[m] = c1[m], 1
        c2 = np.where(skip, prev[:-2], NEG_INF)
        m = c2 > best
        best[m], d[m] = c2[m], 2
        cur = best + lp[t, ext].astype(np.float64)
        bp[t] = d
    last = float(cur[S - 1])
    second = float(cur[S - 2]) if S > 1 else NEG_INF
    s = S - 1 if (S == 1 or last >= second) else S - 2
    score = float(cur[s])
    if not score > NEG_INF:
        return infeasible()
    states = np.empty(T, np.int64)
    for t in range(T - 1, -1, -1):
        states[t] = s
        s -= int(bp[t, s])
    labels = ext[states]
    spans = np.full((L, 2), -1, np.int64)
    for t in range(T):
        s = states[t]
        if s & 1:
            k = s >> 1
            if spans[k, 0] < 0:
                spans[k, 0] = t
            spans[k, 1] = t + 1
    return dict(labels=labels, frame_log_probs=lp[np.arange(T), labels].astype(np.float64), spans=spans, score=score,
                final=(last, second))


def collapse(labels, blank=0):
    """the CTC collapse of a frame-label path: merge repeats, drop blanks (and the -1 padding)"""
    out, prev = [], None
    for c in labels:
        c = int(c)
        if c != prev and c != blank and c >= 0:
            out.append(c)
        prev = c
    return out
