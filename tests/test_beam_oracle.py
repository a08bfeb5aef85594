"""CPU: the beam-search oracle (`oracle/beam_oracle.py`, row N5) against implementation-independent pins, and the
host side of `BeamCTCDecoder` / `load_decoder` / `LMConfig`.

- Exhaustive width: with W >= the number of feasible labellings, every feasible labelling comes out exactly once, its
  score is the float64 CTC negative log-likelihood (`O.ctc_loss_and_grad`) minus the per-frame normaliser
  sum_t log sum_c p_tc that fp32 inputs carry, and the top beam is the brute-force most probable labelling.
- Pruning to one character (cutoff_top_n = 1, or a tiny cutoff_prob) is greedy decoding (`O.greedy_path`).
- A prefix that leaves the list and returns keeps its node (timestep record) and restarts its probabilities."""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import beam_oracle as BO
from oracle import ds2_oracle as O

import deepspeech_pytorch_b200 as ds


def softmax_probs(rng, T, C, scale):
    lg = rng.standard_normal((T, C)) * scale
    return (np.exp(lg) / np.exp(lg).sum(-1, keepdims=True)).astype(np.float32)


def feasible_labellings(T, C, blank=0):
    """every label sequence (blank excluded) that fits T frames: n + #repeats <= T"""
    labs = set()
    chars = [c for c in range(C) if c != blank]
    for n in range(T + 1):
        for s in itertools.product(chars, repeat=n):
            if n + sum(s[i] == s[i + 1] for i in range(n - 1)) <= T:
                labs.add(s)
    return labs


@pytest.mark.parametrize("C,T,n_lab", [(3, 6, 41), (4, 4, 61), (5, 3, 57)])
@pytest.mark.parametrize("seed", [0, 1])
def test_exhaustive_width_is_the_ctc_likelihood_of_every_labelling(C, T, n_lab, seed):
    rng = np.random.default_rng(100 * C + T + seed)
    pr = softmax_probs(rng, T, C, 1.5)
    labs = feasible_labellings(T, C)
    assert len(labs) == n_lab
    beams, _ = BO.beam_search(pr, None, 0, 128, 40, 1.0)
    got = {tuple(lab): s for lab, _, s in beams}
    assert len(got) == len(beams), "a prefix is listed twice"
    assert set(got) == labs
    logZ = float(np.log(pr.astype(np.float64).sum(-1)).sum())
    lp = np.log(pr.astype(np.float64))[:, None, :]
    best = None
    for s in labs:
        nll, _ = O.ctc_loss_and_grad(lp, np.array(s, np.int64), [T], [len(s)], blank=0)
        want = float(nll[0]) - logZ
        assert abs(got[s] - want) <= 1e-12 * max(1.0, abs(want)), (s, got[s], want)
        if best is None or want < best[0]:
            best = (want, s)
    assert tuple(beams[0][0]) == best[1]
    assert [s for _, _, s in beams] == sorted(s for _, _, s in beams)


@pytest.mark.parametrize("top_n,cprob", [(1, 1.0), (40, 1e-9)])
@pytest.mark.parametrize("blank", [0, 28])
def test_pruning_to_one_character_is_greedy_decoding(top_n, cprob, blank):
    rng = np.random.default_rng(7 + blank)
    for _ in range(4):
        pr = softmax_probs(rng, 80, 29, 3.0)
        g_lab, g_off = O.greedy_path(torch.from_numpy(pr)[None], None, blank=blank)[0]
        beams, _ = BO.beam_search(pr, None, blank, 10, top_n, cprob)
        assert len(beams) == 1
        lab, ts, score = beams[0]
        assert lab == g_lab and ts == g_off
        want = -float(np.log(pr.astype(np.float64).max(-1)).sum())
        assert abs(score - want) <= 1e-12 * abs(want)


def test_a_prefix_that_leaves_and_returns_keeps_its_node():
    """C = 3 (blank 0, a = 1, b = 2), W = 2.  Frame 0 lists {'', a}; frame 1 lists {b, ''} (a drops out); frame 2
    extends the listed '' by a again: a returns with restarted probabilities and its frame-0 timestep."""
    pr = np.array([[0.5, 0.4, 0.1], [0.47, 0.03, 0.5], [0.1, 0.8, 0.1]], np.float32)
    trace = []
    beams, _ = BO.beam_search(pr, None, 0, 2, 40, 1.0, trace=trace)
    lists = [[p for p, _, _ in fr] for fr in trace]
    for fr in lists:
        assert len(set(fr)) == len(fr)
    assert lists[0] == [(), (1,)]
    assert lists[1] == [(2,), ()]
    assert lists[2] == [(2, 1), (1,)]
    lp = np.log(pr.astype(np.float64))
    _, b_empty, nb_empty = trace[1][1]
    _, b_a, nb_a = trace[2][1]
    assert b_a == -math.inf and nb_a == lp[2, 1] + BO.lse(b_empty, nb_empty)    # restarted, no frame-0 mass
    assert beams[1][0] == [1] and beams[1][1] == [0]                            # record of frame 0 kept
    assert beams[0][0] == [2, 1] and beams[0][1] == [1, 2]


def test_timestep_moves_to_a_larger_extension_of_the_listed_parent():
    """a at frame 0 (p = 0.5); frame 1 is mostly blank, so '' and a stay listed; at frame 2 the listed '' is extended
    by a with p = 0.9 > 0.5 while a is listed: a's record moves to frame 2"""
    pr = np.array([[0.3, 0.5, 0.2], [0.8, 0.1, 0.1], [0.05, 0.9, 0.05]], np.float32)
    trace = []
    beams, _ = BO.beam_search(pr, None, 0, 3, 40, 1.0, trace=trace)
    assert (1,) in [p for p, _, _ in trace[1]] and () in [p for p, _, _ in trace[1]]
    rec = {tuple(lab): ts for lab, ts, _ in beams}
    assert rec[(1,)] == [2]


def test_pruned_blank_contributes_nothing():
    """cutoff_top_n = 2 with the blank third at frame 1: the same result as a zero blank probability there, and no
    listed prefix ends in blank after that frame"""
    pr = np.array([[0.5, 0.3, 0.15, 0.05], [0.2, 0.42, 0.38, 0.0], [0.6, 0.2, 0.1, 0.1]], np.float32)
    trace = []
    beams, _ = BO.beam_search(pr, None, 0, 8, 2, 1.0, trace=trace)
    assert all(b == -math.inf for _, b, _ in trace[1])
    z = pr.copy()
    z[1, 0] = 0.0
    beams_z, _ = BO.beam_search(z, None, 0, 8, 2, 1.0)
    assert beams == beams_z


def test_sizes_zero_ragged_and_fewer_than_w():
    rng = np.random.default_rng(3)
    pr = np.stack([softmax_probs(rng, 12, 5, 1.0) for _ in range(3)])
    out = BO.beam_decode(pr, [12, 4, 0], blank=0, beam_width=6, cutoff_top_n=40, cutoff_prob=1.0)
    assert out["n_beams"][2] == 1 and out["lengths"][2, 0] == 0 and out["scores"][2, 0] == 0.0
    assert np.all(out["scores"][2, 1:] == math.inf) and np.all(out["lengths"][2, 1:] == 0)
    ragged, _ = BO.beam_search(pr[1, :4], None, 0, 6, 40, 1.0)
    assert out["n_beams"][1] == len(ragged)
    for r, (lab, ts, s) in enumerate(ragged):
        n = out["lengths"][1, r]
        assert out["labels"][1, r, :n].tolist() == lab and out["timesteps"][1, r, :n].tolist() == ts
        assert out["scores"][1, r] == s
    # one frame over {blank, a, b}: '', a, b -- three prefixes for W = 10
    one, _ = BO.beam_search(np.array([[0.2, 0.5, 0.3]], np.float32), None, 0, 10, 40, 1.0)
    assert [lab for lab, _, _ in one] == [[1], [2], []]


def test_lm_config_defaults_mirror_the_reference():
    c = ds.LMConfig()
    assert c.decoder_type == ds.DecoderType.greedy and c.lm_path == '' and c.top_paths == 1
    assert (c.alpha, c.beta, c.cutoff_top_n, c.cutoff_prob, c.beam_width, c.lm_workers) == (0.0, 0.0, 40, 1.0, 10, 4)


def test_load_decoder_dispatch_and_lm_path_refused():
    g = ds.load_decoder(ds.LABELS, ds.LMConfig())
    assert isinstance(g, ds.GreedyDecoder) and g.blank_index == ds.LABELS.index('_')
    b = ds.load_decoder(ds.LABELS, ds.LMConfig(decoder_type=ds.DecoderType.beam, beam_width=7, cutoff_top_n=5,
                                               cutoff_prob=0.9, alpha=0.5, beta=1.0))
    assert isinstance(b, ds.BeamCTCDecoder)
    assert (b.beam_width, b.cutoff_top_n, b.cutoff_prob, b.blank_index) == (7, 5, 0.9, ds.LABELS.index('_'))
    d = ds.BeamCTCDecoder(ds.LABELS)
    assert (d.beam_width, d.cutoff_top_n, d.cutoff_prob, d.blank_index) == (100, 40, 1.0, 0)
    with pytest.raises(ds.Ds2Error, match="language-model scoring"):
        ds.BeamCTCDecoder(ds.LABELS, lm_path="lm.binary")
    with pytest.raises(ds.Ds2Error, match="language-model scoring"):
        ds.load_decoder(ds.LABELS, ds.LMConfig(decoder_type=ds.DecoderType.beam, lm_path="x.arpa"))


@pytest.mark.parametrize("sizes", [[5, 5], [5, 5, 5, 5], [[5, 5, 5]]])
def test_sizes_must_hold_one_length_per_utterance(sizes):
    """the kernel reads sizes[b] for every utterance: a shorter (or longer, or 2-D) `sizes` is refused before any
    device work"""
    with pytest.raises(ds.Ds2Error, match="one length per utterance"):
        ds.BeamCTCDecoder(ds.LABELS).decode_beams(torch.full((3, 5, 29), 1 / 29), sizes)
