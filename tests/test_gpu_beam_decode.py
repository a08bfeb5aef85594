"""-m gpu: `ds2_beam_decode` / `BeamCTCDecoder` (row N5) against the float64 oracle `oracle/beam_oracle.py`.

Exact comparison: n_beams, the order of each list, labels, lengths and timesteps are equal, and scores agree within
1e-10 relative.  Each seeded case also asserts that the oracle's smallest decision margin (the score gap at every
comparison that decided membership or order, and the distance of every cumulative sum from cutoff_prob) is above
1e-8, so that exact equality is a fair demand of two fp64 implementations whose logs and exps round differently.
Inputs are peaked, alignment-like rows (a label run plus noise) and flat ones (softmax of 0.3 N(0,1), where every
prefix branches and the W-th and (W+1)-th candidates are closest)."""
import numpy as np
import pytest
import torch

from oracle import beam_oracle as BO
from oracle import ds2_oracle as O

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.metrics import WordErrorRate

pytestmark = pytest.mark.gpu

DEV = "cuda"


def peaked_probs(B, T, C, blank, seed):
    rng = np.random.default_rng(seed)
    lab = np.zeros((B, T), np.int64)
    for b in range(B):
        t = 0
        while t < T:
            c = blank if rng.random() < 0.3 else int(rng.integers(0, C))
            n = int(rng.integers(1, 5))
            lab[b, t:t + n] = c
            t += n
    lg = rng.standard_normal((B, T, C)) * 0.5 + 6.0 * np.eye(C)[lab]
    e = np.exp(lg - lg.max(-1, keepdims=True))
    return torch.from_numpy((e / e.sum(-1, keepdims=True)).astype(np.float32))


def flat_probs(B, T, C, seed):
    lg = np.random.default_rng(seed).standard_normal((B, T, C)) * 0.3
    e = np.exp(lg)
    return torch.from_numpy((e / e.sum(-1, keepdims=True)).astype(np.float32))


def assert_equal_to_oracle(got, ref, what=""):
    labels, scores, timesteps, lengths, n_beams = got
    assert n_beams.tolist() == ref["n_beams"].tolist(), what
    assert torch.equal(lengths, torch.from_numpy(ref["lengths"])), what
    assert torch.equal(labels, torch.from_numpy(ref["labels"])), what
    assert torch.equal(timesteps, torch.from_numpy(ref["timesteps"])), what
    s, r = scores.numpy(), ref["scores"]
    assert np.array_equal(np.isinf(s), np.isinf(r)), what
    f = np.isfinite(r)
    assert np.all(np.abs(s[f] - r[f]) <= 1e-10 * np.maximum(1.0, np.abs(r[f]))), what


CASES = [  # id, kind, B, T, C, blank, W, cutoff_top_n, cutoff_prob, sizes
    ("peaked_c29_w10_ragged", "peaked", 8, 300, 29, 0, 10, 40, 1.0, [300, 299, 250, 180, 97, 31, 1, 0]),
    ("peaked_c29_blank28_w100", "peaked", 4, 200, 29, 28, 100, 40, 1.0, None),
    ("peaked_c29_w128_top5_cp095", "peaked", 4, 200, 29, 0, 128, 5, 0.95, [200, 150, 60, 0]),
    ("peaked_c64_blank63_w100_cp095", "peaked", 3, 150, 64, 63, 100, 40, 0.95, None),
    ("peaked_c29_w1", "peaked", 4, 300, 29, 0, 1, 40, 1.0, [300, 211, 5, 0]),
    ("peaked_c29_w10_top1", "peaked", 4, 300, 29, 0, 10, 1, 1.0, None),
    ("flat_c29_w100", "flat", 2, 100, 29, 0, 100, 40, 1.0, [100, 37]),
    ("flat_c29_blank28_w10_cp095", "flat", 4, 200, 29, 28, 10, 40, 0.95, None),
    ("flat_c29_w128_top5", "flat", 2, 150, 29, 0, 128, 5, 1.0, [150, 0]),
    ("flat_c64_w128", "flat", 2, 60, 64, 0, 128, 40, 1.0, None),
    ("flat_c64_w100_top5", "flat", 2, 120, 64, 0, 100, 5, 1.0, [120, 64]),
]


def case_probs(kind, B, T, C, blank, seed):
    return peaked_probs(B, T, C, blank, seed) if kind == "peaked" else flat_probs(B, T, C, seed)


@pytest.mark.parametrize("tag,kind,B,T,C,blank,W,top_n,cprob,sizes", CASES, ids=[c[0] for c in CASES])
def test_beam_decode_equals_oracle(tag, kind, B, T, C, blank, W, top_n, cprob, sizes):
    probs = case_probs(kind, B, T, C, blank, seed=T + C + W)
    ref = BO.beam_decode(probs, sizes, blank=blank, beam_width=W, cutoff_top_n=top_n, cutoff_prob=cprob)
    assert ref["margin"] > 1e-8, f"{tag}: knife-edge input (oracle decision margin {ref['margin']:.3g})"
    dec = ds.BeamCTCDecoder(ds.LABELS, beam_width=W, cutoff_top_n=top_n, cutoff_prob=cprob, blank_index=blank)
    got = dec.decode_beams(probs.to(DEV), None if sizes is None else torch.tensor(sizes))
    assert_equal_to_oracle(got, ref, tag)
    if W > 1 and top_n > 1:
        assert int(got[4].max()) > 1, f"{tag}: the search never branched"


def test_top_n_1_at_t20000_is_greedy_decoding():
    """cutoff_top_n = 1 over 20000 frames (node pool of 80001 nodes per utterance) equals GreedyDecoder exactly"""
    B, T, C = 3, 20000, 29
    sizes = torch.tensor([20000, 13001, 0])
    rng = np.random.default_rng(T)
    lab = np.zeros((B, T), np.int64)
    for b in range(B):
        t = 0
        while t < T:
            c = 0 if rng.random() < 0.3 else int(rng.integers(0, C))
            n = int(rng.integers(1, 5))
            lab[b, t:t + n] = c
            t += n
    lg = torch.from_numpy(rng.standard_normal((B, T, C))).float() * 0.5 + 6.0 * torch.nn.functional.one_hot(
        torch.from_numpy(lab), C).float()
    probs = torch.softmax(lg, -1).to(DEV)
    g_lab, g_off, g_cnt = ds.GreedyDecoder(ds.LABELS).decode_indices(probs, sizes)
    labels, scores, timesteps, lengths, n_beams = ds.BeamCTCDecoder(ds.LABELS, beam_width=4, cutoff_top_n=1
                                                                    ).decode_beams(probs, sizes)
    assert n_beams.tolist() == [1, 1, 1]
    assert torch.equal(lengths[:, 0], g_cnt) and int(g_cnt[0]) > 1000
    assert torch.equal(labels[:, 0], g_lab) and torch.equal(timesteps[:, 0], g_off)
    assert bool((scores[:, 1:] == float("inf")).all()) and float(scores[2, 0]) == 0.0


def test_repeated_calls_are_bit_identical():
    probs = flat_probs(6, 200, 29, seed=11).to(DEV)
    dec = ds.BeamCTCDecoder(ds.LABELS, beam_width=100)
    a = dec.decode_beams(probs, [200, 190, 150, 100, 20, 0])
    b = dec.decode_beams(probs, [200, 190, 150, 100, 20, 0])
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_cpu_and_non_contiguous_inputs():
    probs = peaked_probs(3, 80, 29, 0, seed=5)
    dec = ds.BeamCTCDecoder(ds.LABELS, beam_width=10)
    ref = dec.decode_beams(probs.to(DEV))
    for x in (probs, probs.transpose(0, 1).contiguous().to(DEV).transpose(0, 1)):
        got = dec.decode_beams(x)
        for p, q in zip(got, ref):
            assert torch.equal(p, q)
    strings, offsets = dec.decode(probs)
    assert len(strings) == 3 and all(len(s) == 10 for s in strings)
    assert strings[0][0] == ''.join(ds.LABELS[int(c)] for c in ref[0][0, 0, :int(ref[3][0, 0])])
    assert torch.equal(offsets[1][0], ref[2][1, 0, :int(ref[3][1, 0])])


def test_fewer_prefixes_than_beams_leave_empty_slots():
    probs = torch.tensor([[[0.2, 0.5, 0.3]]]).to(DEV)
    dec = ds.BeamCTCDecoder(['_', 'a', 'b'], beam_width=10)
    labels, scores, timesteps, lengths, n_beams = dec.decode_beams(probs)
    assert int(n_beams[0]) == 3 and lengths[0].tolist() == [1, 1, 0] + [0] * 7
    assert bool((scores[0, 3:] == float("inf")).all())
    strings, offsets = dec.decode(probs)
    assert strings == [['a', 'b', ''] + [''] * 7] and offsets[0][5].numel() == 0


@pytest.mark.parametrize("kw,shape", [
    (dict(beam_width=0), (1, 10, 29)), (dict(beam_width=129), (1, 10, 29)), (dict(cutoff_top_n=0), (1, 10, 29)),
    (dict(cutoff_prob=0.0), (1, 10, 29)), (dict(cutoff_prob=1.5), (1, 10, 29)), (dict(blank_index=29), (1, 10, 29)),
    (dict(blank_index=-1), (1, 10, 29)), (dict(), (1, 10, 65)), (dict(), (1, 10, 1)), (dict(), (1, 0, 29)),
])
def test_bound_violations_raise(kw, shape):
    dec = ds.BeamCTCDecoder(ds.LABELS, **kw)
    with pytest.raises(ds.Ds2Error, match="ds2_beam_decode"):
        dec.decode_beams(torch.full(shape, 0.5, device=DEV))


def test_deepspeech_eval_output_end_to_end():
    """a small DeepSpeech in eval mode: its softmax output, decoded by BeamCTCDecoder(beam_width=10), equals the
    oracle run on the same tensor; WordErrorRate accumulates with the beam decoder"""
    torch.manual_seed(0)
    cfg = ds.BiDirectionalConfig(rnn_type=ds.RNNType.lstm, hidden_size=64, hidden_layers=2)
    model = ds.DeepSpeech(ds.LABELS, cfg, 32, ds.AdamConfig(), ds.SpectConfig()).to(DEV).eval()
    x, targets, pct, tsz = O.synth_batch(B=4, T=200, seed=3, lmin=5, lmax=12)
    lengths = (pct * x.size(3)).int()
    with torch.no_grad():
        out, out_sizes, _ = model(x.to(DEV), lengths)
    assert not out.is_contiguous()                       # forward() returns a transposed (B, T, C) view
    dec = ds.BeamCTCDecoder(ds.LABELS, beam_width=10)
    got = dec.decode_beams(out, out_sizes)
    ref = BO.beam_decode(out.cpu(), out_sizes.cpu(), blank=0, beam_width=10, cutoff_top_n=40, cutoff_prob=1.0)
    assert_equal_to_oracle(got, ref, f"eval output (oracle margin {ref['margin']:.3g})")
    wer = WordErrorRate(dec, ds.GreedyDecoder(ds.LABELS))
    wer.update(out, out_sizes, targets, tsz)
    wer.update(out, out_sizes, targets, tsz)
    assert int(wer.n_tokens) > 0 and np.isfinite(float(wer.compute()))
