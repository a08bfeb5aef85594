"""-m gpu: `ds2_beam_decode_lm` / `BeamCTCDecoder(lm_path=...)` (row N6) against the float64 oracle
`oracle/lm_oracle.py`.

Exact comparison as in test_gpu_beam_decode.py: n_beams, order, labels, lengths and timesteps equal, scores within
1e-10 relative, and each case asserts an oracle decision margin above 1e-8 (now including every full-beam filter
comparison and the end-of-utterance reorder).  Models are seeded synthetic ARPA files over a few letters of LABELS,
dense enough that most extensions are words or word prefixes."""
import numpy as np
import pytest
import torch

from oracle import lm_oracle as LO

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.metrics import WordErrorRate
from test_gpu_beam_decode import assert_equal_to_oracle, flat_probs

pytestmark = pytest.mark.gpu

DEV = "cuda"
ALPHA = "ABCDE'"
SPACE = ds.LABELS.index(' ')


def model_file(tmp_path_factory, order, seed, n_words=150):
    counts = [400, 500, 300, 300][:order - 1]
    p = str(tmp_path_factory.mktemp("lm") / f"o{order}_s{seed}.arpa")
    LO.synthetic_arpa(p, n_words, order, counts, seed=seed, alphabet=ALPHA, max_len=4)
    return p


def peaked_lm_probs(B, T, seed):
    """alignment-like rows over the model's letters, the space and the blank"""
    rng = np.random.default_rng(seed)
    chars = [0, SPACE] + [ds.LABELS.index(c) for c in ALPHA]
    lab = np.zeros((B, T), np.int64)
    for b in range(B):
        t = 0
        while t < T:
            c = 0 if rng.random() < 0.3 else chars[int(rng.integers(0, len(chars)))]
            n = int(rng.integers(1, 5))
            lab[b, t:t + n] = c
            t += n
    lg = rng.standard_normal((B, T, 29)) * 0.5 + 4.0 * np.eye(29)[lab]
    e = np.exp(lg - lg.max(-1, keepdims=True))
    return torch.from_numpy((e / e.sum(-1, keepdims=True)).astype(np.float32))


CASES = [  # id, kind, B, T, W, order, alpha, beta, top_n, cprob, sizes
    ("peaked_w10_o3", "peaked", 6, 120, 10, 3, 0.8, 1.5, 40, 1.0, [120, 119, 80, 31, 1, 0]),
    ("peaked_w100_o2_a0", "peaked", 3, 100, 100, 2, 0.0, -1.0, 40, 1.0, None),
    ("peaked_w128_o5_top5_cp095", "peaked", 3, 100, 128, 5, 2.5, 0.0, 5, 0.95, [100, 64, 0]),
    ("peaked_w1_o1", "peaked", 3, 120, 1, 1, 0.8, 0.0, 40, 1.0, [120, 50, 0]),
    ("peaked_w10_o4_b_neg", "peaked", 4, 120, 10, 4, 2.5, -1.0, 40, 0.95, None),
    ("flat_w100_o3", "flat", 2, 60, 100, 3, 0.8, 1.5, 40, 1.0, [60, 37]),
    ("flat_w10_o2_top12", "flat", 3, 80, 10, 2, 2.5, 1.5, 12, 1.0, None),
    ("flat_w128_o5", "flat", 2, 50, 128, 5, 0.0, 0.0, 40, 1.0, [50, 0]),
]


@pytest.mark.parametrize("tag,kind,B,T,W,order,alpha,beta,top_n,cprob,sizes", CASES, ids=[c[0] for c in CASES])
def test_beam_decode_lm_equals_oracle(tmp_path_factory, tag, kind, B, T, W, order, alpha, beta, top_n, cprob,
                                      sizes):
    path = model_file(tmp_path_factory, order, seed=order + W)
    probs = peaked_lm_probs(B, T, seed=T + W) if kind == "peaked" else flat_probs(B, T, 29, seed=T + W)
    lm = LO.read_arpa(path)
    stats = {}
    ref = LO.beam_decode_lm(probs, sizes, ds.LABELS, lm, alpha, beta, blank=0, beam_width=W, cutoff_top_n=top_n,
                            cutoff_prob=cprob, stats=stats)
    assert ref["margin"] > 1e-8, f"{tag}: knife-edge input (oracle decision margin {ref['margin']:.3g})"
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=path, alpha=alpha, beta=beta, beam_width=W, cutoff_top_n=top_n,
                            cutoff_prob=cprob)
    got = dec.decode_beams(probs.to(DEV), None if sizes is None else torch.tensor(sizes))
    assert_equal_to_oracle(got, ref, tag)
    if kind == "peaked" and W >= 10:
        assert stats["l4_drops"] > 0, f"{tag}: the full-beam filter never fired"
    if top_n > 5:
        assert W == 1 or int(got[4].max()) > 1
        words = [''.join(ds.LABELS[c] for c in got[0][b, 0, :int(got[3][b, 0])]).split() for b in range(B)]
        assert any(words), f"{tag}: no words decoded"
    else:       # the blank and every admissible character pruned in some frame: the list empties (rule 5)
        assert int(got[4].min()) == 0


def test_recovers_the_transcript_where_greedy_and_no_lm_beam_make_non_words(tmp_path):
    """each letter of the transcript is acoustically confused with the next letter of the alphabet (p 0.45 against
    0.40), so greedy and beam search without a language model spell non-words; the dictionary constraint and the
    model bring back the transcript"""
    words = ["THE", "CAT", "SAT", "ON", "A", "MAT", "DOG", "RAN"]
    p = str(tmp_path / "rec.arpa")
    LO.synthetic_arpa(p, 0, 2, [20], seed=5, words=words)
    text = ["THE CAT SAT ON A MAT", "A DOG RAN ON THE MAT"]
    C = 29
    rows = []
    for s in text:
        fr = []
        for ch in s:
            if ch == ' ':
                v = np.full(C, 0.1 / 27)
                v[SPACE], v[0] = 0.85, 0.05
                fr.append(v)
                continue
            c = ds.LABELS.index(ch)
            conf = ds.LABELS.index(chr((ord(ch) - ord('A') + 1) % 26 + ord('A')))
            v = np.full(C, 0.05 / 26)
            v[c], v[conf], v[0] = 0.40, 0.45, 0.10
            v = v / v.sum()
            b = np.full(C, 0.1 / 28)
            b[0] = 0.9
            fr += [v, v, b]
        rows.append(np.array(fr))
    T = max(len(r) for r in rows)
    probs = np.zeros((2, T, C), np.float32)
    probs[:, :, 0] = 1.0
    for k, r in enumerate(rows):
        probs[k, :len(r)] = r
    probs = torch.from_numpy(probs).to(DEV)
    sizes = torch.tensor([len(r) for r in rows])
    targets = torch.tensor([ds.LABELS.index(ch) for s in text for ch in s])
    tsz = torch.tensor([len(s) for s in text])
    greedy = ds.GreedyDecoder(ds.LABELS)
    nolm = ds.BeamCTCDecoder(ds.LABELS, beam_width=20)
    withlm = ds.BeamCTCDecoder(ds.LABELS, lm_path=p, alpha=0.5, beta=1.0, beam_width=20)
    assert [s[0] for s in withlm.decode(probs, sizes)[0]] == text
    for d in (greedy, nolm):
        assert all(s[0] != t for s, t in zip(d.decode(probs, sizes)[0], text))
    wers = []
    for d in (greedy, nolm, withlm):
        w = WordErrorRate(d, greedy)
        w.update(probs, sizes, targets, tsz)
        wers.append(w.compute())
    assert wers[2] == 0.0 and wers[0] >= 50.0 and wers[1] >= 50.0, wers


def test_repeated_calls_alternating_models_and_inputs(tmp_path_factory):
    """repeated calls are bit-identical; two decoders with different models used alternately each give their own
    result; CPU and non-contiguous probs are accepted"""
    a = ds.BeamCTCDecoder(ds.LABELS, lm_path=model_file(tmp_path_factory, 3, seed=1), alpha=0.8, beta=1.0,
                          beam_width=64)
    b = ds.BeamCTCDecoder(ds.LABELS, lm_path=model_file(tmp_path_factory, 2, seed=2), alpha=1.5, beta=0.5,
                          beam_width=64)
    probs = peaked_lm_probs(4, 150, seed=9)
    sizes = [150, 140, 60, 0]
    ra = a.decode_beams(probs.to(DEV), sizes)
    rb = b.decode_beams(probs.to(DEV), sizes)
    assert not all(torch.equal(x, y) for x, y in zip(ra, rb))
    for _ in range(2):
        for dec, ref in ((a, ra), (b, rb)):
            for x in (probs, probs.to(DEV), probs.transpose(0, 1).contiguous().to(DEV).transpose(0, 1)):
                got = dec.decode_beams(x, sizes)
                for p, q in zip(got, ref):
                    assert torch.equal(p, q)
    a.reset_params(0.0, 0.0)
    r0 = a.decode_beams(probs, sizes)
    assert not torch.equal(r0[1], ra[1])
