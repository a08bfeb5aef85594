"""-m gpu: `ds2_beam_decode_lm_grid` (many (alpha, beta) pairs per launch) against per-pair `ds2_beam_decode_lm`
decodes, exactly; `ds2_error_counts` against `metrics.py`'s string edit distances, exactly."""
import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.evaluation import error_counts
from deepspeech_pytorch_b200.metrics import edit_distance
from test_gpu_beam_decode import flat_probs
from test_gpu_beam_decode_lm import SPACE, model_file, peaked_lm_probs

pytestmark = pytest.mark.gpu

DEV = "cuda"


def pairs_of(K, seed):
    """K pairs with beta < 0 and beta > 0 (the full-beam filter's max(0, beta)) and alpha = 0 among them"""
    rng = np.random.default_rng(seed)
    p = np.stack([rng.uniform(0.0, 3.0, K), rng.uniform(-1.5, 2.0, K)], 1)
    p[0] = (0.8, 1.5)
    if K > 1:
        p[1] = (2.5, -1.0)
    if K > 2:
        p[2] = (0.0, 0.0)
    return [tuple(map(float, r)) for r in p]


def per_pair(dec, probs, sizes, pairs):
    out = []
    for a, b in pairs:
        dec.reset_params(a, b)
        labels, _, _, lengths, _ = dec.decode_beams(probs, sizes)
        out.append((labels[:, 0], lengths[:, 0]))
    return out


def assert_grid_equals(got, ref, tag):
    labels, lengths = got[0].cpu(), got[1].cpu()
    for k, (lab, ln) in enumerate(ref):
        assert torch.equal(lengths[k], ln), f"{tag}: pair {k}: lengths differ"
        assert torch.equal(labels[k], lab), f"{tag}: pair {k}: labels differ"


GRID = [  # id, kind, B, T, W, order, top_n, cprob, sizes, K
    ("peaked_w10_o3_k3", "peaked", 6, 120, 10, 3, 40, 1.0, [120, 119, 80, 31, 1, 0], 3),
    ("peaked_w100_o2_k1", "peaked", 3, 100, 100, 2, 40, 1.0, None, 1),
    ("peaked_w128_o5_top5_cp095_k3", "peaked", 3, 100, 128, 5, 5, 0.95, [100, 64, 0], 3),
    ("peaked_w1_o1_k40", "peaked", 3, 120, 1, 1, 40, 1.0, [120, 50, 0], 40),
    ("peaked_w10_o4_cp095_k40_loops", "peaked", 8, 120, 10, 4, 40, 0.95, [120, 118, 100, 90, 77, 40, 3, 0], 40),
    ("flat_w100_o3_k3", "flat", 2, 60, 100, 3, 40, 1.0, [60, 37], 3),
    ("flat_w10_o2_top12_k40", "flat", 3, 80, 10, 2, 12, 1.0, None, 40),
    ("flat_w128_o5_k1", "flat", 2, 50, 128, 5, 40, 1.0, [50, 0], 1),
]


@pytest.mark.parametrize("tag,kind,B,T,W,order,top_n,cprob,sizes,K", GRID, ids=[c[0] for c in GRID])
def test_grid_equals_per_pair_decodes(tmp_path_factory, tag, kind, B, T, W, order, top_n, cprob, sizes, K):
    path = model_file(tmp_path_factory, order, seed=order + W)
    probs = (peaked_lm_probs(B, T, seed=T + W) if kind == "peaked" else flat_probs(B, T, 29, seed=T + W)).to(DEV)
    sz = None if sizes is None else torch.tensor(sizes)
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=path, beam_width=W, cutoff_top_n=top_n, cutoff_prob=cprob)
    pairs = pairs_of(K, seed=K + W)
    got = dec.decode_best_grid(probs, sz, pairs)
    assert tuple(got[0].shape) == (K, B, T) and tuple(got[1].shape) == (K, B)
    if "loops" in tag:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert B * K > 2 * sms, "this case must make CTAs run several items"
    ref = per_pair(dec, probs, sz, pairs)
    assert_grid_equals(got, ref, tag)
    # labels are zero after each length
    L = got[0].cpu()
    pos = torch.arange(T)[None, None]
    assert int(L.masked_select(pos >= got[1].cpu()[..., None]).abs().sum()) == 0


def test_grid_permutation_and_repeatability(tmp_path_factory):
    path = model_file(tmp_path_factory, 3, seed=13)
    probs = peaked_lm_probs(12, 140, seed=4).to(DEV)
    sizes = torch.tensor([140, 139, 130, 120, 110, 100, 90, 80, 60, 40, 10, 0])
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=path, beam_width=32)
    pairs = pairs_of(23, seed=5)
    a = dec.decode_best_grid(probs, sizes, pairs)
    b = dec.decode_best_grid(probs, sizes, pairs)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    perm = np.random.default_rng(0).permutation(len(pairs))
    c = dec.decode_best_grid(probs, sizes, [pairs[i] for i in perm])
    assert torch.equal(c[0], a[0][perm]) and torch.equal(c[1], a[1][perm])
    one = [dec.decode_best_grid(probs, sizes, [p]) for p in pairs[:4]]
    for k in range(4):
        assert torch.equal(one[k][0][0], a[0][k]) and torch.equal(one[k][1][0], a[1][k])


# ------------------------------------------------------------------------------------------------ counts
def string_counts(hyp, ref, labels, blank=0):
    """what metrics.CharErrorRate / WordErrorRate accumulate for one (hypothesis, reference) pair"""
    h = ''.join(labels[x] for x in hyp)
    r = ''.join(labels[x] for x in ref if x != blank)
    return [edit_distance(h.replace(' ', ''), r.replace(' ', '')), len(r.replace(' ', '')),
            edit_distance(h.split(), r.split()), len(r.split())]


def run_counts(hyps, refs, labels, K=1):
    """hyps: K*B label lists, refs: B label lists -> (rows (K,B,4), pairs (K,4)) from the device"""
    B = len(refs)
    T = max(1, max(len(h) for h in hyps))
    lab = torch.zeros(K, B, T, dtype=torch.int32)
    ln = torch.zeros(K, B, dtype=torch.int32)
    for i, h in enumerate(hyps):
        lab[i // B, i % B, :len(h)] = torch.tensor(h, dtype=torch.int32)
        ln[i // B, i % B] = len(h)
    targets = torch.tensor([x for r in refs for x in r], dtype=torch.int64)
    sizes = torch.tensor([len(r) for r in refs], dtype=torch.int32)
    space = labels.index(' ') if ' ' in labels else len(labels)
    pair = torch.zeros(K, 4, dtype=torch.int64, device=DEV)
    rows = error_counts(lab.to(DEV), ln.to(DEV), targets, sizes, 0, space, pair_counts=pair)
    return rows.cpu(), pair.cpu()


def test_counts_equal_metrics_on_random_rows():
    rng = np.random.default_rng(3)
    K, B = 3, 70
    alphabet = [SPACE, SPACE, 2, 3, 4, 5, 6]        # few letters: many equal and near-equal words
    refs = [rng.choice(alphabet + [0], int(rng.integers(0, 120))).tolist() for _ in range(B)]
    hyps = [rng.choice(alphabet, int(rng.integers(0, 150))).tolist() for _ in range(K * B)]
    rows, pair = run_counts(hyps, refs, ds.LABELS, K)
    for i, h in enumerate(hyps):
        assert rows[i // B, i % B].tolist() == string_counts(h, refs[i % B], ds.LABELS), i
    assert torch.equal(pair, rows.sum(1))


def test_counts_equal_metrics_on_edge_rows():
    L = ds.LABELS
    enc = lambda s: [L.index(c) for c in s]
    rng = np.random.default_rng(9)
    long_ref = rng.choice([SPACE] + list(range(2, 28)), 1100).tolist()
    long_hyp = rng.choice([SPACE] + list(range(2, 28)), 2000).tolist()
    huge_ref = rng.choice([SPACE, 2, 3, 4], 4500).tolist()         # over 64 x 64 symbols: the workspace path
    cases = [  # (hypothesis, reference)
        ([], []), ([], enc("THE CAT")), (enc("THE CAT"), []), (enc("   "), enc("A B")), (enc("A B"), enc("   ")),
        (enc("  THE  CAT "), enc("THE CAT")), (enc("THE CAT"), enc(" THE   CAT  ")), (enc(" "), enc(" ")),
        (enc("HELLO WORLD"), enc("HELLO WORLE")), (enc("HELLO WORLD"), enc("HELLP WORLD")),
        (enc("AB AB AB"), enc("AB ABC AB")), (enc("ABCD"), enc("ABCE")), (enc("THE_CAT"), enc("THE CAT")),
        (long_hyp, long_ref), (long_hyp[:600], huge_ref), (huge_ref[:3000], huge_ref),
        ([0, 2, 3], [0, 0, 2, 0, 3, 0]),
    ]
    refs = [r for _, r in cases]
    hyps = [h for h, _ in cases]
    rows, _ = run_counts(hyps, refs, L)
    for i, (h, r) in enumerate(cases):
        assert rows[0, i].tolist() == string_counts(h, r, L), i
    # labels without a space: space = len(labels), a non-empty row is one word
    L2 = list(L)
    L2[SPACE] = '#'
    rows, _ = run_counts(hyps[:13], refs[:13], L2)
    for i in range(13):
        assert rows[0, i].tolist() == string_counts(hyps[i], refs[i], L2), i
