"""CPU checks of forced alignment: the float64 oracle (oracle/align_oracle.py) against torchaudio's forced_align and
against the recursion's own rules, the host side of the records, the manifest-order mapping and the workspace
formula of `ds2_ctc_align`.  No GPU here."""
import math

import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import alignment as AL
from deepspeech_pytorch_b200.input_pipeline import SpectrogramBatcher
from oracle import align_oracle as A

C = 29


def _lp(T, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((T, C)) * 3
    return x - np.log(np.exp(x).sum(1, keepdims=True))


def _min_frames(tg):
    return len(tg) + sum(1 for i in range(1, len(tg)) if tg[i] == tg[i - 1])


CASES = [([], 7), ([5], 1), ([5], 9), ([3, 3], 3), ([1, 2, 3, 4, 5, 6], 6), ([4, 4, 4, 7, 7, 2], 9),
         ([1, 2, 3, 4, 5, 6, 7, 8], 40), ([9, 9, 1, 9, 9, 9, 2, 2, 5], 60)]


@pytest.mark.parametrize("tg,T", CASES)
def test_oracle_matches_torchaudio(tg, T):
    F = pytest.importorskip("torchaudio.functional")
    assert T >= _min_frames(tg)
    lp = _lp(T, seed=T + len(tg))
    ref = A.ctc_align(lp, tg)
    if not tg:       # torchaudio needs a non-empty target: the all-blank path
        assert ref["labels"].tolist() == [0] * T and math.isclose(ref["score"], lp[:, 0].sum(), rel_tol=1e-12)
        return
    em = torch.from_numpy(lp)[None]
    labels, scores = F.forced_align(em, torch.tensor([tg], dtype=torch.int32), blank=0)
    assert labels[0].tolist() == ref["labels"].tolist()
    assert math.isclose(float(scores[0].sum()), ref["score"], rel_tol=1e-12, abs_tol=1e-12)


@pytest.mark.parametrize("tg,T", CASES)
def test_oracle_path_collapses_to_the_target(tg, T):
    ref = A.ctc_align(_lp(T, seed=3 * T), tg)
    assert A.collapse(ref["labels"]) == tg
    assert math.isclose(ref["frame_log_probs"].sum(), ref["score"], rel_tol=1e-12, abs_tol=1e-12)
    for k, (s, e) in enumerate(ref["spans"]):
        assert 0 <= s < e <= T and set(ref["labels"][s:e].tolist()) == {tg[k]}
        assert k == 0 or s >= ref["spans"][k - 1][1]


def test_uniform_log_probs_follow_the_tie_rule():
    # every path scores the same: each state is entered from itself when it can be (stay first), so walking back from
    # the end (S-1: ties prefer it) the path lingers in the last states, i.e. it moves through the target at once
    T, tg = 8, [1, 2, 3]
    ref = A.ctc_align(np.full((T, C), -math.log(C)), tg)
    assert ref["labels"].tolist() == [1, 2, 3, 0, 0, 0, 0, 0]
    assert ref["spans"].tolist() == [[0, 1], [1, 2], [2, 3]]
    ref = A.ctc_align(np.full((T, C), -math.log(C)), [1, 1])      # the repeat needs its blank: s-2 is not allowed
    assert ref["labels"].tolist() == [1, 0, 1, 0, 0, 0, 0, 0]
    ref = A.ctc_align(np.full((4, C), -math.log(C)), [])
    assert ref["labels"].tolist() == [0, 0, 0, 0]


def test_final_state_tie_prefers_the_trailing_blank():
    lp = np.full((3, C), -5.0)
    ref = A.ctc_align(lp, [4])
    assert ref["labels"][-1] == 0 and ref["final"][0] == ref["final"][1]


def test_infeasible_inputs():
    lp = _lp(5, seed=1)
    for tg in ([1, 2, 3, 4, 5, 6], [2, 2, 2, 2]):          # too few frames (repeats need blanks between them)
        ref = A.ctc_align(lp, tg)
        assert ref["score"] == -np.inf and (ref["labels"] == -1).all() and (ref["spans"] == -1).all()
    lp2 = lp.copy()
    lp2[:, 3] = -np.inf                                   # every path runs through a -inf entry
    assert A.ctc_align(lp2, [1, 3])["score"] == -np.inf
    assert A.ctc_align(np.zeros((0, C)), [1])["score"] == -np.inf
    assert A.ctc_align(np.zeros((0, C)), [])["score"] == 0.0
    assert A.ctc_align(lp, [2, 2, 2])["score"] > -np.inf  # exactly the minimum


# ---------------------------------------------------------------------------------------------- host records
def test_records_from_spans():
    text = " HI  THERE "
    n = len(text)
    spans = [[2 * i, 2 * i + 1 + (i % 2)] for i in range(n)]
    scores = [0.5 + 0.01 * i for i in range(n)]
    rec = AL.alignment_record(text, spans, scores, -12.5, 40, 0.01, 10.0)
    assert rec["feasible"] and rec["score"] == -12.5 and rec["frames"] == 40 and rec["transcript"] == text
    assert "".join(c["char"] for c in rec["chars"]) == text
    assert [w["word"] for w in rec["words"]] == ["HI", "THERE"]
    hi = rec["words"][0]
    assert hi["start"] == AL.frame_seconds(2, 0.01) and hi["end"] == AL.frame_seconds(5, 0.01)
    w = [(e - s) for s, e in spans[1:3]]
    assert math.isclose(hi["score"], (scores[1] * w[0] + scores[2] * w[1]) / sum(w))
    assert rec["chars"][0] == {"char": " ", "start": 0.0, "end": AL.frame_seconds(1, 0.01), "score": 0.5}


def test_records_edge_cases():
    rec = AL.alignment_record("", [], [], -3.0, 5, 0.01, 1.0)
    assert rec["feasible"] and rec["chars"] == [] and rec["words"] == []
    rec = AL.alignment_record("AB", [[-1, -1], [-1, -1]], [0.0, 0.0], float("-inf"), 5, 0.01, 1.0)
    assert not rec["feasible"] and rec["score"] is None and rec["chars"] == [] and rec["words"] == []
    rec = AL.alignment_record("A", [[3, 5]], [1.0], -1.0, 5, 0.01, 0.09)   # the last frame reaches past the end
    assert rec["chars"][0]["start"] == 0.06 and rec["chars"][0]["end"] == 0.09


def test_seconds():
    assert AL.frame_seconds(0, 0.01) == 0.0
    assert math.isclose(AL.frame_seconds(50, 0.01), 1.0)
    assert math.isclose(AL.frame_seconds(7, 0.02), 0.28)


def test_manifest_order_mapping():
    hop = 160
    n_samples = [16000, 48000, 11000, 48000, 35200]
    order, frames = SpectrogramBatcher.order_and_frames(n_samples, hop)
    rows = [f"row{j}" for j in range(len(order))]          # row j of the sorted batch
    items = AL.unsort_rows(rows, order)
    assert order == [1, 3, 4, 0, 2]
    assert items == ["row3", "row0", "row4", "row1", "row2"]
    assert [frames[i] for i in order] == sorted(frames, reverse=True)


def _pad(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("T,B,Cn,L", [(500, 32, 29, 200), (500, 32, 29, 250), (30000, 4, 29, 6000), (1, 1, 2, 0),
                                      (37, 3, 29, 5), (250, 7, 1000, 61), (13000, 2, 29, 6144)])
def test_workspace_formula(T, B, Cn, L):
    want = _pad(T * B * Cn * 4) + _pad(B * T * ((2 * L + 1 + 31) // 32) * 8) + _pad(B * 8)
    assert ds.get_lib().ds2_ctc_align_workspace_bytes(T, B, Cn, L) == want
    assert ds.get_lib().ds2_ctc_align_workspace_bytes(500, 32, 29, 250) == 3904256   # the header's example


def test_model_forward_default_is_unchanged():
    import inspect
    sig = inspect.signature(ds.DeepSpeech.forward)
    assert sig.parameters["logits"].kind is inspect.Parameter.KEYWORD_ONLY and sig.parameters["logits"].default is False
