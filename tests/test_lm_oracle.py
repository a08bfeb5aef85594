"""CPU: the ARPA language model (row N6) -- the package's parse and vocabulary trie, the float64 scorer and beam
search of `oracle/lm_oracle.py` against hand-computed values and implementation-independent pins, and the host side
of `BeamCTCDecoder(lm_path=...)`.

- Parser: every refusal of rule L0; .arpa.gz and .arpa parse alike; values are fp32 and an unwritten backoff is 0.
- Scorer (rule L2) on a hand-written 3-gram file: listed trigram, back-off to the bigram and to the unigram, an
  unlisted context, <s> padding, OOV.
- Dictionary (rule L1): admissible extensions of chosen partial words; words with non-label characters are not in V.
- Exhaustive width: with W above the number of admissible labellings, every admissible labelling comes out once, with
  score = CTC log-likelihood + sum of a(w) over its words (+ the L5 term), and the best one first.
- L4: a hand-built case where the full-beam filter drops what the unfiltered search keeps."""
import gzip
import itertools

import numpy as np
import pytest

from oracle import beam_oracle as BO
from oracle import ds2_oracle as O
from oracle import lm_oracle as LO

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import lm as LMmod

TINY3 = """
\\data\\
ngram 1=7
ngram 2=5
ngram 3=2

\\1-grams:
-1.0\t<s>\t-0.5
-2.0\t</s>
-1.5\tA\t-0.25
-1.25\tAB\t-0.125
-1.75\tB
-2.5\tBA
-3.0\tax

\\2-grams:
-0.5\t<s> A\t-0.3
-0.75\tA AB\t-0.2
-0.4\tA B
-0.6\tAB B
-0.9\t<s> AB

\\3-grams:
-0.1\t<s> A AB
-0.2\tA AB B

\\end\\
"""
SMALL_LABELS = ['_', 'A', 'B', ' ']


def f32(x):
    return float(np.float32(x))


@pytest.fixture
def tiny3(tmp_path):
    p = tmp_path / "tiny3.arpa"
    p.write_text(TINY3)
    return str(p)


def write(tmp_path, name, text, gz=False):
    p = tmp_path / name
    p.write_bytes(gzip.compress(text.encode()) if gz else text.encode())
    return str(p)


# ---- parser (rule L0)

def _refusals():
    base = TINY3
    return [
        ("counts", base.replace("ngram 2=5", "ngram 2=6")),
        ("duplicate", base.replace("-0.4\tA B\n", "-0.4\tA B\n-0.41\tA B\n").replace("ngram 2=5", "ngram 2=6")),
        ("no_bos", base.replace("<s>", "<x>")),
        ("order6", "\\data\\\n" + "".join(f"ngram {n}=1\n" for n in range(1, 7)) + "\n" + "".join(
            f"\\{n}-grams:\n-1.0\t" + " ".join(["<s>"] * n) + "\n\n" for n in range(1, 7)) + "\\end\\\n"),
        ("char_based", "\\data\\\nngram 1=4\n\n\\1-grams:\n-1\t<s>\n-1\t</s>\n-1\tA\n-1\tB\n\n\\end\\\n"),
        ("unspellable", base.lower()),
        ("binary", None),
    ]


@pytest.mark.parametrize("what,text", _refusals(), ids=[r[0] for r in _refusals()])
def test_every_l0_refusal_raises(tmp_path, what, text):
    if text is None:
        p = tmp_path / "lm.binary"
        p.write_bytes(b"mmap lm http://kheafield.com/code format version 5\n\0\0\x01\x02" + bytes(range(256)))
        path = str(p)
    else:
        path = write(tmp_path, what + ".arpa", text)
    with pytest.raises(ds.Ds2Error, match="language-model scoring"):
        ds.BeamCTCDecoder(ds.LABELS, lm_path=path)


def test_refusals_of_the_labels_and_missing_file(tiny3, tmp_path):
    for bad in (tiny3 + ".missing", str(tmp_path)):
        with pytest.raises(ds.Ds2Error, match="language-model scoring"):
            ds.BeamCTCDecoder(ds.LABELS, lm_path=bad)
    with pytest.raises(ds.Ds2Error, match="language-model scoring"):
        ds.BeamCTCDecoder([c for c in ds.LABELS if c != ' '], lm_path=tiny3)
    big = "\\data\\\nngram 1=%d\n\n\\1-grams:\n" % (1 << 24)
    with pytest.raises(ds.Ds2Error, match="language-model scoring"):
        ds.BeamCTCDecoder(ds.LABELS, lm_path=write(tmp_path, "big.arpa", big + "\\end\\\n"))


def test_gzip_and_plain_parse_alike_fp32_and_missing_backoff_zero(tiny3, tmp_path):
    a = LMmod.read_arpa(tiny3)
    b = LMmod.read_arpa(write(tmp_path, "tiny3.arpa.gz", TINY3, gz=True))
    assert a.order == b.order == 3 and a.words == b.words
    for n in range(3):
        assert np.array_equal(a.ids[n], b.ids[n]) and np.array_equal(a.logp[n], b.logp[n])
        assert np.array_equal(a.backoff[n], b.backoff[n])
        assert a.logp[n].dtype == np.float32 and a.backoff[n].dtype == np.float32
    assert a.words[:3] == [b"<s>", b"</s>", b"A"]
    assert a.logp[2][0] == np.float32(-0.1) and a.backoff[0][1] == 0.0     # </s> has no backoff written
    assert a.ids[2].tolist() == [[0, 2, 3], [2, 3, 4]]
    o = LO.read_arpa(tiny3)                                                 # the oracle's dicts hold the same values
    for n in range(3):
        for g, lp, bo in zip(a.ids[n], a.logp[n], a.backoff[n]):
            key = tuple(a.words[i].decode() for i in g)
            assert o.prob[key] == float(lp) and o.bo.get(key, 0.0) == float(bo)


def test_synthetic_file_parses_to_the_oracle_tables(tmp_path):
    p = str(tmp_path / "syn.arpa.gz")
    LO.synthetic_arpa(p, 60, 4, [150, 150, 100], seed=3, alphabet="ABC'", gz=True)
    a, o = LMmod.read_arpa(p), LO.read_arpa(p)
    assert a.order == o.order == 4
    assert sum(len(x) for x in a.logp) == len(o.prob)
    for n in range(4):
        for g, lp, bo in zip(a.ids[n], a.logp[n], a.backoff[n]):
            key = tuple(a.words[i].decode() for i in g)
            assert o.prob[key] == float(lp) and o.bo.get(key, 0.0) == float(bo)


# ---- scorer (rule L2)

def test_scorer_hand_computed_values(tiny3):
    lm = LO.read_arpa(tiny3)
    ctx = lm.context
    assert ctx(()) == ("<s>", "<s>") and ctx(("A",)) == ("<s>", "A") and ctx(("A", "AB", "B")) == ("AB", "B")
    # listed trigram
    assert lm.lm("AB", ctx(("A",))) == f32(-0.1)
    # back-off to the bigram with bo(<s> A) applied
    assert lm.lm("B", ctx(("A",))) == f32(-0.3) + f32(-0.4)
    # back-off to the unigram through two levels: bo(<s> A) + bo(A) + p(A)
    assert lm.lm("A", ctx(("A",))) == (f32(-0.3) + f32(-0.25)) + f32(-1.5)
    # unlisted context (A A): backoff 0, then the listed bigram (A AB)
    assert lm.lm("AB", ctx(("A", "A"))) == 0.0 + f32(-0.75)
    # <s> padding: first word (<s> <s> A) -> bigram (<s> A); second word (<s> A AB) listed
    assert lm.lm("A", ctx(())) == f32(-0.5)
    # first word, two levels down: (<s> <s>) unlisted (0), (<s> BA) unlisted, bo(<s>) = -0.5, p(BA) = -2.5
    assert lm.lm("BA", ctx(())) == (0.0 + f32(-0.5)) + f32(-2.5)
    # OOV
    assert lm.lm("ZZ", ctx(())) == -1000.0


# ---- dictionary (rule L1)

def test_dictionary_extensions_and_excluded_words(tiny3):
    lm = LO.read_arpa(tiny3)
    D = LO.Dictionary(lm, SMALL_LABELS, 0)
    A, B, SP = 1, 2, 3
    assert set(D.word_of.values()) == {"A", "AB", "B", "BA"}              # "ax" has a non-label character
    assert [c for c in (A, B, SP) if D.allowed((), c)] == [A, B]          # no leading space
    assert [c for c in (A, B, SP) if D.allowed((A,), c)] == [B, SP]
    assert [c for c in (A, B, SP) if D.allowed((A, B), c)] == [SP]
    assert [c for c in (A, B, SP) if D.allowed((B, A), c)] == [SP]
    tr = LMmod.build_trie(LMmod.read_arpa(tiny3), SMALL_LABELS, 0)
    for pre in D.prefixes:                                                 # the package's trie spells the same V
        nd = 0
        for c in pre:
            nd = tr.child(nd, c)
            assert nd >= 0
        allowed = int(tr.mask[nd]) | ((1 << SP) if tr.word[nd] >= 0 else 0)
        assert allowed == sum(1 << c for c in (A, B, SP) if D.allowed(pre, c)), pre
    assert tr.n_words == 4 and tr.child(0, SP) == -1


# ---- exhaustive width

def admissible(T, V):
    """label strings over {A, B, ' '} that fit T frames, whose completed words are in V and whose partial word is a
    prefix of a word of V"""
    pref = {w[:k] for w in V for k in range(len(w) + 1)}
    out = []
    for n in range(T + 1):
        for s in itertools.product("AB ", repeat=n):
            if n + sum(s[i] == s[i + 1] for i in range(n - 1)) > T:
                continue
            parts = ''.join(s).split(' ')
            if all(w in V for w in parts[:-1]) and parts[-1] in pref:
                out.append(''.join(s))
    return out


@pytest.mark.parametrize("alpha", [0.0, 1.3])
@pytest.mark.parametrize("beta", [-0.7, 0.0, 2.0])
@pytest.mark.parametrize("T,seed", [(5, 0), (6, 1)])
def test_exhaustive_width_is_ctc_likelihood_plus_lm_terms(tiny3, alpha, beta, T, seed):
    lm = LO.read_arpa(tiny3)
    V = {"A", "AB", "B", "BA"}
    labs = admissible(T, V)
    assert 20 < len(labs) < 128
    rng = np.random.default_rng(10 * T + seed)
    lg = rng.standard_normal((T, 4)) * 1.2
    pr = (np.exp(lg) / np.exp(lg).sum(-1, keepdims=True)).astype(np.float32)
    trace = []
    beams, _ = LO.beam_search_lm(pr, None, 0, 128, 40, 1.0, SMALL_LABELS, lm, alpha, beta, trace=trace)
    assert max(len(fr) for fr in trace) < 128                              # the list is never full: no L4
    got = {''.join(SMALL_LABELS[c] for c in lab): s for lab, _, s in beams}
    assert len(got) == len(beams) and set(got) == set(labs)
    logZ = float(np.log(pr.astype(np.float64).sum(-1)).sum())
    lp = np.log(pr.astype(np.float64))[:, None, :]
    best = None
    for s in labs:
        tgt = np.array([SMALL_LABELS.index(ch) for ch in s], np.int64)
        nll, _ = O.ctc_loss_and_grad(lp, tgt, [T], [len(s)], blank=0)
        parts = s.split(' ')
        lmsum = 0.0
        for k, w in enumerate(parts[:-1]):
            lmsum += alpha * lm.lm(w, lm.context(tuple(parts[:k]))) + beta
        if parts[-1]:                                                      # L5: the partial word
            w = parts[-1]
            v = lm.lm(w, lm.context(tuple(parts[:-1]))) if w in V else -1000.0
            lmsum += alpha * v + beta
        want = float(nll[0]) - logZ - lmsum
        assert abs(got[s] - want) <= 1e-12 * max(1.0, abs(want)), (s, got[s], want)
        if best is None or want < best[0]:
            best = (want, s)
    top = ''.join(SMALL_LABELS[c] for c in beams[0][0])
    assert top == best[1] or abs(got[top] - best[0]) <= 1e-12 * max(1.0, abs(best[0]))
    assert [s for _, _, s in beams] == sorted(s for _, _, s in beams)


# ---- L4

def test_full_beam_filter_drops_what_the_unfiltered_search_keeps(tiny3):
    """W = 2.  Frame 0 lists ('' 0.45, A 0.4).  At frame 1 the list is full and m = log 0.4 + log 0.5: A's second nb
    term from '' (0.41 * 0.45 < 0.4 * 0.5) and its repeat (0.41 * 0.4) are dropped, so A keeps only its blank term
    (0.2 < 0.225) and falls behind '', and its timestep does not move to frame 1 (p = 0.41 > 0.4).  The unfiltered
    search (alpha = beta = 0 makes every LM term 0, so it is the no-LM oracle) lists A first with timestep 1."""
    lm = LO.read_arpa(tiny3)
    pr = np.array([[0.45, 0.4, 0.15, 0.0], [0.5, 0.41, 0.09, 0.0]], np.float32)
    trace, stats = [], {}
    beams, margin = LO.beam_search_lm(pr, None, 0, 2, 40, 1.0, SMALL_LABELS, lm, 0.0, 0.0, trace=trace,
                                      stats=stats)
    ref_trace = []
    ref, _ = BO.beam_search(pr, None, 0, 2, 40, 1.0, trace=ref_trace)
    assert [p for p, _, _ in trace[0]] == [p for p, _, _ in ref_trace[0]] == [(), (1,)]
    assert [p for p, _, _ in trace[1]] == [(), (1,)]
    assert [p for p, _, _ in ref_trace[1]] == [(1,), ()]
    assert stats["l4_drops"] == 5 and margin > 1e-3
    assert [(lab, ts) for lab, ts, _ in beams] == [([], []), ([1], [0])]
    assert [(lab, ts) for lab, ts, _ in ref] == [([1], [1]), ([], [])]
    lp = np.log(pr.astype(np.float64))
    assert beams[1][2] == -(lp[0, 1] + lp[1, 0])                           # A: its blank term only


# ---- API

def test_decoder_with_an_arpa_model_needs_no_gpu(tiny3):
    d = ds.BeamCTCDecoder(SMALL_LABELS, lm_path=tiny3, alpha=0.5, beta=1.0)
    assert d.lm is not None and d.lm.order == 3 and d.lm.trie.n_words == 4
    assert (d.alpha, d.beta) == (0.5, 1.0)
    d.reset_params(1.7, -0.25)
    assert (d.alpha, d.beta) == (1.7, -0.25)
    d._decoder.reset_params(0.3, 2.0)                    # what the reference's search_lm_params.py calls
    assert (d.alpha, d.beta) == (0.3, 2.0)
    g = ds.load_decoder(ds.LABELS, ds.LMConfig(decoder_type=ds.DecoderType.beam, lm_path=tiny3, alpha=0.8,
                                               beta=1.5, beam_width=16))
    assert isinstance(g, ds.BeamCTCDecoder) and g.lm is not None and (g.alpha, g.beta) == (0.8, 1.5)
    assert g.lm.space == ds.LABELS.index(' ') and g.beam_width == 16
