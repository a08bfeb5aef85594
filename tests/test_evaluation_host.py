"""CPU tests of the evaluation and language-model search surface: input parsing, loader order, config defaults, trial
sampling and the best-pair rule, the results file, `load_model`, argument refusals, and a numpy restatement of the
bit-parallel edit distance of csrc/error_rate.cu against `metrics.edit_distance`."""
import ctypes as C
import json
import os
import pickle
import sys
import types

import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.evaluation import AudioDataLoader, SpectrogramDataset, load_model, rates
from deepspeech_pytorch_b200.lm_search import best_result, sample_pairs, write_results
from deepspeech_pytorch_b200.metrics import edit_distance
from oracle import lm_oracle as LO

SR = 16000


def _wav(path, n, seed):
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    wavfile.write(path, SR, (rng.standard_normal(n) * 3000).astype(np.int16))


def _txt(path, text):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w", encoding="utf8") as f:
        f.write(text)


# ------------------------------------------------------------------------------------------------ parsing
def test_manifest_parsing_and_transcript_filter(tmp_path):
    root = tmp_path / "data"
    _wav(str(root / "a" / "x.wav"), 800, 0)
    _wav(str(root / "b" / "y.wav"), 1600, 1)
    _txt(str(root / "a" / "x.txt"), "HEL_LO wo#rld\n2\n")
    _txt(str(root / "b" / "y.txt"), "IT'S\n")
    man = tmp_path / "m.json"
    man.write_text(json.dumps({"root_path": str(root), "samples": [
        {"wav_path": "b/y.wav", "transcript_path": "b/y.txt"},
        {"wav_path": "a/x.wav", "transcript_path": "a/x.txt"}]}))
    d = SpectrogramDataset(ds.SpectConfig(), str(man), ds.LABELS, normalize=True)
    assert len(d) == 2
    assert d.ids == [(str(root / "b" / "y.wav"), str(root / "b" / "y.txt")),
                     (str(root / "a" / "x.wav"), str(root / "a" / "x.txt"))]
    wave, tr = d[1]
    assert wave.dtype == np.float32 and wave.shape == (800,)
    # '_' is label 0 (dropped by filter(None, ...)); lowercase, '#', '2' are not labels
    assert ''.join(ds.LABELS[i] for i in tr) == "HELLO "
    assert ''.join(ds.LABELS[i] for i in d[0][1]) == "IT'S"


def test_directory_parsing(tmp_path):
    root = tmp_path / "set"
    for k, name in enumerate(["s1", "s2", "deep/s3"]):
        _wav(str(root / "wav" / f"{name}.wav"), 400 * (k + 1), k)
        _txt(str(root / "txt" / f"{name}.txt"), f"A B{k}")
    d = SpectrogramDataset(ds.SpectConfig(), str(root), ds.LABELS)
    from pathlib import Path
    expect = [(p, str(p).replace('/wav/', '/txt/').replace('.wav', '.txt')) for p in Path(str(root)).rglob('*.wav')]
    assert d.ids == expect and len(d) == 3
    for i in range(3):
        assert ''.join(ds.LABELS[c] for c in d[i][1]) == "A B"


def test_loader_items_keep_dataset_order_and_batcher_sorts(tmp_path):
    root = tmp_path / "set"
    lens = [1200, 3000, 800, 3000, 2000]
    samples = []
    for k, n in enumerate(lens):
        _wav(str(root / f"{k}.wav"), n, k)
        _txt(str(root / f"{k}.txt"), "AB"[k % 2] * (k + 1))
        samples.append({"wav_path": f"{k}.wav", "transcript_path": f"{k}.txt"})
    man = tmp_path / "m.json"
    man.write_text(json.dumps({"root_path": str(root), "samples": samples}))
    d = SpectrogramDataset(ds.SpectConfig(), str(man), ds.LABELS)
    for workers in (0, 2):
        loader = AudioDataLoader(d, batch_size=3, num_workers=workers)
        got = list(loader.raw_batches())
        assert [[len(w) for w in ws] for ws, _ in got] == [lens[:3], lens[3:]]
        assert [len(t) for t in got[0][1] + got[1][1]] == [1, 2, 3, 4, 5]
    order, frames = ds.input_pipeline.SpectrogramBatcher.order_and_frames(lens[:3] + lens[3:4], 160)
    assert order == [1, 3, 0, 2]                     # descending frames, ties in dataset order


# ------------------------------------------------------------------------------------------------ configs
def test_config_defaults_equal_the_reference():
    e = ds.EvalConfig()
    assert (e.test_path, e.verbose, e.save_output, e.batch_size, e.num_workers) == ('', True, '', 20, 4)
    assert e.lm == ds.LMConfig() and e.model == ds.ModelConfig()
    o = ds.OptimizerConfig()
    assert (o.model_path, o.test_path, o.is_character_based, o.lm_path, o.beam_width, o.alpha_from, o.alpha_to,
            o.beta_from, o.beta_to, o.n_trials, o.n_jobs, o.precision, o.batch_size, o.num_workers) == \
        ('', '', True, '', 10, 0.0, 3.0, 0.0, 1.0, 500, 2, 16, 1, 1)
    assert o.spect_cfg == ds.SpectConfig() and o.seed == 0 and o.output_path == ''


def test_trial_sampling_is_seeded_and_in_range():
    cfg = ds.OptimizerConfig(alpha_from=0.5, alpha_to=2.0, beta_from=-1.0, beta_to=0.25, n_trials=300, seed=11)
    p = sample_pairs(cfg)
    assert p == sample_pairs(cfg) and len(p) == 300
    a, b = np.array(p).T
    assert a.min() >= 0.5 and a.max() < 2.0 and b.min() >= -1.0 and b.max() < 0.25
    assert p != sample_pairs(ds.OptimizerConfig(alpha_from=0.5, alpha_to=2.0, beta_from=-1.0, beta_to=0.25,
                                                n_trials=300, seed=12))
    rng = np.random.default_rng(11)
    assert a.tolist() == rng.uniform(0.5, 2.0, 300).tolist()


def test_best_pair_rule_and_ties():
    res = [(0.1, 0.2, 30.0, 12.0), (0.3, 0.4, 20.0, 15.0), (0.5, 0.6, 20.0, 12.0), (0.7, 0.8, 25.0, 12.0)]
    assert best_result(res, True) == res[0]          # lowest CER, earliest of the ties
    assert best_result(res, False) == res[1]         # lowest WER, earliest of the ties


def test_results_json_layout(tmp_path):
    res = [(0.1, 0.2, 30.0, 12.5), (1.5, 0.0, 0.0, 100.0)]
    p = tmp_path / "r.json"
    write_results(str(p), res)
    got = json.loads(p.read_text())
    assert got == [[0.1, 0.2, 30.0, 12.5], [1.5, 0.0, 0.0, 100.0]]
    assert min(got, key=lambda x: x[2]) == [1.5, 0.0, 0.0, 100.0]    # select_lm_params.py's use


def test_rates_formula():
    assert rates([3, 7, 2, 0]) == (float(2) / 1 * 100, float(3) / 7 * 100)


# ------------------------------------------------------------------------------------------------ load_model
def _model_args():
    return dict(labels=ds.LABELS, model_cfg=ds.BiDirectionalConfig(rnn_type=ds.RNNType.gru, hidden_size=16,
                                                                    hidden_layers=2),
                precision=32, optim_cfg=ds.AdamConfig(), spect_cfg=ds.SpectConfig())


def test_load_model_rebuilds_from_a_checkpoint(tmp_path):
    torch.manual_seed(3)
    m = ds.DeepSpeech(**_model_args())
    p = tmp_path / "m.ckpt"
    torch.save({"state_dict": m.state_dict(), "hyper_parameters": _model_args(), "epoch": 1}, str(p))
    got = load_model(torch.device("cpu"), str(p))
    assert not got.training and got.labels == ds.LABELS
    a, b = m.state_dict(), got.state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    sd = dict(m.state_dict())
    sd.pop(next(iter(sd)))
    torch.save({"state_dict": sd, "hyper_parameters": _model_args()}, str(p))
    with pytest.raises(RuntimeError):                # strict loading
        load_model(torch.device("cpu"), str(p))


def test_load_model_refusals(tmp_path):
    bad = tmp_path / "bad.ckpt"
    bad.write_bytes(b"not a checkpoint")
    with pytest.raises(ds.Ds2Error, match="cannot read"):
        load_model("cpu", str(bad))
    with pytest.raises(ds.Ds2Error, match="cannot read"):
        load_model("cpu", str(tmp_path / "missing.ckpt"))
    torch.save({"state_dict": {}}, str(bad))
    with pytest.raises(ds.Ds2Error, match="hyper_parameters"):
        load_model("cpu", str(bad))
    # hyper-parameters pickled as omegaconf objects, read where omegaconf is not installed
    fake = types.ModuleType("omegaconf")

    class DictConfig(dict):
        pass
    DictConfig.__module__ = "omegaconf"
    DictConfig.__qualname__ = "DictConfig"
    fake.DictConfig = DictConfig
    saved = sys.modules.get("omegaconf")
    sys.modules["omegaconf"] = fake
    try:
        torch.save({"state_dict": {}, "hyper_parameters": DictConfig(labels=ds.LABELS)}, str(bad))
    finally:
        if saved is None:
            del sys.modules["omegaconf"]
        else:
            sys.modules["omegaconf"] = saved
    if saved is None:
        with pytest.raises(ds.Ds2Error, match="omegaconf"):
            load_model("cpu", str(bad))


# ------------------------------------------------------------------------------------------------ refusals
def _tiny_lm(tmp_path):
    p = str(tmp_path / "t.arpa")
    LO.synthetic_arpa(p, 0, 2, [10], seed=1, words=["AB", "BA", "ABBA"])
    return p


@pytest.mark.parametrize("pairs,match", [([], "K = 0"), ([(0.5, float("nan"))], "finite"),
                                         ([(float("inf"), 0.0), (1.0, 1.0)], "finite")])
def test_grid_refuses_bad_pairs(tmp_path, pairs, match):
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=_tiny_lm(tmp_path), beam_width=4)
    with pytest.raises(ds.Ds2Error, match=match):
        dec.decode_best_grid(torch.zeros(1, 3, 29), None, pairs)


def test_library_refuses_bad_pairs_before_any_device_work():
    lib = ds.get_lib()
    buf = np.zeros(64, np.float32)
    lab = np.zeros(64, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for K, pairs, msg in ((0, np.zeros(2), "K=0"), (2, np.array([0.5, 0.5, np.nan, 1.0]), "not finite"),
                          (1, np.array([1.0, -np.inf]), "not finite")):
        rc = lib.ds2_beam_decode_lm_grid(1, 2, 29, p(buf), None, 0, 4, 40, 1.0, p(lab), 2, K, p(pairs), 28, p(lab),
                                         p(lab), p(lab), 64, None)
        assert rc == -1 and msg in lib.ds2_last_error().decode()


# ------------------------------------------------------------------------------------------------ edit distance
MASK = (1 << 64) - 1


def bitlev(pattern, text):
    """numpy/int restatement of BitLev (csrc/error_rate.cu): Hyyroe's block form of Myers' recurrence in 64-bit
    words, the pattern down the column, hin = +1 into block 0, the score read at bit (m-1) mod 64 of the last block"""
    m = len(pattern)
    nb = (m + 63) // 64
    pat = np.asarray(pattern, dtype=object)
    P, M = [MASK] * nb, [0] * nb
    score = m
    for x in text:
        hin = 1
        for w in range(nb):
            eq = 0
            for j in range(64 * w, min(m, 64 * w + 64)):
                if pat[j] == x:
                    eq |= 1 << (j - 64 * w)
            Pv, Mv = P[w], M[w]
            neg = 1 if hin < 0 else 0
            Xv = eq | Mv
            eq |= neg
            Xh = ((((eq & Pv) + Pv) & MASK) ^ Pv) | eq
            Ph = (Mv | ~(Xh | Pv)) & MASK
            Mh = Pv & Xh
            hb = (m - 1) & 63 if w == nb - 1 else 63
            hout = ((Ph >> hb) & 1) - ((Mh >> hb) & 1)
            Ph = (Ph << 1) & MASK
            Mh = (Mh << 1) & MASK
            Mh |= neg
            Ph |= 1 if hin > 0 else 0
            P[w] = (Mh | ~(Xv | Ph)) & MASK
            M[w] = Ph & Xv
            hin = hout
        score += hin if nb else 1
    return score


def test_bit_parallel_recurrence_equals_edit_distance():
    rng = np.random.default_rng(0)
    cases = [([], []), ([], [1, 2]), ([3], []), ([1] * 64, [1] * 63), ([1] * 65, [2] * 65), (list(range(64)), [5]),
             ([1, 2, 3] * 43, [1, 3, 2] * 44)]
    for _ in range(150):
        m, n = int(rng.integers(0, 200)), int(rng.integers(0, 200))
        a = int(rng.integers(1, 6))
        cases.append((rng.integers(0, a, m).tolist(), rng.integers(0, a, n).tolist()))
    for pat, txt in cases:
        assert bitlev(pat, txt) == edit_distance(pat, txt), (pat, txt)


def test_word_and_char_definitions_match_the_string_forms():
    """the label-level definitions of ds2_error_counts (spaces removed for characters, maximal non-space runs for
    words, exact word equality) reproduce `s.replace(' ', '')` and `s.split()`"""
    rng = np.random.default_rng(1)
    sp = ds.LABELS.index(' ')

    def words(seq):
        out, cur = [], []
        for x in seq:
            if x == sp:
                if cur:
                    out.append(tuple(cur))
                cur = []
            else:
                cur.append(x)
        if cur:
            out.append(tuple(cur))
        return out
    for _ in range(200):
        h = rng.choice([sp, 1, 2, 3], size=int(rng.integers(0, 40))).tolist()
        r = rng.choice([sp, 1, 2, 3, 0], size=int(rng.integers(0, 40))).tolist()
        r_nb = [x for x in r if x != 0]
        hs, rs = ''.join(ds.LABELS[x] for x in h), ''.join(ds.LABELS[x] for x in r_nb)
        ids = {}
        hw = [ids.setdefault(w, len(ids)) for w in words(h)]
        rw = [ids.setdefault(w, len(ids)) for w in words(r_nb)]
        assert bitlev(rw, hw) == edit_distance(hs.split(), rs.split())
        assert bitlev([x for x in r_nb if x != sp], [x for x in h if x != sp]) == \
            edit_distance(hs.replace(' ', ''), rs.replace(' ', ''))
