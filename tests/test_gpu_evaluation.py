"""-m gpu: `run_evaluation`, `evaluate`, `LMParamSearch` and `search_lm_params` end to end on seeded WAV files, against
the reference formula: the `metrics.py` classes updated on the same batches (validation.py:135-170)."""
import json

import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from conftest import Golden
from deepspeech_pytorch_b200.evaluation import AudioDataLoader, SpectrogramDataset, model_forward, run_evaluation
from deepspeech_pytorch_b200.lm_search import LMParamSearch, best_result, sample_pairs
from deepspeech_pytorch_b200.metrics import CharErrorRate, WordErrorRate
from gpu_helpers import model_from_golden
from oracle import lm_oracle as LO

pytestmark = pytest.mark.gpu

SR = 16000
WORDS = ["ABE", "BAD", "CAB", "DEED", "ACE", "BEAD", "DAB", "ECE"]


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    """11 seeded WAV files (0.3 - 1.4 s) with transcripts over the model's words, a manifest, and a 2-gram model"""
    root = tmp_path_factory.mktemp("eval")
    rng = np.random.default_rng(7)
    samples = []
    for k in range(11):
        n = int(rng.integers(int(0.3 * SR), int(1.4 * SR)))
        t = np.arange(n) / SR
        y = 0.3 * np.sin(2 * np.pi * (200 + 40 * k) * t) + 0.05 * rng.standard_normal(n)
        wavfile.write(str(root / f"u{k}.wav"), SR, np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16))
        text = ' '.join(rng.choice(WORDS, int(rng.integers(0, 4))).tolist()) + ("\n" if k % 3 else "")
        (root / f"u{k}.txt").write_text(text)
        samples.append({"wav_path": f"u{k}.wav", "transcript_path": f"u{k}.txt"})
    man = root / "manifest.json"
    man.write_text(json.dumps({"root_path": str(root), "samples": samples}))
    lm = str(root / "lm.arpa")
    LO.synthetic_arpa(lm, 0, 2, [30], seed=3, words=WORDS)
    return {"manifest": str(man), "lm": lm, "root": root}


def models():
    return {name: model_from_golden(Golden(name)).eval() for name in ("bilstm_h24_l2", "unigru_h16_l2_la5")}


def loader_of(data, model, batch_size=4):
    d = SpectrogramDataset(model.spect_cfg, data["manifest"], model.labels, normalize=True)
    return AudioDataLoader(d, batch_size=batch_size, num_workers=0)


def reference_rates(loader, model, decoder, precision):
    """validation.py:135-170 with metrics.py's classes"""
    target = ds.GreedyDecoder(model.labels)
    wer, cer = WordErrorRate(decoder, target), CharErrorRate(decoder, target)
    with torch.no_grad():
        for inputs, targets, pct, tsz in loader:
            out, osz, _ = model_forward(model, inputs, pct.mul_(int(inputs.size(3))).int(), precision)
            wer.update(out, osz, targets, tsz)
            cer.update(out, osz, targets, tsz)
    return wer.compute(), cer.compute()


def decoders(data, labels):
    return {"greedy": ds.GreedyDecoder(labels),
            "beam": ds.BeamCTCDecoder(labels, beam_width=16),
            "beam_lm": ds.BeamCTCDecoder(labels, lm_path=data["lm"], alpha=0.7, beta=0.4, beam_width=16)}


@pytest.mark.parametrize("precision", [32, 16])
def test_run_evaluation_equals_the_metrics_classes(data, precision):
    for name, model in models().items():
        loader = loader_of(data, model)
        for kind, dec in decoders(data, model.labels).items():
            ref = reference_rates(loader, model, dec, precision)
            got = run_evaluation(loader, model, dec, torch.device("cuda"), ds.GreedyDecoder(model.labels), precision)
            assert got == ref, (name, kind, precision, got, ref)
            assert all(isinstance(x, float) for x in got)


def test_evaluate_from_a_checkpoint(data, capsys):
    g = Golden("bilstm_h24_l2")
    model = model_from_golden(g).eval()
    ckpt = str(data["root"] / "model.ckpt")
    hp = dict(labels=model.labels, model_cfg=model.model_cfg, precision=32, optim_cfg=model.optim_cfg,
              spect_cfg=model.spect_cfg)
    torch.save({"state_dict": {k: v.cpu() for k, v in model.state_dict().items()}, "hyper_parameters": hp}, ckpt)
    for dtype, lm_path in ((ds.DecoderType.greedy, ''), (ds.DecoderType.beam, data["lm"])):
        cfg = ds.EvalConfig(test_path=data["manifest"], batch_size=3, num_workers=0)
        cfg.model.model_path = ckpt
        cfg.lm = ds.LMConfig(decoder_type=dtype, lm_path=lm_path, alpha=0.7, beta=0.4, beam_width=16)
        got = ds.evaluate(cfg)
        assert "Test Summary" in capsys.readouterr().out
        dec = ds.load_decoder(model.labels, cfg.lm)
        assert got == reference_rates(loader_of(data, model, 3), model, dec, 32)


def test_search_equals_repeated_evaluation(data):
    model = models()["unigru_h16_l2_la5"]
    loader = loader_of(data, model, batch_size=4)
    W = 16
    pairs = [(0.0, 0.0), (0.7, 0.4), (2.5, -0.5), (1.2, 1.0), (3.0, 0.9)]
    base = ds.BeamCTCDecoder(model.labels, lm_path=data["lm"], beam_width=W)
    search = LMParamSearch(loader, model, base, precision=32)
    assert search.n_utterances == 11 and search.device_bytes > 0
    together = search.evaluate(pairs)
    split = [search.evaluate([p])[0] for p in pairs]
    small = LMParamSearch(loader, model, base, precision=32, group_size=3, label_bytes=1)    # 4 groups, 1 pair each
    assert together == split == small.evaluate(pairs)
    for (a, b), r in zip(pairs, together):
        dec = ds.BeamCTCDecoder(model.labels, lm_path=data["lm"], alpha=a, beta=b, beam_width=W)
        ref = run_evaluation(loader, model, dec, torch.device("cuda"), ds.GreedyDecoder(model.labels), 32)
        assert r == (a, b) + ref, (r, ref)
        assert ref == reference_rates(loader, model, dec, 32)


def test_search_lm_params_writes_and_picks(data, capsys):
    model = models()["bilstm_h24_l2"]
    ckpt = str(data["root"] / "search.ckpt")
    hp = dict(labels=model.labels, model_cfg=model.model_cfg, precision=32, optim_cfg=model.optim_cfg,
              spect_cfg=model.spect_cfg)
    torch.save({"state_dict": {k: v.cpu() for k, v in model.state_dict().items()}, "hyper_parameters": hp}, ckpt)
    out = str(data["root"] / "results.json")
    for char_based in (True, False):
        cfg = ds.OptimizerConfig(model_path=ckpt, test_path=data["manifest"], lm_path=data["lm"], beam_width=8,
                                 n_trials=24, precision=32, batch_size=5, num_workers=0, seed=4, output_path=out,
                                 is_character_based=char_based, beta_from=-0.5)
        res = ds.search_lm_params(cfg)
        text = capsys.readouterr().out
        saved = json.loads(open(out).read())
        assert saved == [list(r) for r in res] and len(saved) == 24
        assert [tuple(r[:2]) for r in res] == sample_pairs(cfg)
        best = best_result(res, char_based)
        key = 'cer' if char_based else 'wer'
        assert f"Best Params\nalpha: {best[0]}\nbeta: {best[1]}\n{key}: {best[3] if char_based else best[2]}" in text
        loader = AudioDataLoader(SpectrogramDataset(cfg.spect_cfg, cfg.test_path, model.labels, normalize=True),
                                 batch_size=5, num_workers=0)
        dec = ds.BeamCTCDecoder(model.labels, lm_path=data["lm"], beam_width=8)
        assert LMParamSearch(loader, model, dec, precision=32).evaluate(sample_pairs(cfg)) == res
