"""-m gpu: `run_transcribe` end to end on a seeded WAV file, against an oracle pipeline (the float64 spectrogram of
each chunk -> oracle forward carrying `hs` -> greedy path), and `ChunkSpectrogramParser` against the oracle
spectrogram."""
import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from gpu_helpers import make_model, oracle_cfg, rel
from oracle import ds2_oracle as O
from oracle import spect_oracle as S

pytestmark = pytest.mark.gpu
SR = 16000


def _wav(tmp_path, seconds, seed=0):
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    t = np.arange(n) / SR
    y = 0.3 * np.sin(2 * np.pi * 440 * t) * np.sin(2 * np.pi * 1.3 * t) + 0.05 * rng.standard_normal(n)
    pcm = np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16)
    path = str(tmp_path / "audio.wav")
    wavfile.write(path, SR, pcm)
    return path, pcm.astype(np.float32) / 32768


def _oracle_transcribe(y, chunk, P, ocfg):
    hs, outs = None, []
    for s, e in ds.inference.chunk_bounds(len(y), SR, chunk):
        spect = torch.from_numpy(S.compute_spectrogram(y[s:e]).astype(np.float32))
        x = spect.view(1, 1, *spect.shape)
        out, _, hs, _ = O.forward(x, torch.tensor([spect.shape[1]]), P, ocfg, training=False, hs=hs)
        outs.append(out)
    probs = torch.cat(outs, dim=1)
    return probs, O.greedy_path(probs, None, blank=0)[0]


def test_chunk_spectrograms_match_the_oracle(tmp_path):
    path, y = _wav(tmp_path, 2.37)
    parser = ds.ChunkSpectrogramParser(ds.SpectConfig(), normalize=True)
    got = list(parser.parse_audio(path, 0.7))
    bounds = ds.inference.chunk_bounds(len(y), SR, 0.7)
    assert len(got) == len(bounds) == 4
    for g, (s, e) in zip(got, bounds):
        ref = S.compute_spectrogram(y[s:e])
        assert g.is_cuda and tuple(g.shape) == ref.shape
        assert rel(g, torch.from_numpy(ref)) < 1e-4


@pytest.mark.parametrize("rnn,bidir,chunk", [("lstm", True, 0.5), ("gru", False, 0.6), ("lstm", True, -1)])
def test_run_transcribe_matches_the_oracle_pipeline(tmp_path, rnn, bidir, chunk):
    path, y = _wav(tmp_path, 1.73, seed=1)
    ocfg = oracle_cfg(rnn, bidir, 64, 2, ctx=5)
    P = O.init_params(ocfg, seed=4)
    P["fc.0.module.1.weight"] = P["fc.0.module.1.weight"] * 50      # peaked outputs: an argmax worth comparing
    model = make_model(rnn, bidir, 64, 2, ctx=5, params=P).eval()
    parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
    ds.set_precision("fp32")
    greedy = ds.GreedyDecoder(model.labels)
    strings, offsets = ds.run_transcribe(path, parser, model, greedy, torch.device("cuda"), 32, chunk)
    probs, (lab, offs) = _oracle_transcribe(y, chunk, P, ocfg)
    top2 = probs.topk(2, dim=2).values
    assert float((top2[..., 0] - top2[..., 1]).min()) > 1e-4, "argmax too close to call"
    assert strings[0][0] == "".join(model.labels[i] for i in lab)
    assert offsets[0][0].tolist() == offs
    # beam search over the same outputs
    beam = ds.BeamCTCDecoder(model.labels, beam_width=10, blank_index=0)
    bstrings, boffsets = ds.run_transcribe(path, parser, model, beam, torch.device("cuda"), 32, chunk)
    ref_b = beam.decode(probs.cuda())
    assert bstrings == ref_b[0]
    assert [[o.tolist() for o in u] for u in boffsets] == [[o.tolist() for o in u] for u in ref_b[1]]


def test_whole_file_equals_one_plain_forward(tmp_path):
    path, y = _wav(tmp_path, 1.2, seed=2)
    model = make_model("lstm", True, 64, 2).eval()
    parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
    ds.set_precision("fp32")

    class Keep:               # a decoder that hands back what it was given
        def decode(self, probs, sizes=None):
            return probs
    got = ds.run_transcribe(path, parser, model, Keep(), torch.device("cuda"), 32, -1)
    spect = next(iter(parser.parse_audio(path)))
    with torch.no_grad():
        ref, _, _ = model(spect.view(1, 1, *spect.shape), torch.tensor([spect.shape[1]], dtype=torch.int32))
    assert torch.equal(got, ref)


def test_precision_16_runs_without_fallback(tmp_path):
    path, _ = _wav(tmp_path, 2.2, seed=3)
    model = make_model("lstm", True, 128, 2).eval()
    parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
    lib = ds.get_lib()
    ds.set_precision("fp32")
    lib.ds2_fallback_count(1)
    strings, _ = ds.run_transcribe(path, parser, model, ds.GreedyDecoder(model.labels), torch.device("cuda"), 16, 0.5)
    assert lib.ds2_fallback_count(1) == 0
    assert ds.get_precision() == "fp32"          # the fp16 mode is switched on for the forwards only
    assert isinstance(strings[0][0], str)
