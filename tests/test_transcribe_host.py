"""Host side of chunked transcription: chunk boundaries (the reference's `get_chunks` float expressions), WAV loading
and its normalisation, the `decode_results` structure and the config defaults."""
import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.inference import chunk_bounds


def test_chunk_bounds_hand_computed():
    # 3 s at 1 s chunks: exact
    assert chunk_bounds(48000, 16000, 1) == [(0, 16000), (16000, 32000), (32000, 48000)]
    # a non-integer duration: ceil(2.5 s) = 3 s, the last chunk is clipped to the signal
    assert chunk_bounds(40000, 16000, 1) == [(0, 16000), (16000, 32000), (32000, 40000)]
    # chunk <= 0: the whole file
    assert chunk_bounds(40000, 16000, -1) == [(0, 40000)]
    assert chunk_bounds(40000, 16000, 0) == [(0, 40000)]
    # 1.01 s at 0.5 s: ceil -> 2 s, 4 chunks, the 4th ([24000, 32000)) lies past the signal and is skipped
    assert chunk_bounds(16160, 16000, 0.5) == [(0, 8000), (8000, 16000), (16000, 16160)]
    # float rounding of i * chunk * sr: int(3 * 0.7 * 10) = int(20.999999999999996) = 20, while chunk 2 ends at
    # int(2 * 0.7 * 10) + int(0.7 * 10) = 21: chunks 2 and 3 share a sample, as in the reference
    assert int(3 * 0.7 * 10) == 20 and int(2 * 0.7 * 10) + int(0.7 * 10) == 21
    assert chunk_bounds(30, 10, 0.7)[:4] == [(0, 7), (7, 14), (14, 21), (20, 27)]
    with pytest.raises(ds.Ds2Error):
        chunk_bounds(0, 16000, 1)


def _write(tmp_path, name, data, rate=8000):
    p = str(tmp_path / name)
    wavfile.write(p, rate, data)
    return p


def test_load_audio_formats(tmp_path):
    i16 = np.array([0, 1, -1, 32767, -32768], np.int16)
    assert np.array_equal(ds.load_audio(_write(tmp_path, "a.wav", i16)), i16.astype(np.float32) / 32768)
    i32 = np.array([0, 1 << 20, -(1 << 31), (1 << 31) - 1], np.int32)
    assert np.array_equal(ds.load_audio(_write(tmp_path, "b.wav", i32)),
                          i32.astype(np.float32) / np.float32(2 ** 31))
    u8 = np.array([0, 128, 255, 7], np.uint8)
    assert np.array_equal(ds.load_audio(_write(tmp_path, "c.wav", u8)), (u8.astype(np.float32) - 128) / 128)
    f32 = np.array([0.5, -0.25, 1.5], np.float32)
    out = ds.load_audio(_write(tmp_path, "d.wav", f32))
    assert out.dtype == np.float32 and np.array_equal(out, f32)
    st = np.array([[100, -300], [5, 6], [-32768, 32767]], np.int16)     # stereo: fp32 mean of the channels
    ref = (st.astype(np.float32) / 32768).mean(axis=1, dtype=np.float32)
    assert np.array_equal(ds.load_audio(_write(tmp_path, "e.wav", st)), ref)


def test_load_audio_refuses_other_formats(tmp_path):
    with pytest.raises(ds.Ds2Error, match="float64"):
        ds.load_audio(_write(tmp_path, "f.wav", np.zeros(4, np.float64)))
    p = tmp_path / "x.flac"
    p.write_bytes(b"fLaC" + bytes(64))
    with pytest.raises(ds.Ds2Error, match="not a WAV file"):
        ds.load_audio(str(p))


def test_decode_results_structure():
    cfg = ds.TranscribeConfig()
    cfg.lm.top_paths = 2
    cfg.offsets = True
    cfg.model.model_path = "m.ckpt"
    out = [["abc", "abd", "abe"]]
    offs = [[torch.tensor([1, 2, 3], dtype=torch.int), torch.tensor([1, 2, 4], dtype=torch.int),
             torch.tensor([0, 2, 4], dtype=torch.int)]]
    r = ds.decode_results(out, offs, cfg)
    assert r["_meta"] == {"acoustic_model": {"path": "m.ckpt"}, "language_model": {"path": ""},
                          "decoder": {"alpha": 0.0, "beta": 0.0, "type": "greedy"}}
    assert r["output"] == [{"transcription": "abc", "offsets": [1, 2, 3]},
                           {"transcription": "abd", "offsets": [1, 2, 4]}]
    cfg.offsets = False
    cfg.lm.top_paths = 5
    assert ds.decode_results(out, offs, cfg)["output"] == [{"transcription": s} for s in out[0]]


def test_config_defaults():
    cfg = ds.TranscribeConfig()
    assert (cfg.audio_path, cfg.offsets, cfg.chunk_size_seconds) == ("", False, -1)
    assert (cfg.model.precision, cfg.model.cuda, cfg.model.model_path) == (32, True, "")
    assert cfg.lm == ds.LMConfig()
    assert ds.TranscribeConfig().lm is not cfg.lm          # no shared mutable default
    assert isinstance(cfg, ds.InferenceConfig)
