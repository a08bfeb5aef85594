"""Transcription of one audio file, the reference's deepspeech_pytorch/inference.py:15-41,79-99 and
loader/data_loader.py:20-26,58-71,171-186, on the GPU.

`run_transcribe` feeds the file through the model one chunk at a time (`chunk_size_seconds > 0`) and carries each
chunk's final recurrent states into the next chunk's forward, as the reference does.  The recurrent sweeps take that
initial state on the tensor cores (DESIGN.md §5.1).  `ChunkSpectrogramParser` computes the spectrograms of all chunks of
a file in one `ds2_spectrogram_batch` launch.

Deviation: the reference's `get_chunks` can produce an empty trailing chunk (the duration is rounded up to whole
seconds first, e.g. 1.01 s at 0.5 s chunks gives [1.5 s, 2 s) of a 1.01 s signal).  Its spectrogram would be a single
all-zero frame; here that chunk is skipped."""
import math
from typing import Iterator, List, Tuple

import numpy as np
import torch

from . import _lib
from .input_pipeline import SpectrogramBatcher, spect_geometry

__all__ = ["load_audio", "chunk_bounds", "ChunkSpectrogramParser", "run_transcribe", "decode_results"]

# torchaudio.load's default normalisation of each sample format (normalize=True)
_WAV_SCALE = {np.dtype(np.int16): (0.0, 1.0 / 2 ** 15), np.dtype(np.int32): (0.0, 1.0 / 2 ** 31),
              np.dtype(np.uint8): (128.0, 1.0 / 128), np.dtype(np.float32): None}


def load_audio(path) -> np.ndarray:
    """data_loader.py:20-26 for WAV files: float32 samples scaled as torchaudio.load scales them (int16 / 2^15,
    int32 / 2^31, uint8 (x - 128) / 128, float32 unchanged), channels averaged in fp32.  The file's sample rate is
    ignored, as in the reference.  Anything but a WAV file of those four sample formats raises Ds2Error."""
    from scipy.io import wavfile
    with open(path, "rb") as f:
        head = f.read(12)
    if len(head) < 12 or head[:4] not in (b"RIFF", b"RIFX") or head[8:12] != b"WAVE":
        raise _lib.Ds2Error(f"load_audio: {path}: not a WAV file (header {head[:12]!r}); only WAV is supported")
    try:
        _, data = wavfile.read(path)
    except ValueError as e:
        raise _lib.Ds2Error(f"load_audio: {path}: unsupported WAV format ({e})") from None
    if data.dtype not in _WAV_SCALE:
        raise _lib.Ds2Error(f"load_audio: {path}: unsupported WAV sample format {data.dtype} (supported: int16, "
                            "int32, uint8, float32)")
    scale = _WAV_SCALE[data.dtype]
    x = data.astype(np.float32)
    if scale is not None:
        off, mul = scale
        if off:
            x -= np.float32(off)
        x *= np.float32(mul)                      # powers of two: the same value as torchaudio's division
    if x.ndim == 2:
        x = x[:, 0] if x.shape[1] == 1 else x.mean(axis=1, dtype=np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


def chunk_bounds(n_samples: int, sample_rate: int, chunk_size_seconds: float = -1) -> List[Tuple[int, int]]:
    """[start, end) sample ranges of `AudioParser.get_chunks` (data_loader.py:58-71), with its float expressions:
    the duration rounded up to whole seconds, chunk i = [int(i * chunk * sr), that + int(chunk * sr)), clipped to the
    signal.  Empty chunks are left out (see the module docstring)."""
    if n_samples <= 0:
        raise _lib.Ds2Error("chunk_bounds: the audio has no samples")
    total = math.ceil(n_samples / sample_rate)
    chunk = total if chunk_size_seconds <= 0 else chunk_size_seconds
    out = []
    for i in range(math.ceil(total / chunk)):
        start = int(i * chunk * sample_rate)
        end = min(start + int(chunk * sample_rate), n_samples)
        if end > start:
            out.append((start, end))
    return out


class ChunkSpectrogramParser:
    """data_loader.py:171-186: `parse_audio(path, chunk_size_seconds)` yields the (161, T) spectrogram of each chunk
    in file order, as CUDA tensors.  All chunks of a file are one `ds2_spectrogram_batch` launch, one row per chunk,
    each normalised on its own (like `compute_spectrogram` per chunk); the frames are librosa's centred frames with
    constant padding (librosa >= 0.10)."""

    def __init__(self, audio_conf, normalize: bool = False, device="cuda"):
        self.sample_rate, self.n_fft, self.hop, _ = spect_geometry(audio_conf)
        self.normalize = normalize
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.Ds2Error("ChunkSpectrogramParser: needs a CUDA device; there is no CPU path")
        self._batcher = SpectrogramBatcher(audio_conf, normalize=normalize, device=self.device)

    def spectrograms(self, y: np.ndarray, chunk_size_seconds: float = -1) -> List[torch.Tensor]:
        # every chunk but a clipped last one has int(chunk * sr) samples, so the batcher's stable sort by descending
        # length leaves them in file order: row i is chunk i
        y = np.ascontiguousarray(y, dtype=np.float32)
        bounds = chunk_bounds(len(y), self.sample_rate, chunk_size_seconds)
        out = self._batcher([y[s:e] for s, e in bounds], [()] * len(bounds))[0]
        return [out[i, 0, :, :1 + (e - s) // self.hop] for i, (s, e) in enumerate(bounds)]

    def parse_audio(self, audio_path, chunk_size_seconds: float = -1) -> Iterator[torch.Tensor]:
        yield from self.spectrograms(load_audio(audio_path), chunk_size_seconds)


def run_transcribe(audio_path, spect_parser: ChunkSpectrogramParser, model, decoder, device, precision: int,
                   chunk_size_seconds: float):
    """inference.py:79-99: the chunks' forwards carry the recurrent states `hs`; the outputs are concatenated along
    time (on the device) and decoded.  `precision == 16` runs each forward in the fp16 mode (the reference's
    autocast); otherwise the model's own `precision` applies.  -> decoder.decode(all_outs)."""
    hs = None
    outs = []
    with torch.no_grad():
        for spect in spect_parser.parse_audio(audio_path, chunk_size_seconds):
            spect = spect.contiguous().view(1, 1, spect.size(0), spect.size(1)).to(device)
            input_sizes = torch.IntTensor([spect.size(3)]).int()
            with _lib.autocast(precision):
                out, _, hs = model(spect, input_sizes, hs)
            outs.append(out)
    return decoder.decode(torch.cat(outs, dim=1))


def decode_results(decoded_output: List, decoded_offsets: List, cfg) -> dict:
    """inference.py:15-41: the JSON structure `transcribe` prints (cfg: TranscribeConfig)."""
    dtype = cfg.lm.decoder_type
    results = {
        "output": [],
        "_meta": {
            "acoustic_model": {"path": cfg.model.model_path},
            "language_model": {"path": cfg.lm.lm_path},
            "decoder": {"alpha": cfg.lm.alpha, "beta": cfg.lm.beta,
                        "type": dtype.value if hasattr(dtype, "value") else dtype},
        },
    }
    for b in range(len(decoded_output)):
        for pi in range(min(cfg.lm.top_paths, len(decoded_output[b]))):
            result = {"transcription": decoded_output[b][pi]}
            if cfg.offsets:
                result["offsets"] = decoded_offsets[b][pi].tolist()
            results["output"].append(result)
    return results
