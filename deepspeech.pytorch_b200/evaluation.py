"""Test-set evaluation, the reference's testing.py (`evaluate`), validation.py:135-170 (`run_evaluation`),
utils.py:29-34 (`load_model`) and loader/data_loader.py:190-280 (`SpectrogramDataset`, `AudioDataLoader`), on the GPU.

`run_evaluation` keeps everything but four integers per batch on the device: the best path comes from the greedy
kernel, beam 0 of `ds2_beam_decode`, or the (alpha, beta)-grid beam search with one pair (with a language model), and
`ds2_error_counts` (csrc/error_rate.cu) computes the edit distances the `metrics.py` classes compute from strings.  Any
other decoder object goes through the `metrics.py` classes, as in the reference.

Differences from the reference: audio is read with `inference.load_audio` (WAV only); the rates use `max(1, n)` as
`metrics.py` does where the reference would divide by zero on empty references; noise injection and speed / volume
perturbation are refused by the batcher."""
import json
import os
from pathlib import Path

import torch

from . import _lib
from ._lib import check, current_stream, get_lib, ptr
from .decoder import BeamCTCDecoder, GreedyDecoder, load_decoder
from .inference import load_audio
from .input_pipeline import SpectrogramBatcher
from .metrics import CharErrorRate, WordErrorRate

__all__ = ["SpectrogramDataset", "AudioDataLoader", "load_model", "error_counts", "best_path", "run_evaluation",
           "evaluate", "rates"]


# ---------------------------------------------------------------------------------------------- data
class SpectrogramDataset(torch.utils.data.Dataset):
    """data_loader.py:190-245: items are (waveform fp32 numpy, transcript label ids).  The spectrograms are computed
    by `SpectrogramBatcher` in the loader's main process, so `__getitem__` only reads files and never touches CUDA."""

    def __init__(self, audio_conf, input_path, labels, normalize=False, aug_cfg=None):
        self.ids = self._parse_input(input_path)
        self.size = len(self.ids)
        self.labels_map = dict([(labels[i], i) for i in range(len(labels))])
        self.audio_conf, self.normalize, self.aug_cfg = audio_conf, normalize, aug_cfg

    def __getitem__(self, index):
        audio_path, transcript_path = self.ids[index]
        return load_audio(audio_path), self.parse_transcript(transcript_path)

    @staticmethod
    def _parse_input(input_path):
        """a directory: every `*.wav` below it (rglob order), transcripts at /wav/ -> /txt/, .wav -> .txt; otherwise a
        JSON manifest {root_path, samples: [{wav_path, transcript_path}]}"""
        ids = []
        if os.path.isdir(input_path):
            for wav_path in Path(input_path).rglob('*.wav'):
                transcript_path = str(wav_path).replace('/wav/', '/txt/').replace('.wav', '.txt')
                ids.append((wav_path, transcript_path))
        else:
            with open(input_path) as f:
                manifest = json.load(f)
            for sample in manifest['samples']:
                ids.append((os.path.join(manifest['root_path'], sample['wav_path']),
                            os.path.join(manifest['root_path'], sample['transcript_path'])))
        return ids

    def parse_transcript(self, transcript_path):
        """newlines removed, characters outside the labels dropped, and -- as `filter(None, ...)` does -- label 0"""
        with open(transcript_path, 'r', encoding='utf8') as transcript_file:
            transcript = transcript_file.read().replace('\n', '')
        return list(filter(None, [self.labels_map.get(x) for x in list(transcript)]))

    def __len__(self):
        return self.size


def _collate_files(batch):
    """worker side of the collate: the raw items, in dataset order"""
    return [b[0] for b in batch], [b[1] for b in batch]


class AudioDataLoader(torch.utils.data.DataLoader):
    """data_loader.py:273-280: yields the reference's `(inputs, targets, input_percentages, target_sizes)`, sorted by
    length, with `inputs` already on the current CUDA device.  Worker processes only read files; the spectrograms and
    the padded batch are one `SpectrogramBatcher` call in the main process.  The dataset's `aug_cfg` goes to the
    batcher unchanged."""

    def __init__(self, dataset, *args, **kwargs):
        kwargs["collate_fn"] = _collate_files
        super().__init__(dataset, *args, **kwargs)
        self._batcher = None

    def raw_batches(self):
        """the (waves, transcripts) lists the workers produce, in dataset order within each batch"""
        return super().__iter__()

    def __iter__(self):
        if self._batcher is None:
            ds = self.dataset
            self._batcher = SpectrogramBatcher(ds.audio_conf, normalize=ds.normalize, augmentation_conf=ds.aug_cfg)
        for waves, transcripts in self.raw_batches():
            yield self._batcher(waves, transcripts)


# ---------------------------------------------------------------------------------------------- model
def load_model(device, model_path):
    """utils.py:29-34: a Lightning-layout checkpoint ({state_dict, hyper_parameters = the DeepSpeech constructor
    arguments}) -> DeepSpeech loaded strictly, in eval mode, on `device`"""
    from .model import DeepSpeech
    try:
        ckpt = torch.load(model_path, map_location="cpu", weights_only=False)
    except ModuleNotFoundError as e:
        if (e.name or "").split(".")[0] == "omegaconf":
            raise _lib.Ds2Error(f"load_model: {model_path}: the checkpoint's hyper-parameters are omegaconf objects "
                                "and omegaconf is not installed; install omegaconf to read it") from None
        raise _lib.Ds2Error(f"load_model: {model_path}: cannot read the checkpoint ({e})") from None
    except Exception as e:
        raise _lib.Ds2Error(f"load_model: {model_path}: cannot read the checkpoint ({type(e).__name__}: {e})") \
            from None
    if not isinstance(ckpt, dict) or "state_dict" not in ckpt or "hyper_parameters" not in ckpt:
        raise _lib.Ds2Error(f"load_model: {model_path}: not a checkpoint with 'state_dict' and 'hyper_parameters'")
    hp = ckpt["hyper_parameters"]
    try:
        model = DeepSpeech(labels=hp["labels"], model_cfg=hp["model_cfg"], precision=hp["precision"],
                           optim_cfg=hp["optim_cfg"], spect_cfg=hp["spect_cfg"])
    except KeyError as e:
        raise _lib.Ds2Error(f"load_model: {model_path}: hyper_parameters lack {e}") from None
    model.load_state_dict(ckpt["state_dict"], strict=True)
    return model.eval().to(device)


# ---------------------------------------------------------------------------------------------- device counts
def error_counts(labels, lengths, targets, target_sizes, blank, space, pair_counts=None, rows=True):
    """`ds2_error_counts`: hypotheses labels (K,B,T) or (B,T) int32 and lengths (K,B) / (B) on the device against B
    references (flat int64 targets + per-utterance sizes, host or device).  -> (K,B,4) int64 on the device
    [char_edits, ref_chars, word_edits, ref_words] if `rows`, else None; `pair_counts` ((K,4) int64 on the device)
    is added to."""
    if not labels.is_cuda:
        raise _lib.Ds2Error("error_counts: labels must be a CUDA tensor")
    dev = labels.device
    if labels.dim() == 2:
        labels, lengths = labels[None], lengths[None]
    K, B, T = labels.shape
    labels = labels.to(torch.int32).contiguous()
    lengths = lengths.to(device=dev, dtype=torch.int32).contiguous()
    sizes_h = torch.as_tensor(target_sizes).cpu()
    if sizes_h.numel() != B or tuple(lengths.shape) != (K, B):
        raise _lib.Ds2Error(f"error_counts: {sizes_h.numel()} references and lengths {tuple(lengths.shape)} for "
                            f"labels {tuple(labels.shape)}")
    max_size = int(sizes_h.max()) if B else 0
    targets = torch.as_tensor(targets).to(device=dev, dtype=torch.int64).contiguous()
    sizes = sizes_h.to(device=dev, dtype=torch.int32)
    out = torch.empty(K, B, 4, dtype=torch.int64, device=dev) if rows else None
    if pair_counts is not None and (pair_counts.dtype != torch.int64 or tuple(pair_counts.shape) != (K, 4)
                                    or not pair_counts.is_contiguous() or pair_counts.device != dev):
        raise _lib.Ds2Error(f"error_counts: pair_counts must be a contiguous ({K}, 4) int64 tensor on {dev}")
    lib = get_lib()
    with torch.cuda.device(dev):
        nws = lib.ds2_error_counts_workspace_bytes(K, B, targets.numel(), max_size)
        ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
        check(lib.ds2_error_counts(K, B, T, ptr(labels), ptr(lengths), ptr(targets) if targets.numel() else None,
                                   targets.numel(), ptr(sizes), max_size, int(blank), int(space), ptr(out),
                                   ptr(pair_counts), ptr(ws), nws, current_stream()), "ds2_error_counts")
    return out


def rates(counts):
    """[char_edits, ref_chars, word_edits, ref_words] (host ints) -> (wer, cer), metrics.py's expression"""
    ce, nc, we, nw = (int(x) for x in counts)
    return float(we) / max(1, nw) * 100, float(ce) / max(1, nc) * 100


def _space_of(labels):
    labels = list(labels)
    return labels.index(' ') if ' ' in labels else len(labels)


def best_path(decoder, probs, sizes):
    """the best path of `decoder` on the device: -> labels (B,T) int32, lengths (B) int32, CUDA.  GreedyDecoder: the
    greedy kernel; BeamCTCDecoder: beam 0 of `ds2_beam_decode`, or of the grid search with the decoder's (alpha,
    beta) when it has a language model"""
    probs = probs.to(torch.float32).contiguous()
    sz = None if sizes is None else torch.as_tensor(sizes).to(device=probs.device, dtype=torch.int32).contiguous()
    if isinstance(decoder, BeamCTCDecoder):
        if decoder.lm is not None:
            labels, lengths = decoder.decode_best_grid(probs, sz, [(decoder.alpha, decoder.beta)])
            return labels[0], lengths[0]
        return decoder.decode_best(probs, sz)
    labels, _, counts = decoder.decode_indices_device(probs, sz)
    return labels, counts


def _on_device_path(decoder, target_decoder):
    return (type(decoder) in (GreedyDecoder, BeamCTCDecoder) and isinstance(target_decoder, GreedyDecoder)
            and list(decoder.labels) == list(target_decoder.labels))


def model_forward(model, inputs, input_sizes, precision, logits=False):
    """the eval forward of validation.py:160-161: precision 16 runs in the library's fp16 mode (the reference's
    autocast), as run_transcribe does.  `logits=True` returns the logits instead of the eval softmax."""
    with _lib.autocast(precision):
        return model(inputs, input_sizes, logits=logits)


@torch.no_grad()
def run_evaluation(test_loader, model, decoder, device, target_decoder, precision):
    """validation.py:135-170 -> (wer, cer) in percent.  For this package's GreedyDecoder and BeamCTCDecoder only the
    four counts per batch leave the GPU (at the end); any other decoder goes through metrics.py's classes."""
    model.eval()
    on_device = _on_device_path(decoder, target_decoder)
    if not on_device:
        wer = WordErrorRate(decoder=decoder, target_decoder=target_decoder)
        cer = CharErrorRate(decoder=decoder, target_decoder=target_decoder)
    counts = None
    for inputs, targets, input_percentages, target_sizes in test_loader:
        input_sizes = input_percentages.mul_(int(inputs.size(3))).int()
        inputs = inputs.to(device)
        out, output_sizes, _ = model_forward(model, inputs, input_sizes, precision)
        if on_device:
            if counts is None:
                counts = torch.zeros(1, 4, dtype=torch.int64, device=out.device)
            labels, lengths = best_path(decoder, out, output_sizes)
            error_counts(labels, lengths, targets, target_sizes, target_decoder.blank_index,
                         _space_of(target_decoder.labels), pair_counts=counts, rows=False)
        else:
            wer.update(preds=out, preds_sizes=output_sizes, targets=targets, target_sizes=target_sizes)
            cer.update(preds=out, preds_sizes=output_sizes, targets=targets, target_sizes=target_sizes)
    if not on_device:
        return wer.compute(), cer.compute()
    return rates([0, 0, 0, 0] if counts is None else counts[0].tolist())


@torch.no_grad()
def evaluate(cfg):
    """testing.py:11-54 (cfg: EvalConfig): prints the "Test Summary" line and returns (wer, cer)"""
    device = torch.device("cuda" if cfg.model.cuda else "cpu")
    model = load_model(device=device, model_path=cfg.model.model_path)
    decoder = load_decoder(labels=model.labels, cfg=cfg.lm)
    target_decoder = GreedyDecoder(labels=model.labels, blank_index=model.labels.index('_'))
    test_dataset = SpectrogramDataset(audio_conf=model.spect_cfg, input_path=cfg.test_path, labels=model.labels,
                                      normalize=True)
    test_loader = AudioDataLoader(test_dataset, batch_size=cfg.batch_size, num_workers=cfg.num_workers)
    wer, cer = run_evaluation(test_loader=test_loader, device=device, model=model, decoder=decoder,
                              target_decoder=target_decoder, precision=cfg.model.precision)
    print('Test Summary \t'
          'Average WER {wer:.3f}\t'
          'Average CER {cer:.3f}\t'.format(wer=wer, cer=cer))
    return wer, cer
