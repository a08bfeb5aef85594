"""CTC forced alignment on the GPU: where each character and word of a KNOWN transcript lies in the audio.

`forced_align` runs `ds2_ctc_align` (csrc/ctc_align.cu) on a batch: the Viterbi path of each target through the CTC
lattice, in fp64, one CTA per utterance.  `align_audio` aligns one WAV file (the shape of `run_transcribe`);
`align_manifest` aligns every entry of a manifest, a batch per forward and per alignment launch, and writes one JSON
record per utterance in manifest order.

Times are in seconds: output frame f starts at f * 2 * window_stride (the conv front-end halves the frame rate; 20 ms
at the default 10 ms stride).  A character's score is the mean posterior probability of its label over its frames; a
word (a maximal run of non-space characters) scores the frame-weighted mean of its characters; the record's `score`
is the path's total log-probability.  A transcript the audio cannot hold (too few frames for its characters) is
reported with `feasible: false`, `score: null` and no character or word records."""
import json

import torch

from . import _lib
from ._lib import check, current_stream, get_lib, ptr
from .input_pipeline import SpectrogramBatcher

__all__ = ["forced_align", "frame_seconds", "char_scores", "alignment_record", "unsort_rows", "align_audio",
           "align_manifest"]


def forced_align(emissions, input_lengths, targets, target_lengths, blank=0, log_probs=False):
    """Viterbi alignment of each utterance's target.
      emissions      (B,T,C) fp32 CUDA: logits (log_probs=False: the kernel applies the fp32 log-softmax) or
                     log-probabilities (log_probs=True, -inf allowed).  The model's output, a transpose view of a
                     (T,B,C) tensor, is read in place.
      input_lengths  (B) frames per utterance, 0 <= n <= T; frames beyond are never read
      targets        flat (sum of target_lengths) or padded (B, Lmax) label ids, none equal to `blank`
      target_lengths (B)
    -> (frame_labels (B,T) int32 (-1 past the utterance), frame_log_probs (B,T) fp32 (0 there), token_spans
        (B, max(target_lengths), 2) int32 [start, end) frames, scores (B) fp64 path log-probs), on the device.
    An utterance with no finite path gets score -inf and -1 labels and spans; the rest of the batch is aligned."""
    if not (emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3):
        raise _lib.Ds2Error("forced_align: emissions must be a (B, T, C) float32 CUDA tensor")
    B, T, Cn = emissions.shape
    dev = emissions.device
    x = emissions.transpose(0, 1)
    if not x.is_contiguous():
        x = x.contiguous()
    in_len = torch.as_tensor(input_lengths).reshape(-1)
    tgt_len_h = torch.as_tensor(target_lengths).reshape(-1).cpu().long()
    if in_len.numel() != B or tgt_len_h.numel() != B:
        raise _lib.Ds2Error(f"forced_align: {in_len.numel()} input and {tgt_len_h.numel()} target lengths for a "
                            f"batch of {B}")
    in_len_h = in_len.cpu().long()
    if B and (int(in_len_h.min()) < 0 or int(in_len_h.max()) > T or int(tgt_len_h.min()) < 0):
        raise _lib.Ds2Error(f"forced_align: input lengths must lie in [0, T={T}] and target lengths be >= 0")
    max_l = int(tgt_len_h.max()) if B else 0
    targets = torch.as_tensor(targets)
    if targets.dim() == 2:
        if targets.shape[0] != B or targets.shape[1] < max_l:
            raise _lib.Ds2Error(f"forced_align: padded targets {tuple(targets.shape)} for a batch of {B} with "
                                f"targets up to {max_l} long")
        keep = torch.arange(targets.shape[1], device=targets.device)[None, :] < tgt_len_h.to(targets.device)[:, None]
        targets = targets[keep]
    elif targets.dim() != 1 or targets.numel() != int(tgt_len_h.sum()):
        raise _lib.Ds2Error(f"forced_align: flat targets must hold sum(target_lengths) = {int(tgt_len_h.sum())} "
                            f"labels, got shape {tuple(targets.shape)}")
    targets = targets.to(device=dev, dtype=torch.int64).contiguous()
    if targets.numel():
        lo, hi = int(targets.min()), int(targets.max())
        if lo < 0 or hi >= Cn or bool((targets == blank).any()):
            raise _lib.Ds2Error(f"forced_align: target labels must lie in [0, {Cn}) and differ from the blank "
                                f"{blank}")
    with torch.cuda.device(dev):
        in_len_d = in_len_h.to(device=dev, dtype=torch.int32)
        tgt_len_d = tgt_len_h.to(device=dev, dtype=torch.int32)
        labels = torch.empty(B, T, dtype=torch.int32, device=dev)
        frame_lp = torch.empty(B, T, dtype=torch.float32, device=dev)
        spans = torch.empty(B, max_l, 2, dtype=torch.int32, device=dev)
        scores = torch.empty(B, dtype=torch.float64, device=dev)
        if B == 0 or T == 0:      # no frame is read: only empty targets are feasible
            scores.copy_(torch.where(tgt_len_h == 0, 0.0, float("-inf")))
            return labels, frame_lp, spans.fill_(-1), scores
        lib = get_lib()
        nws = lib.ds2_ctc_align_workspace_bytes(T, B, Cn, max_l)
        ws = torch.empty(nws, dtype=torch.uint8, device=dev)
        check(lib.ds2_ctc_align(T, B, Cn, ptr(x), int(not log_probs), ptr(targets) if targets.numel() else None,
                                ptr(in_len_d), ptr(tgt_len_d), max_l, int(blank), ptr(labels), ptr(frame_lp),
                                ptr(spans) if max_l else None, ptr(scores), ptr(ws), nws,
                                current_stream()), "ds2_ctc_align")
    return labels, frame_lp, spans, scores


def frame_seconds(frame, window_stride):
    """seconds at output frame `frame`: the conv front-end's time stride of 2 input frames of `window_stride` s"""
    return frame * 2 * window_stride


def char_scores(frame_log_probs, spans):
    """mean posterior probability exp(log-prob) of each token over its [start, end) frames, on the device:
    (B,T) fp32, (B,L,2) int32 -> (B,L) fp64 (0 for spans of -1)"""
    B, T = frame_log_probs.shape
    cs = torch.zeros(B, T + 1, dtype=torch.float64, device=frame_log_probs.device)
    torch.cumsum(frame_log_probs.double().exp(), dim=1, out=cs[:, 1:])
    st, en = spans[..., 0].long().clamp(min=0), spans[..., 1].long().clamp(min=0)
    n = (en - st).clamp(min=1)
    return (cs.gather(1, en) - cs.gather(1, st)) / n


def alignment_record(text, spans, scores, path_score, frames, window_stride, duration):
    """The record of one utterance from its token spans (host values).
      text        the transcript's tokens, one character each (what the labels kept), spaces included
      spans       per token [start, end) output frames, or -1 when not aligned
      scores      per token mean posterior probability
      path_score  the path's log-probability (-inf: not feasible)
      frames      output frames of the utterance
      duration    the audio's length in seconds: times are clipped to it (the last frame may reach past the end)
    -> {"transcript", "feasible", "score", "frames", "chars": [{char, start, end, score}],
        "words": [{word, start, end, score}]}, times in seconds"""
    feasible = path_score > float("-inf")
    rec = {"transcript": text, "feasible": bool(feasible), "score": float(path_score) if feasible else None,
           "frames": int(frames), "chars": [], "words": []}
    if not feasible:
        return rec
    word = None
    for ch, (s, e), sc in zip(text, spans, scores):
        s, e, sc = int(s), int(e), float(sc)
        start, end = (min(frame_seconds(f, window_stride), duration) for f in (s, e))
        rec["chars"].append({"char": ch, "start": start, "end": end, "score": sc})
        if ch == " ":
            word = None
            continue
        if word is None:
            word = {"word": "", "start": start, "end": 0.0, "score": 0.0, "_n": 0, "_sum": 0.0}
            rec["words"].append(word)
        word["word"] += ch
        word["end"] = end
        word["_n"] += e - s
        word["_sum"] += sc * (e - s)
    for w in rec["words"]:
        n, total = w.pop("_n"), w.pop("_sum")
        w["score"] = total / n if n else 0.0
    return rec


def _records(model, out, output_sizes, targets, target_sizes, texts, n_samples):
    """forced alignment of a batch of the model's logits -> one record per row"""
    labels, frame_lp, spans, scores = forced_align(out, output_sizes, targets, target_sizes, blank=model.blank)
    cscores = char_scores(frame_lp, spans)
    spans_h, cscores_h, scores_h = spans.cpu().tolist(), cscores.cpu().tolist(), scores.cpu().tolist()
    stride = float(model.spect_cfg.window_stride)
    sizes = torch.as_tensor(output_sizes).tolist()
    sr = model.spect_cfg.sample_rate
    return [alignment_record(texts[b], spans_h[b], cscores_h[b], scores_h[b], sizes[b], stride, n_samples[b] / sr)
            for b in range(len(texts))]


def _transcript_labels(transcript, labels):
    """SpectrogramDataset.parse_transcript on a string: newlines removed, characters outside the labels and label 0
    dropped"""
    labels_map = {c: i for i, c in enumerate(labels)}
    return list(filter(None, [labels_map.get(x) for x in transcript.replace("\n", "")]))


@torch.no_grad()
def align_audio(audio_path, transcript, spect_parser, model, device, precision):
    """Aligns `transcript` (a string) to one WAV file with one whole-file forward of `model` (in eval mode).  `precision == 16` runs the
    forward in the fp16 mode, as `run_transcribe` does.  -> the record of `alignment_record`."""
    from .evaluation import model_forward
    from .inference import load_audio
    y = load_audio(audio_path)
    spect = spect_parser.spectrograms(y)[0]
    x = spect.contiguous().view(1, 1, spect.size(0), spect.size(1)).to(device)
    out, output_sizes, _ = model_forward(model, x, torch.IntTensor([spect.size(1)]), precision, logits=True)
    ids = _transcript_labels(transcript, model.labels)
    text = "".join(model.labels[i] for i in ids)
    return _records(model, out, output_sizes, torch.tensor(ids, dtype=torch.int64), [len(ids)], [text], [len(y)])[0]


def unsort_rows(rows, order):
    """rows of a `SpectrogramBatcher` batch (sorted by length: row j holds item order[j], `order` as
    `SpectrogramBatcher.order_and_frames` gives it) -> the same rows in the items' order"""
    out = [None] * len(rows)
    for j, item in enumerate(order):
        out[item] = rows[j]
    return out


@torch.no_grad()
def align_manifest(cfg):
    """Aligns every entry of `cfg.manifest_path` (cfg: AlignConfig) to its transcript: batches of `batch_size` read
    by `AudioDataLoader`'s workers, one forward and one `ds2_ctc_align` per batch.  Writes one JSON record per
    utterance, in manifest order, with `wav_path` and `transcript_path` added, to `cfg.output_path` (JSON lines)
    when it is set.  -> the records."""
    from .evaluation import AudioDataLoader, SpectrogramDataset, load_model, model_forward
    if not cfg.model.cuda:
        raise _lib.Ds2Error("align_manifest: needs a CUDA device (model.cuda = True); there is no CPU path")
    device = torch.device("cuda")
    model = load_model(device=device, model_path=cfg.model.model_path)
    dataset = SpectrogramDataset(audio_conf=model.spect_cfg, input_path=cfg.manifest_path, labels=model.labels,
                                 normalize=True)
    loader = AudioDataLoader(dataset, batch_size=cfg.batch_size, num_workers=cfg.num_workers, shuffle=False)
    batcher = SpectrogramBatcher(model.spect_cfg, normalize=True)
    records = []
    for waves, transcripts in loader.raw_batches():
        inputs, targets, input_percentages, target_sizes = batcher(waves, transcripts)
        order, _ = SpectrogramBatcher.order_and_frames([len(w) for w in waves], batcher.hop)
        input_sizes = input_percentages.mul_(int(inputs.size(3))).int()
        out, output_sizes, _ = model_forward(model, inputs, input_sizes, cfg.model.precision, logits=True)
        texts = ["".join(model.labels[i] for i in transcripts[item]) for item in order]
        rows = _records(model, out, output_sizes, targets, target_sizes, texts, [len(waves[i]) for i in order])
        records.extend(unsort_rows(rows, order))
    for rec, (wav_path, transcript_path) in zip(records, dataset.ids):
        rec["wav_path"], rec["transcript_path"] = str(wav_path), str(transcript_path)
    if cfg.output_path:
        with open(cfg.output_path, "w") as f:
            for rec in records:
                f.write(json.dumps(rec) + "\n")
    return records
