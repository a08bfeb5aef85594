"""CTC decoding on the GPU.

GreedyDecoder (SURVEY.md §8f row N2): argmax -> collapse repeats -> drop blank, with per-character frame offsets — the
integer result of the reference's deepspeech_pytorch/decoder.py:121-181 (GreedyDecoder), bit-exact.

BeamCTCDecoder (rows N5, N6): prefix beam search, without or with an ARPA n-gram language model (`lm_path`), with the
reference's constructor and return shapes (decoder.py:56-118) and `load_decoder` (utils.py:37-54).  The search is
defined by the rules in csrc/beam_decode.cu (DESIGN.md §5.7); ctcdecode and KenLM themselves are not pinned."""
import torch

from . import _lib
from ._lib import check, current_stream, get_lib, ptr


class GreedyDecoder:
    def __init__(self, labels, blank_index=0):
        self.labels = labels
        self.int_to_char = dict(enumerate(labels))
        self.blank_index = blank_index
        self.space_index = labels.index(' ') if ' ' in labels else len(labels)

    def decode_indices(self, probs, sizes=None):
        """probs (B,T,C) CUDA -> (labels (B,T) int32, offsets (B,T) int32, counts (B) int32) on the CPU"""
        labels, offsets, counts = self.decode_indices_device(probs, sizes)
        return labels.cpu(), offsets.cpu(), counts.cpu()

    def decode_indices_device(self, probs, sizes=None):
        """`decode_indices` left on the device: the first counts[b] entries of row b are set, the rest are 0"""
        if not probs.is_cuda:
            raise _lib.Ds2Error("GreedyDecoder: probs must be a CUDA tensor")
        probs = probs.float().contiguous()
        B, T, Cn = probs.shape
        dev = probs.device
        labels = torch.zeros(B, T, dtype=torch.int32, device=dev)
        offsets = torch.zeros(B, T, dtype=torch.int32, device=dev)
        counts = torch.zeros(B, dtype=torch.int32, device=dev)
        sz = None if sizes is None else torch.as_tensor(sizes).int().to(dev)
        with torch.cuda.device(dev):                         # launches bind to the current device
            check(get_lib().ds2_greedy_decode(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, ptr(labels),
                                              ptr(offsets), ptr(counts), current_stream()), "ds2_greedy_decode")
        return labels, offsets, counts

    def convert_to_strings(self, sequences, sizes=None, remove_repetitions=False, return_offsets=False):
        """label-index sequences -> [[str]] (decoder.py:125-163): blanks dropped, optional repeat collapsing; used by
        the WER/CER accumulators for the reference transcripts (host integers, tiny)"""
        strings, offsets = [], []
        blank = self.int_to_char[self.blank_index]
        for x in range(len(sequences)):
            seq = [int(v) for v in sequences[x]]
            n = int(sizes[x]) if sizes is not None else len(seq)
            out, offs = [], []
            for i in range(n):
                ch = self.int_to_char[seq[i]]
                if ch == blank or (remove_repetitions and i != 0 and seq[i] == seq[i - 1]):
                    continue
                out.append(ch)
                offs.append(i)
            strings.append([''.join(out)])
            offsets.append([torch.tensor(offs, dtype=torch.int)])
        return (strings, offsets) if return_offsets else strings

    def decode(self, probs, sizes=None):
        """same return shape as the reference: (strings [[str]], offsets [[IntTensor]])"""
        labels, offsets, counts = self.decode_indices(probs, sizes)
        strings, offs = [], []
        for b in range(labels.size(0)):
            n = int(counts[b])
            strings.append([''.join(self.int_to_char[int(c)] for c in labels[b, :n])])
            offs.append([offsets[b, :n].clone()])
        return strings, offs


class BeamCTCDecoder:
    """decoder.py:56-118 on the GPU.  Without `lm_path` this is `ds2_beam_decode` and `alpha` / `beta` have no
    effect, as in ctcdecode without a scorer.  With `lm_path`, an ARPA n-gram model (plain or gzip'd) is parsed here
    and the search is `ds2_beam_decode_lm` (rules L0-L5 of csrc/beam_decode.cu): words restricted to the model's
    vocabulary, alpha * log10 p + beta added at every completed word.  `num_processes` is ignored."""

    def __init__(self, labels, lm_path=None, alpha=0, beta=0, cutoff_top_n=40, cutoff_prob=1.0, beam_width=100,
                 num_processes=4, blank_index=0):
        self.labels = list(labels)
        self.int_to_char = dict(enumerate(self.labels))
        self.blank_index = blank_index
        self.space_index = self.labels.index(' ') if ' ' in self.labels else len(self.labels)
        self.alpha, self.beta, self.num_processes = float(alpha), float(beta), num_processes
        self.cutoff_top_n, self.cutoff_prob, self.beam_width = int(cutoff_top_n), float(cutoff_prob), int(beam_width)
        self.lm = None
        if lm_path:
            from .lm import LanguageModel
            self.lm = LanguageModel(lm_path, self.labels, blank_index)
        self._decoder = self          # the reference's search_lm_params.py calls decoder._decoder.reset_params

    def reset_params(self, alpha, beta):
        """ctcdecode's CTCBeamDecoder.reset_params: the language-model weight and word bonus of later decodes"""
        self.alpha, self.beta = float(alpha), float(beta)

    def decode_beams(self, probs, sizes=None):
        """probs (B,T,C) fp32 probabilities (a CPU tensor is copied to the current CUDA device) -> on the CPU:
        labels (B,W,T) int32, scores (B,W) float64 (-log-likelihood, +inf for unused slots), timesteps (B,W,T) int32,
        lengths (B,W) int32, n_beams (B) int32.  With a language model the scores include its terms (rule L5)"""
        if probs.dim() != 3:
            raise _lib.Ds2Error(f"BeamCTCDecoder: probs must be (B, T, C), got {tuple(probs.shape)}")
        if sizes is not None:                                # the kernel reads one length per utterance
            sizes = torch.as_tensor(sizes)
            if sizes.dim() != 1 or sizes.numel() != probs.size(0):
                raise _lib.Ds2Error(f"BeamCTCDecoder: sizes must hold one length per utterance (B = {probs.size(0)}),"
                                    f" got shape {tuple(sizes.shape)}")
        dev = probs.device if probs.is_cuda else torch.device("cuda", torch.cuda.current_device())
        probs = probs.to(device=dev, dtype=torch.float32).contiguous()
        B, T, Cn = probs.shape
        W = self.beam_width
        lib = get_lib()
        with torch.cuda.device(dev):                         # launches bind to the current device
            Wa = max(W, 1)                                   # the library refuses a bad width with a message
            lm = None if self.lm is None else self.lm.device_tables(dev)
            nws = (lib.ds2_beam_decode_workspace_bytes if lm is None else lib.ds2_beam_decode_lm_workspace_bytes)(
                B, T, Cn, W)
            ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
            labels = torch.empty(B, Wa, T, dtype=torch.int32, device=dev)
            timesteps = torch.empty_like(labels)
            lengths = torch.empty(B, Wa, dtype=torch.int32, device=dev)
            scores = torch.empty(B, Wa, dtype=torch.float64, device=dev)
            n_beams = torch.empty(B, dtype=torch.int32, device=dev)
            sz = None if sizes is None else sizes.to(device=dev, dtype=torch.int32).contiguous()
            stream = current_stream()
            if lm is None:
                check(lib.ds2_beam_decode(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, W, self.cutoff_top_n,
                                          self.cutoff_prob, ptr(labels), ptr(timesteps), ptr(lengths), ptr(scores),
                                          ptr(n_beams), ptr(ws), nws, stream), "ds2_beam_decode")
            else:
                check(lib.ds2_beam_decode_lm(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, W, self.cutoff_top_n,
                                             self.cutoff_prob, ptr(lm), self.lm.order, self.alpha, self.beta,
                                             self.lm.space, ptr(labels), ptr(timesteps), ptr(lengths), ptr(scores),
                                             ptr(n_beams), ptr(ws), nws, stream), "ds2_beam_decode_lm")
        return labels.cpu(), scores.cpu(), timesteps.cpu(), lengths.cpu(), n_beams.cpu()

    def decode_best(self, probs, sizes=None):
        """beam 0 of `decode_beams` left on the device: probs (B,T,C) CUDA -> labels (B,T) int32, lengths (B) int32"""
        if self.lm is not None:
            labels, lengths = self.decode_best_grid(probs, sizes, [(self.alpha, self.beta)])
            return labels[0], lengths[0]
        probs = probs.to(torch.float32).contiguous()
        B, T, Cn = probs.shape
        dev, W = probs.device, self.beam_width
        lib = get_lib()
        with torch.cuda.device(dev):
            Wa = max(W, 1)
            nws = lib.ds2_beam_decode_workspace_bytes(B, T, Cn, W)
            ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
            labels = torch.empty(B, Wa, T, dtype=torch.int32, device=dev)
            timesteps = torch.empty_like(labels)
            lengths = torch.empty(B, Wa, dtype=torch.int32, device=dev)
            scores = torch.empty(B, Wa, dtype=torch.float64, device=dev)
            n_beams = torch.empty(B, dtype=torch.int32, device=dev)
            sz = None if sizes is None else torch.as_tensor(sizes).to(device=dev, dtype=torch.int32).contiguous()
            check(lib.ds2_beam_decode(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, W, self.cutoff_top_n,
                                      self.cutoff_prob, ptr(labels), ptr(timesteps), ptr(lengths), ptr(scores),
                                      ptr(n_beams), ptr(ws), nws, current_stream()), "ds2_beam_decode")
        return labels[:, 0].contiguous(), lengths[:, 0].contiguous()

    def decode_best_grid(self, probs, sizes, pairs):
        """`ds2_beam_decode_lm_grid`: the best beam for each of K (alpha, beta) pairs in one launch.  probs (B,T,C)
        CUDA, sizes (B) or None, pairs K x (alpha, beta) -> labels (K,B,T) int32, lengths (K,B) int32 on the device;
        (k, b) is beam 0 of `decode_beams` after `reset_params(*pairs[k])`.  Pass the utterances longest first: the
        items start in utterance order."""
        import ctypes as C
        import numpy as np
        if self.lm is None:
            raise _lib.Ds2Error("BeamCTCDecoder.decode_best_grid: needs a language model (lm_path)")
        pr = np.ascontiguousarray(np.asarray(pairs, dtype=np.float64).reshape(-1, 2))
        if pr.shape[0] < 1:
            raise _lib.Ds2Error("BeamCTCDecoder.decode_best_grid: K = 0 (alpha, beta) pairs")
        if not np.all(np.isfinite(pr)):
            raise _lib.Ds2Error(f"BeamCTCDecoder.decode_best_grid: alpha and beta must be finite, got "
                                f"{pr[~np.all(np.isfinite(pr), axis=1)].tolist()}")
        if not probs.is_cuda:
            raise _lib.Ds2Error("BeamCTCDecoder.decode_best_grid: probs must be a CUDA tensor")
        probs = probs.to(torch.float32).contiguous()
        B, T, Cn = probs.shape
        K, dev, W = pr.shape[0], probs.device, self.beam_width
        lib = get_lib()
        with torch.cuda.device(dev):
            lm = self.lm.device_tables(dev)
            nws = lib.ds2_beam_decode_lm_grid_workspace_bytes(B, T, Cn, W, K)
            ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
            labels = torch.empty(K, B, T, dtype=torch.int32, device=dev)
            lengths = torch.empty(K, B, dtype=torch.int32, device=dev)
            sz = None if sizes is None else torch.as_tensor(sizes).to(device=dev, dtype=torch.int32).contiguous()
            check(lib.ds2_beam_decode_lm_grid(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, W, self.cutoff_top_n,
                                              self.cutoff_prob, ptr(lm), self.lm.order, K,
                                              pr.ctypes.data_as(C.c_void_p), self.lm.space, ptr(labels),
                                              ptr(lengths), ptr(ws), nws, current_stream()), "ds2_beam_decode_lm_grid")
        return labels, lengths

    def convert_to_strings(self, out, seq_len):
        """decoder.py:79-91: [[str]] over utterances and beams, '' where the length is 0"""
        results = []
        for b, batch in enumerate(out):
            utterances = []
            for p, utt in enumerate(batch):
                size = int(seq_len[b][p])
                utterances.append(''.join(self.int_to_char[int(x)] for x in utt[0:size]) if size > 0 else '')
            results.append(utterances)
        return results

    def convert_tensor(self, offsets, sizes):
        """decoder.py:93-104: [[IntTensor]], empty where the length is 0"""
        results = []
        for b, batch in enumerate(offsets):
            utterances = []
            for p, utt in enumerate(batch):
                size = int(sizes[b][p])
                utterances.append(utt[0:size] if size > 0 else torch.tensor([], dtype=torch.int))
            results.append(utterances)
        return results

    def decode(self, probs, sizes=None):
        """same return shape as the reference: (strings [[W str]], offsets [[W IntTensor]]), best beam first"""
        out, _, offsets, seq_lens, _ = self.decode_beams(probs, sizes)
        return self.convert_to_strings(out, seq_lens), self.convert_tensor(offsets, seq_lens)


def load_decoder(labels, cfg):
    """utils.py:37-54 without hydra: `cfg` is an LMConfig (this package's or the reference's)"""
    kind = getattr(cfg.decoder_type, "value", cfg.decoder_type)
    if kind == "beam":
        return BeamCTCDecoder(labels=labels, lm_path=cfg.lm_path, alpha=cfg.alpha, beta=cfg.beta,
                              cutoff_top_n=cfg.cutoff_top_n, cutoff_prob=cfg.cutoff_prob, beam_width=cfg.beam_width,
                              num_processes=cfg.lm_workers, blank_index=labels.index('_'))
    return GreedyDecoder(labels=labels, blank_index=labels.index('_'))
