"""Greedy CTC decoding on the GPU (SURVEY.md §8f row N2): argmax -> collapse repeats -> drop blank,
with per-character frame offsets — the integer result of the reference's
deepspeech_pytorch/decoder.py:121-181 (GreedyDecoder), bit-exact."""
import torch

from . import _lib
from ._lib import check, get_lib, ptr


class GreedyDecoder:
    def __init__(self, labels, blank_index=0):
        self.labels = labels
        self.int_to_char = dict(enumerate(labels))
        self.blank_index = blank_index
        self.space_index = labels.index(' ') if ' ' in labels else len(labels)

    def decode_indices(self, probs, sizes=None):
        """probs (B,T,C) CUDA -> (labels (B,T) int32, offsets (B,T) int32, counts (B) int32) on the CPU"""
        if not probs.is_cuda:
            raise _lib.Ds2Error("GreedyDecoder: probs must be a CUDA tensor")
        import ctypes as C
        probs = probs.float().contiguous()
        B, T, Cn = probs.shape
        dev = probs.device
        labels = torch.zeros(B, T, dtype=torch.int32, device=dev)
        offsets = torch.zeros(B, T, dtype=torch.int32, device=dev)
        counts = torch.zeros(B, dtype=torch.int32, device=dev)
        sz = None if sizes is None else torch.as_tensor(sizes).int().to(dev)
        with torch.cuda.device(dev):                         # launches bind to the current device
            check(get_lib().ds2_greedy_decode(B, T, Cn, ptr(probs), ptr(sz), self.blank_index, ptr(labels),
                                              ptr(offsets), ptr(counts),
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  "ds2_greedy_decode")
        return labels.cpu(), offsets.cpu(), counts.cpu()

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
