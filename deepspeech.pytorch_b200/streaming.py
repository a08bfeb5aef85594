"""Streaming transcription on the GPU: live audio streams fed a piece at a time and advanced together, one batch per
step, with a unidirectional (Lookahead) model.  Once a frame is decided, its output equals the offline forward of the
whole stream (DESIGN.md §5.11).

    st = StreamingTranscriber(model, GreedyDecoder(labels), max_sessions=128, max_seconds=600.0)
    sid = st.open()                                   # running normalisation; open(mean, std) fixes it
    res = st.step({sid: pcm_chunk}, finish=())        # -> {sid: StreamResult}

Frame rules (spectrogram frame j covers samples [j*hop - n_fft/2, j*hop + n_fft/2)):

* spectrogram frame j is emitted once its last sample has arrived; at finish, frames up to 1 + n // hop with zero
  padding (`spect_frames_ready`);
* conv output u needs spectrogram frames 2u-15 .. 2u+15 (conv1: time kernel 11, stride 2, pad 5; conv2: kernel 11,
  stride 1, pad 5): final once frame 2u+15 exists, or at finish (`conv_outputs_ready`).  Each step's window starts at
  the even frame max(0, 2U - 16), U = the first undecided conv output, which keeps conv1's stride-2 phase; at most 31
  normalised frames are carried to the next step;
* the recurrent stack runs only on the newly final conv outputs, from each layer's carried state;
* head output u is final once recurrent output u + ctx - 1 exists, or at finish (`head_outputs_ready`); the last
  ctx - 1 recurrent outputs are carried.

Normalisation is causal: either fixed (mean, std given at `open`) or running (frame j with the statistics of frames
0..j).  Both deliberately depart from the offline per-utterance statistics, which need the whole stream, and from
`run_transcribe`'s per-chunk statistics.

`StreamCore` is the bookkeeping: it takes the four model blocks as callables, so it runs on the GPU with the library's
ops and on the CPU with the oracle blocks of `oracle/ds2_oracle.py` (tests/test_streaming_host.py).
"""
import functools
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import Ds2Error, check, current_stream, get_lib, ptr
from .configs import is_kind
from .decoder import BeamCTCDecoder, GreedyDecoder
from .input_pipeline import analysis_window, spect_geometry

__all__ = ["StreamingTranscriber", "StreamResult", "StreamCore", "StreamSpectrogram", "StreamBeamSearch",
           "spect_frames_ready",
           "conv_outputs_ready", "head_outputs_ready", "STREAM_SPECT_DTYPE"]

N_FREQ = 161
CONV_FEATURES = 32 * 41
CTX_FRAMES = 32            # room for the <= 31 spectrogram frames a session carries between steps

# Ds2StreamSpect (include/ds2_b200.h)
STREAM_SPECT_DTYPE = np.dtype([("wave_off", "<i8"), ("wave_len", "<i8"), ("base", "<i8"), ("first_frame", "<i8"),
                               ("n_frames", "<i4"), ("slot", "<i4"), ("norm", "<i4"), ("mean", "<f4"),
                               ("std", "<f4"), ("reserved", "<i4", (3,))])
assert STREAM_SPECT_DTYPE.itemsize == 64
NORM_FIXED, NORM_RUNNING, NORM_NONE = 1, 0, -1


def spect_frames_ready(n_samples: int, n_fft: int, hop: int, finished: bool) -> int:
    """spectrogram frames of a stream of n_samples: those whose last sample has arrived, all 1 + n // hop at finish"""
    if finished:
        return 1 + n_samples // hop
    half = n_fft // 2
    return 0 if n_samples < half else (n_samples - half) // hop + 1


def conv_outputs_ready(n_spec: int, finished: bool) -> int:
    """conv outputs final after n_spec spectrogram frames: u with 2u + 15 < n_spec; (n_spec - 1) // 2 + 1 at finish"""
    if finished:
        return (n_spec - 1) // 2 + 1 if n_spec > 0 else 0
    return max(0, (n_spec - 16) // 2 + 1)


def head_outputs_ready(n_rnn: int, ctx: int, finished: bool) -> int:
    """head outputs final after n_rnn recurrent outputs: u with u + ctx - 1 < n_rnn; all n_rnn at finish"""
    return n_rnn if finished else max(0, n_rnn - ctx + 1)


class StreamCore:
    """Window and frame bookkeeping of the streaming forward, for up to `max_sessions` slots.

    Blocks (all on `device`, fp32):
      conv(x (B, 1, 161, T), out_len (B) int32) -> (T', B, 1312), T' = (T - 1) // 2 + 1
      rnn(layer, x (T, B, In), lens (B) int32 descending, h0 (1, B, H), c0 (1, B, H) or None) -> (y, hn, cn)
      lookahead(x (T, B, H)) -> (T, B, H), the Hardtanh included
      head(x (T, B, H)) -> (T, B, C)

    Per-slot state on the device: the carried normalised spectrogram frames, each layer's h (and c), the pending
    recurrent outputs of the lookahead.  Gathering and scattering it takes a fixed number of ops per step."""

    def __init__(self, conv: Callable, rnn: Callable, lookahead: Callable, head: Callable, *, n_layers: int,
                 hidden: int, lstm: bool, context: int, max_sessions: int, device):
        self.conv, self.rnn, self.lookahead, self.head = conv, rnn, lookahead, head
        self.L, self.H, self.lstm, self.ctx, self.S = n_layers, hidden, lstm, context, max_sessions
        self.device = torch.device(device)
        z = dict(device=self.device, dtype=torch.float32)
        S, H = max_sessions, hidden
        self.spec = torch.zeros(S, N_FREQ, CTX_FRAMES, **z)
        self.h = [torch.zeros(S, H, **z) for _ in range(n_layers)]
        self.c = [torch.zeros(S, H, **z) for _ in range(n_layers)] if lstm else None
        self.P = max(context - 1, 1)
        self.pend = torch.zeros(S, self.P, H, **z)
        self.n_spec = [0] * S      # spectrogram frames received
        self.ctx0 = [0] * S        # stream index of the first carried spectrogram frame
        self.U = [0] * S           # conv outputs decided (= recurrent outputs computed)
        self.D = [0] * S           # head outputs decided

    def reset(self, slot: int):
        self.n_spec[slot] = self.ctx0[slot] = self.U[slot] = self.D[slot] = 0

    def _idx(self, a):
        return torch.as_tensor(np.asarray(a, np.int64)).to(self.device, non_blocking=True)

    def step(self, items: Sequence[Tuple[int, int, bool]], new: Optional[torch.Tensor]):
        """items: (slot, new frames, finish) per session, `new` (len(items), 161, Tn) with session i's new normalised
        frames at [i, :, :n_i] (None if no session has any).  -> (out (N, C) or None, [(first head output, count)]
        per item): the newly decided head outputs, session after session in item order."""
        B = len(items)
        slots = [s for s, _, _ in items]
        fresh = [s for s, _, _ in items if self.n_spec[s] == 0 and self.U[s] == 0]
        if fresh:                                    # a session's first step starts from a zero recurrent state
            fi = self._idx(fresh)
            for t in self.h + (self.c or []):
                t.index_fill_(0, fi, 0.0)
        # ---- plan (host integers)
        Tn = 0 if new is None else new.shape[2]
        e = [self.n_spec[s] + n for s, n, _ in items]
        carried = [self.n_spec[s] - self.ctx0[s] for s, _, _ in items]
        U1 = [max(self.U[s], conv_outputs_ready(ei, f)) for (s, _, f), ei in zip(items, e)]
        k = [u1 - self.U[s] for (s, _, _), u1 in zip(items, U1)]
        # ---- spectrogram windows: carried frames | new frames, one source for the conv and the carry
        zc = CTX_FRAMES + Tn                         # index of the zero column
        parts = [self.spec.index_select(0, self._idx(slots))]
        if new is not None:
            parts.append(new)
        parts.append(torch.zeros(B, N_FREQ, 1, device=self.device))
        src = torch.cat(parts, 2)

        def wcol(i, t):                              # source column of window column t of item i
            c, n = carried[i], items[i][1]
            return t if t < c else (CTX_FRAMES + t - c if t - c < n else zc)

        conv_rows = sorted([i for i in range(B) if k[i] > 0], key=lambda i: -k[i])   # stable: ties keep item order
        r_out, col_of = None, {}
        if conv_rows:
            Tw = max(carried[i] + items[i][1] for i in conv_rows)
            widx = [[wcol(i, t) for t in range(Tw)] for i in conv_rows]
            wi = self._idx(widx)[:, None, :].expand(len(conv_rows), N_FREQ, Tw)
            x = torch.gather(src.index_select(0, self._idx(conv_rows)), 2, wi).unsqueeze(1).contiguous()
            out_len = torch.tensor([(carried[i] + items[i][1] - 1) // 2 + 1 for i in conv_rows], dtype=torch.int32)
            y = self.conv(x, out_len.to(self.device))
            Tp, Bc = y.shape[0], y.shape[1]
            K = k[conv_rows[0]]
            zr = Tp * Bc
            ridx = [[(t + self.U[items[i][0]] - self.ctx0[items[i][0]] // 2) * Bc + j if t < k[i] else zr
                     for j, i in enumerate(conv_rows)] for t in range(K)]
            yf = torch.cat([y.reshape(Tp * Bc, CONV_FEATURES), torch.zeros(1, CONV_FEATURES, device=self.device)])
            r = yf.index_select(0, self._idx(ridx).view(-1)).view(K, Bc, CONV_FEATURES)
            lens = torch.tensor([k[i] for i in conv_rows], dtype=torch.int32).to(self.device)
            cs = self._idx([items[i][0] for i in conv_rows])
            for l in range(self.L):
                h0 = self.h[l].index_select(0, cs).unsqueeze(0)
                c0 = self.c[l].index_select(0, cs).unsqueeze(0) if self.lstm else None
                r, hn, cn = self.rnn(l, r, lens, h0, c0)
                self.h[l].index_copy_(0, cs, hn[0])
                if self.lstm:
                    self.c[l].index_copy_(0, cs, cn[0])
            r_out = r
            col_of = {i: j for j, i in enumerate(conv_rows)}
        # ---- lookahead + head on [pending | new] recurrent outputs
        D1 = [max(self.D[s], head_outputs_ready(u1, self.ctx, f)) for (s, _, f), u1 in zip(items, U1)]
        Kr = 0 if r_out is None else r_out.shape[0]
        Bc = 0 if r_out is None else r_out.shape[1]
        zr2 = self.S * self.P + Kr * Bc
        src2 = torch.cat([self.pend.view(self.S * self.P, self.H)]
                         + ([r_out.reshape(Kr * Bc, self.H)] if r_out is not None else [])
                         + [torch.zeros(1, self.H, device=self.device)])

        def rrow(i, u):                              # src2 row of recurrent output u of item i
            s = items[i][0]
            if u < self.U[s]:
                return s * self.P + (u - self.D[s])
            return self.S * self.P + (u - self.U[s]) * Bc + col_of[i] if u < U1[i] else zr2

        la_rows = [i for i in range(B) if D1[i] > self.D[items[i][0]]]
        out, spans = None, [(self.D[s], D1[i] - self.D[s]) for i, (s, _, _) in enumerate(items)]
        if la_rows:
            Tl = max(U1[i] - self.D[items[i][0]] for i in la_rows)
            Bl = len(la_rows)
            lidx = [[rrow(i, self.D[items[i][0]] + t) for i in la_rows] for t in range(Tl)]
            xl = src2.index_select(0, self._idx(lidx).view(-1)).view(Tl, Bl, self.H)
            o = self.head(self.lookahead(xl))
            Cn = o.shape[2]
            oidx = [t * Bl + j for j, i in enumerate(la_rows) for t in range(D1[i] - self.D[items[i][0]])]
            out = o.reshape(Tl * Bl, Cn).index_select(0, self._idx(oidx))
        # ---- carry: the pending recurrent outputs [D1, U1) and the spectrogram frames from max(0, 2 U1 - 16)
        moved = [i for i in range(B) if U1[i] != self.U[items[i][0]] or D1[i] != self.D[items[i][0]]]
        if moved:
            pidx = [[rrow(i, D1[i] + p) if D1[i] + p < U1[i] else zr2 for p in range(self.P)] for i in moved]
            self.pend.index_copy_(0, self._idx([items[i][0] for i in moved]),
                                  src2.index_select(0, self._idx(pidx).view(-1)).view(len(moved), self.P, self.H))
        ctx1 = [max(0, 2 * U1[i] - 16) for i in range(B)]
        keep = [i for i in range(B) if items[i][1] > 0 or ctx1[i] != self.ctx0[items[i][0]]]
        if keep:
            cidx = []
            for i in keep:
                off = ctx1[i] - self.ctx0[items[i][0]]
                n_keep = e[i] - ctx1[i]
                assert n_keep <= CTX_FRAMES or items[i][2]
                cidx.append([wcol(i, off + t) if t < n_keep else zc for t in range(CTX_FRAMES)])
            ci = self._idx(cidx)[:, None, :].expand(len(keep), N_FREQ, CTX_FRAMES)
            self.spec.index_copy_(0, self._idx([items[i][0] for i in keep]),
                                  torch.gather(src.index_select(0, self._idx(keep)), 2, ci))
        for i, (s, n, f) in enumerate(items):
            self.n_spec[s], self.U[s], self.D[s], self.ctx0[s] = e[i], U1[i], D1[i], ctx1[i]
        return out, spans


class StreamSpectrogram:
    """The spectrogram stage: keeps each slot's undecided PCM tail on the host, packs tail + new audio of all
    sessions of a step into one pinned staging buffer (one H2D copy, as `SpectrogramBatcher` does) and runs
    `ds2_spectrogram_stream`.  `norm`: per slot NORM_FIXED (with mean / std), NORM_RUNNING or NORM_NONE."""

    def __init__(self, spect_cfg, max_sessions: int, device="cuda"):
        self.device = torch.device(device)
        self.sample_rate, self.n_fft, self.hop, wname = spect_geometry(spect_cfg)
        if self.n_fft // 2 + 1 != N_FREQ:
            raise Ds2Error(f"streaming: the front-end needs {N_FREQ} frequency bins, got {self.n_fft // 2 + 1}")
        lib = get_lib()
        with torch.cuda.device(self.device):
            self.window = torch.from_numpy(analysis_window(wname, self.n_fft)).to(self.device)
            self.state = torch.zeros(lib.ds2_spectrogram_stream_state_bytes(max_sessions), dtype=torch.uint8,
                                     device=self.device)
        S = max_sessions
        self.n = [0] * S                        # samples received
        self.j = [0] * S                        # frames emitted
        self.tail = [np.zeros(0, np.float32) for _ in range(S)]
        self.base = [0] * S                     # stream index of tail[0]
        self.norm = [(NORM_RUNNING, 0.0, 1.0)] * S
        self._stage, self._staged, self._ws = None, None, None

    def reset(self, slot: int, norm=NORM_RUNNING, mean: float = 0.0, std: float = 1.0):
        self.n[slot] = self.j[slot] = self.base[slot] = 0
        self.tail[slot] = np.zeros(0, np.float32)
        self.norm[slot] = (norm, float(mean), float(std))

    def step(self, items: Sequence[Tuple[int, np.ndarray, bool]]):
        """items: (slot, pcm, finish) -> (frames (len(items), 161, Tcap) CUDA tensor or None, [new frames per item])"""
        B = len(items)
        meta = np.zeros(B, STREAM_SPECT_DTYPE)
        waves, counts, pos = [], [], 0
        half = self.n_fft // 2
        for i, (s, pcm, fin) in enumerate(items):
            buf = np.concatenate([self.tail[s], pcm]) if len(pcm) else self.tail[s]
            n_total = self.n[s] + len(pcm)
            j1 = max(self.j[s], spect_frames_ready(n_total, self.n_fft, self.hop, fin))
            nf = j1 - self.j[s]
            mode, mean, std = self.norm[s]
            meta[i] = (pos, len(buf), self.base[s], self.j[s], nf, s, mode, mean, std, (0, 0, 0))
            waves.append(buf)
            pos += len(buf)
            counts.append(nf)
            nb = max(self.base[s], j1 * self.hop - half)      # first sample frame j1 needs
            self.tail[s] = buf[nb - self.base[s]:].copy()
            self.base[s], self.n[s], self.j[s] = nb, n_total, j1
        Tcap = max(counts)
        if Tcap == 0:
            return None, counts
        lib = get_lib()
        mb = B * STREAM_SPECT_DTYPE.itemsize
        nbytes = mb + 4 * pos
        with torch.cuda.device(self.device):
            if self._staged is not None:
                self._staged.synchronize()          # the previous copy out of the pinned buffer has run
            if self._stage is None or self._stage.numel() < nbytes:
                self._stage = torch.empty(int(nbytes * 1.25) + 4096, dtype=torch.uint8).pin_memory()
            st = self._stage.numpy()
            st[:mb] = meta.view(np.uint8)
            if pos:
                st[mb:nbytes].view(np.float32)[:] = np.concatenate(waves)
            dev = self._stage[:max(nbytes, mb + 4)].to(self.device, non_blocking=True)
            if self._staged is None:
                self._staged = torch.cuda.Event()
            self._staged.record()
            out = torch.empty(B, N_FREQ, Tcap, device=self.device)
            nws = lib.ds2_spectrogram_stream_workspace_bytes(B, Tcap)
            if self._ws is None or self._ws.numel() < nws:
                self._ws = torch.empty(int(nws * 1.25) + 256, dtype=torch.uint8, device=self.device)
            check(lib.ds2_spectrogram_stream(B, ptr(dev[mb:]), ptr(dev), Tcap, self.n_fft, self.hop, ptr(self.window),
                                             ptr(out), Tcap, ptr(self.state), ptr(self._ws), self._ws.numel(),
                                             current_stream()), "ds2_spectrogram_stream")
        return out, counts


class StreamBeamSearch:
    """The resumable beam search of a `BeamCTCDecoder` (`ds2_beam_decode_stream` / `ds2_beam_decode_lm_stream`) for up
    to `max_sessions` slots of at most `max_frames` output frames each: its beam width, cutoffs, alpha, beta and
    language model as they are.  The per-slot node pools and beam lists live on the device across calls."""

    def __init__(self, decoder: BeamCTCDecoder, max_sessions: int, max_frames: int, device="cuda"):
        self.dec, self.S, self.max_frames = decoder, int(max_sessions), int(max_frames)
        self.W = decoder.beam_width
        self.device = torch.device(device)
        lib = get_lib()
        with torch.cuda.device(self.device):
            self.lm = None if decoder.lm is None else decoder.lm.device_tables(self.device)
            nbytes = (lib.ds2_beam_decode_stream_state_bytes if self.lm is None else
                      lib.ds2_beam_decode_lm_stream_state_bytes)(self.S, self.max_frames, self.W)
            if nbytes <= 0:
                raise Ds2Error(f"StreamBeamSearch: no state for max_sessions={max_sessions}, max_frames={max_frames}, "
                               f"beam_width={self.W}")
            self.state = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self._dummy = torch.zeros(1, len(decoder.labels), device=self.device)
        self.frames = [0] * self.S
        self.fresh = set()

    def reset(self, slot: int):
        self.frames[slot] = 0
        self.fresh.add(slot)

    def step(self, probs: Optional[torch.Tensor], items: Sequence[Tuple[int, int, bool]]):
        """probs (N, C) CUDA probabilities of the items' new frames, item after item (None if there are none); items:
        (slot, new frames, final).  -> per item (labels, timesteps, lengths, scores, n_beams) as numpy arrays: all W
        beams of a final item (rows as `decode_beams` gives them), only the current best of the others."""
        W, n = self.W, len(items)
        rec = np.zeros((n, 5), np.int32)
        row = out_row = 0
        for i, (s, k, fin) in enumerate(items):
            if self.frames[s] + k > self.max_frames:
                raise Ds2Error(f"StreamBeamSearch: slot {s} would exceed {self.max_frames} frames")
            rec[i] = (row, k, s, (1 if s in self.fresh else 0) | (2 if fin else 0), out_row)
            row += k
            out_row += W if fin else 1
        Tout = max(1, max(self.frames[s] + k for s, k, _ in items))
        lib, d = get_lib(), self.dec
        with torch.cuda.device(self.device):
            p = self._dummy if probs is None else probs.float().contiguous()
            it = torch.from_numpy(rec).to(self.device)
            labels = torch.empty(out_row, Tout, dtype=torch.int32, device=self.device)
            timesteps = torch.empty_like(labels)
            lengths = torch.empty(out_row, dtype=torch.int32, device=self.device)
            scores = torch.empty(out_row, dtype=torch.float64, device=self.device)
            n_beams = torch.empty(n, dtype=torch.int32, device=self.device)
            common = (ptr(labels), ptr(timesteps), ptr(lengths), ptr(scores), ptr(n_beams), ptr(self.state),
                      self.state.numel(), current_stream())
            if self.lm is None:
                check(lib.ds2_beam_decode_stream(n, p.shape[1], ptr(p), ptr(it), d.blank_index, W, d.cutoff_top_n,
                                                 d.cutoff_prob, self.S, self.max_frames, Tout, *common),
                      "ds2_beam_decode_stream")
            else:
                check(lib.ds2_beam_decode_lm_stream(n, p.shape[1], ptr(p), ptr(it), d.blank_index, W,
                                                    d.cutoff_top_n, d.cutoff_prob, ptr(self.lm), d.lm.order,
                                                    d.alpha, d.beta, d.lm.space, self.S, self.max_frames, Tout,
                                                    *common), "ds2_beam_decode_lm_stream")
            labels, timesteps = labels.cpu().numpy(), timesteps.cpu().numpy()
            lengths, scores, n_beams = lengths.cpu().numpy(), scores.cpu().numpy(), n_beams.cpu().numpy()
        out = []
        for i, (s, k, fin) in enumerate(items):
            r0, r1 = rec[i, 4], rec[i, 4] + (W if fin else 1)
            out.append((labels[r0:r1], timesteps[r0:r1], lengths[r0:r1], scores[r0:r1], int(n_beams[i])))
            self.frames[s] += k
            self.fresh.discard(s)
        return out


@dataclass
class StreamResult:
    text: str                        # greedy: the collapsed labels so far; beam: the current best prefix
    offsets: List[int]               # output frame of each character, counted from the stream start
    frames_decided: int              # output frames final so far
    final: bool
    beams: Optional[list] = None     # beam decoder, on finish: (text, offsets, score) of each of the n_beams beams
    outputs: Optional[torch.Tensor] = field(default=None, repr=False)   # this step's decided head outputs


class StreamingTranscriber:
    """Live sessions of a unidirectional `DeepSpeech` (eval mode), advanced together: `step` runs one spectrogram
    launch, one conv front-end, one call per recurrent layer, one lookahead + head and one decode launch for all the
    sessions it touches.  `precision == 16` selects the fp16 mode for the step, as `forward` does.  `decoder` is a
    `GreedyDecoder` or a `BeamCTCDecoder` (with or without `lm_path`), whose search resumes where the last step
    stopped (`StreamBeamSearch`; its device state is sized from `max_sessions` and `max_seconds`, DESIGN.md §5.11).
    `logits=True` makes the head return logits instead of the softmax (greedy decoding only: the argmax is the
    same)."""

    def __init__(self, model, decoder, max_sessions: int = 128, max_seconds: float = 600.0, *, logits: bool = False):
        if getattr(model, "bidirectional", True) or not is_kind(model.model_cfg, "UniDirectionalConfig"):
            raise Ds2Error("StreamingTranscriber: a bidirectional model has no causal forward; streaming needs a "
                           "UniDirectionalConfig model")
        if model.training:
            raise Ds2Error("StreamingTranscriber: the model must be in eval mode (model.eval())")
        if not isinstance(decoder, (GreedyDecoder, BeamCTCDecoder)):
            raise Ds2Error(f"StreamingTranscriber: unsupported decoder {type(decoder).__name__}; expected this "
                           "package's GreedyDecoder or BeamCTCDecoder")
        if logits and isinstance(decoder, BeamCTCDecoder):
            raise Ds2Error("StreamingTranscriber: the beam search needs probabilities; logits=True is for greedy "
                           "decoding only")
        if max_sessions <= 0 or max_seconds <= 0:
            raise Ds2Error("StreamingTranscriber: max_sessions and max_seconds must be positive")
        self.model, self.decoder = model, decoder
        self.device = next(model.parameters()).device
        if self.device.type != "cuda":
            raise Ds2Error("StreamingTranscriber: the model must be on a CUDA device; there is no CPU path")
        self.max_sessions = int(max_sessions)
        self.spect = StreamSpectrogram(model.spect_cfg, self.max_sessions, self.device)
        self.max_samples = int(max_seconds * self.spect.sample_rate)
        cfg = model.model_cfg
        # the model's blocks in eval mode, whatever model.train() may later set
        blocks = (functools.partial(model.conv_block, training=False),
                  lambda l, x, lens, h0, c0: model.rnn_block(l, x, lens, False, h0, c0), model.lookahead_block,
                  functools.partial(model.head_block, training=False, softmax=not logits))
        self.core = StreamCore(*blocks, n_layers=len(model.rnns), hidden=cfg.hidden_size,
                               lstm=model.rnns[0].rnn_code == _lib.RNN_LSTM, context=cfg.lookahead_context,
                               max_sessions=self.max_sessions, device=self.device)
        self.carry = torch.full((self.max_sessions,), -1, dtype=torch.int32, device=self.device)
        self.beam = None
        if isinstance(decoder, BeamCTCDecoder):
            max_frames = conv_outputs_ready(spect_frames_ready(self.max_samples, self.spect.n_fft, self.spect.hop,
                                                               True), True)
            self.beam = StreamBeamSearch(decoder, self.max_sessions, max_frames, self.device)
        self._free = list(range(self.max_sessions - 1, -1, -1))
        self._slot: Dict[int, int] = {}
        self._text: Dict[int, Tuple[List[str], List[int]]] = {}
        self._fresh = set()
        self._next_id = 0            # ids are never reused: an id below it that has no slot is a finished session

    def open(self, mean: Optional[float] = None, std: Optional[float] = None) -> int:
        """a new session: fixed normalisation (x - mean) / std if both are given, running statistics if neither"""
        if (mean is None) != (std is None):
            raise Ds2Error("StreamingTranscriber.open: give both mean and std, or neither")
        if std is not None and not std > 0:
            raise Ds2Error(f"StreamingTranscriber.open: std must be positive, got {std}")
        if not self._free:
            raise Ds2Error(f"StreamingTranscriber.open: all {self.max_sessions} sessions are open")
        slot = self._free.pop()
        sid = self._next_id
        self._next_id += 1
        self._slot[sid] = slot
        self._text[sid] = ([], [])
        self._fresh.add(slot)
        if self.beam is not None:
            self.beam.reset(slot)
        self.spect.reset(slot, NORM_RUNNING if mean is None else NORM_FIXED, mean or 0.0, std or 1.0)
        self.core.reset(slot)
        return sid

    def _check(self, sid):
        if sid in self._slot:
            return
        if isinstance(sid, int) and 0 <= sid < self._next_id:
            raise Ds2Error(f"StreamingTranscriber: session {sid} is finished")
        raise Ds2Error(f"StreamingTranscriber: unknown session {sid}")

    def step(self, feeds: Dict[int, np.ndarray], finish: Sequence[int] = (), *,
             return_outputs: bool = False) -> Dict[int, StreamResult]:
        """feeds: session -> 1-D float32 PCM at the model's sample rate (any length); finish: sessions to flush and
        close.  -> {session: StreamResult} for every session touched.  Everything is checked before any launch."""
        finish = set(finish)
        sids = list(feeds) + [s for s in finish if s not in feeds]
        pcm = {}
        for sid in sids:
            self._check(sid)
            a = np.asarray(feeds.get(sid, np.zeros(0, np.float32)), dtype=np.float32)
            if a.ndim != 1:
                raise Ds2Error(f"StreamingTranscriber.step: session {sid}: PCM must be 1-D, got shape {a.shape}")
            if self.spect.n[self._slot[sid]] + len(a) > self.max_samples:
                raise Ds2Error(f"StreamingTranscriber.step: session {sid} would exceed max_seconds "
                               f"({self.max_samples} samples)")
            pcm[sid] = a
        if not sids:
            return {}
        slots = [self._slot[s] for s in sids]
        fin = [s in finish for s in sids]
        with _lib.autocast(self.model.precision), torch.no_grad(), torch.cuda.device(self.device):
            fresh = [s for s in slots if s in self._fresh]
            if fresh:
                self.carry.index_fill_(0, torch.tensor(fresh, device=self.device), -1)
                self._fresh.difference_update(fresh)
            frames, counts = self.spect.step([(s, pcm[sid], f) for s, sid, f in zip(slots, sids, fin)])
            out, spans = self.core.step([(s, n, f) for s, n, f in zip(slots, counts, fin)], frames)
            labels = beams = None
            if self.beam is not None:
                beams = self.beam.step(out, [(s, n, f) for s, (_, n), f in zip(slots, spans, fin)])
            elif out is not None:
                rows = np.zeros(len(sids) + 1, np.int32)
                rows[1:] = np.cumsum([n for _, n in spans])
                meta = torch.from_numpy(np.concatenate([rows, np.asarray(slots, np.int32)])).to(self.device)
                lab = torch.empty(out.shape[0], dtype=torch.int32, device=self.device)
                check(get_lib().ds2_greedy_decode_stream(len(sids), out.shape[1], ptr(out), ptr(meta),
                                                         ptr(meta[len(sids) + 1:]), self.decoder.blank_index,
                                                         ptr(self.carry), ptr(lab), current_stream()),
                      "ds2_greedy_decode_stream")
                labels = lab.cpu().numpy()
        res, r0 = {}, 0
        i2c = self.decoder.int_to_char
        for i, sid in enumerate(sids):
            d0, n = spans[i]
            chars, offs = self._text[sid]
            if beams is not None:     # the best prefix can change anywhere: it replaces the previous one
                lab, ts, ln, sc, nb = beams[i]
                chars[:] = [i2c[int(c)] for c in lab[0, :ln[0]]] if nb else []
                offs[:] = [int(t) for t in ts[0, :ln[0]]] if nb else []
            elif n:
                for t in range(n):
                    c = int(labels[r0 + t])
                    if c >= 0:
                        chars.append(self.decoder.int_to_char[c])
                        offs.append(d0 + t)
            res[sid] = StreamResult("".join(chars), list(offs), d0 + n, fin[i],
                                    outputs=out[r0:r0 + n] if return_outputs and out is not None else None)
            if beams is not None and fin[i]:
                res[sid].beams = [("".join(i2c[int(c)] for c in lab[r, :ln[r]]), [int(t) for t in ts[r, :ln[r]]],
                                   float(sc[r])) for r in range(nb)]
            r0 += n
            if fin[i]:
                self._free.append(self._slot.pop(sid))
                del self._text[sid]
        return res
