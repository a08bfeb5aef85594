"""CPU checks of the streaming transcriber's bookkeeping: the frame-count rules over many chunkings, `StreamCore`
driven by the oracle's blocks against the oracle's offline forward of the whole normalised spectrogram, the refusals
made before a device is needed, and the state sizes.  The session refusals (unknown, finished, capacity, max_seconds)
need a transcriber, which needs a CUDA model: tests/test_gpu_streaming.py checks them."""
import random

import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.streaming import (StreamCore, conv_outputs_ready, head_outputs_ready,
                                               spect_frames_ready)
from oracle import ds2_oracle as O

N_FFT, HOP = 320, 160


def _chunkings(n, rng):
    """feed lengths (in samples) summing to n: 1-sample feeds, empty feeds, feeds shorter than a hop, random"""
    yield [1] * min(n, 400) + ([n - 400] if n > 400 else [])
    yield [0, 0] + [n] + [0]
    out, left = [], n
    while left > 0:
        c = min(left, rng.randrange(0, HOP))
        out.append(c)
        left -= c
    yield out
    out, left = [], n
    while left > 0:
        c = min(left, rng.randrange(1, 8000))
        out.append(c)
        left -= c
    yield out


@pytest.mark.parametrize("n", [0, 1, 159, 160, 161, 2399, 2400, 4801, 16000, 16001, 33333])
@pytest.mark.parametrize("finish_with_last", [True, False])
def test_frame_counts_follow_the_closed_forms(n, finish_with_last):
    rng = random.Random(n)
    for feeds in _chunkings(n, rng):
        feeds = feeds or [0]
        got = 0
        spec = conv = head = 0
        for i, f in enumerate(feeds):
            got += f
            last = finish_with_last and i == len(feeds) - 1
            s1 = max(spec, spect_frames_ready(got, N_FFT, HOP, last))
            assert s1 == (1 + got // HOP if last else (max(0, (got - N_FFT // 2) // HOP + 1)
                                                       if got >= N_FFT // 2 else 0))
            # a frame is emitted once its last sample has arrived
            assert last or s1 == 0 or (s1 - 1) * HOP + N_FFT // 2 <= got
            c1 = max(conv, conv_outputs_ready(s1, last))
            assert last or c1 == 0 or 2 * (c1 - 1) + 15 <= s1 - 1
            h1 = max(head, head_outputs_ready(c1, 20, last))
            spec, conv, head = s1, c1, h1
        if not finish_with_last:
            spec = max(spec, spect_frames_ready(got, N_FFT, HOP, True))
            conv = max(conv, conv_outputs_ready(spec, True))
            head = max(head, head_outputs_ready(conv, 20, True))
        assert spec == 1 + n // HOP
        assert conv == (spec - 1) // 2 + 1 == int(O.get_seq_lens(torch.tensor([spec]))[0])
        assert head == conv


def test_algorithmic_latency_at_context_20():
    """head output u is decided once spectrogram frame 2u + 53 exists: 2u + 15 for the conv output u + 19"""
    for u in range(0, 50):
        spec = next(e for e in range(1, 1000) if head_outputs_ready(conv_outputs_ready(e, False), 20, False) > u)
        assert spec - 1 == 2 * u + 15 + 2 * 19
        # its centre is frame 2u: 53 frames later, plus the n_fft/2 samples that frame needs (0.54 s at 10 ms)


def _oracle_blocks(P, ocfg):
    lstm = ocfg.rnn_type == "lstm"

    def conv(x, out_len):
        y = O.conv_frontend(x, out_len, P, False, {})
        B, Cc, Dd, Tp = y.shape
        return y.reshape(B, Cc * Dd, Tp).permute(2, 0, 1)

    def rnn(l, x, lens, h0, c0):
        y, h = O.batch_rnn(x, lens, P, f"rnns.{l}.", ocfg, batch_norm=l > 0, training=False, new_buffers={},
                           h0=(h0, c0) if lstm else h0)
        return (y, h[0], h[1]) if lstm else (y, h, None)

    def lookahead(x):
        return torch.clamp(O.lookahead(x, P["lookahead.0.conv.weight"]), 0.0, 20.0)

    def head(x):
        return torch.softmax(O.fc_head(x, P, False, {}), -1)

    return conv, rnn, lookahead, head


def _perturbed_params(ocfg, seed):
    P = O.init_params(ocfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in list(P):
        if k.endswith("running_mean"):
            P[k] = 0.1 * torch.randn(P[k].shape, generator=g)
        elif k.endswith("running_var"):
            P[k] = 0.5 + torch.rand(P[k].shape, generator=g)
    return P


def _split(n, rng, kind):
    if kind == "ones":
        return [1] * n
    if kind == "whole":
        return [n]
    out, left = [], n
    while left > 0:
        c = min(left, rng.randrange(0, 40))
        out.append(c)
        left -= c
    return out


@pytest.mark.parametrize("rnn_type", ["gru", "lstm", "rnn"])
@pytest.mark.parametrize("ctx", [5, 20])
def test_core_with_oracle_blocks_equals_offline_forward(rnn_type, ctx):
    torch.manual_seed(0)
    H, layers = 16, 2
    ocfg = O.OracleConfig(rnn_type=rnn_type, hidden_size=H, hidden_layers=layers, bidirectional=False,
                          lookahead_context=ctx)
    P = _perturbed_params(ocfg, 7)
    rng = random.Random(ctx)
    lengths = [1, 9, 15, 16, 17, 40, 95]                # spectrogram frames; < 16 is shorter than the receptive field
    kinds = ["ones", "whole", "random", "random", "ones", "random", "random"]
    specs = [torch.randn(161, n, generator=torch.Generator().manual_seed(n)) for n in lengths]
    feeds = [_split(n, rng, kd) for n, kd in zip(lengths, kinds)]
    core = StreamCore(*_oracle_blocks(P, ocfg), n_layers=layers, hidden=H, lstm=rnn_type == "lstm", context=ctx,
                      max_sessions=10, device="cpu")
    slots = [9, 0, 3, 4, 5, 6, 7]
    for s in slots:
        core.reset(s)
    got = [[] for _ in lengths]
    pos = [0] * len(lengths)
    step = 0
    # sessions start at different steps and finish at different steps (finish with and without a last feed)
    while any(pos[i] <= len(feeds[i]) for i in range(len(lengths))):
        items, new = [], []
        for i in range(len(lengths)):
            if step < i or pos[i] > len(feeds[i]):
                continue
            if pos[i] == len(feeds[i]):
                n, fin = 0, True
            else:
                n = feeds[i][pos[i]]
                fin = (i % 2 == 0) and pos[i] == len(feeds[i]) - 1
            done = sum(feeds[i][:pos[i]])
            new.append(specs[i][:, done:done + n])
            items.append((i, slots[i], n, fin))
            pos[i] += 2 if fin and pos[i] < len(feeds[i]) else 1
        step += 1
        if not items:
            continue
        Tn = max(x.shape[1] for x in new)
        nt = torch.zeros(len(items), 161, max(Tn, 1))
        for j, x in enumerate(new):
            nt[j, :, :x.shape[1]] = x
        before = [core.D[s] for _, s, _, _ in items]
        out, spans = core.step([(s, n, f) for _, s, n, f in items], nt if Tn else None)
        r = 0
        for j, (i, s, n, f) in enumerate(items):
            d0, cnt = spans[j]
            assert d0 == before[j]
            got[i].append(out[r:r + cnt] if cnt else torch.zeros(0, 29))
            r += cnt
            if f:
                assert core.D[s] == (lengths[i] - 1) // 2 + 1
        assert out is None or r == out.shape[0]
    for i, n in enumerate(lengths):
        ref, _, _, _ = O.forward(specs[i][None, None], torch.tensor([n]), P, ocfg, training=False)
        stream = torch.cat(got[i])
        assert stream.shape == ref[0].shape, (i, stream.shape, ref.shape)
        err = float((stream - ref[0]).abs().max() / ref[0].abs().max())
        assert err < 1e-5, (rnn_type, ctx, n, err)


def test_refusals_without_a_gpu():
    uni = ds.UniDirectionalConfig(hidden_size=8, hidden_layers=1, lookahead_context=5)
    bi = ds.BiDirectionalConfig(hidden_size=8, hidden_layers=1)
    m_bi = ds.DeepSpeech(ds.LABELS, bi, 32, ds.AdamConfig(), ds.SpectConfig()).eval()
    m_uni = ds.DeepSpeech(ds.LABELS, uni, 32, ds.AdamConfig(), ds.SpectConfig()).eval()
    with pytest.raises(ds.Ds2Error, match="bidirectional"):
        ds.StreamingTranscriber(m_bi, ds.GreedyDecoder(ds.LABELS))
    with pytest.raises(ds.Ds2Error, match="decoder"):
        ds.StreamingTranscriber(m_uni, object())
    with pytest.raises(ds.Ds2Error, match="probabilities"):
        ds.StreamingTranscriber(m_uni, ds.BeamCTCDecoder(ds.LABELS), logits=True)
    with pytest.raises(ds.Ds2Error, match="eval"):
        ds.StreamingTranscriber(m_uni.train(), ds.GreedyDecoder(ds.LABELS))


@pytest.mark.parametrize("S,nbytes", [(1, 256), (128, 2048), (129, 2304)])
def test_spectrogram_stream_state_bytes(S, nbytes):
    assert ds.get_lib().ds2_spectrogram_stream_state_bytes(S) == nbytes        # 16 bytes per slot, 256-aligned


@pytest.mark.parametrize("B,T,nbytes", [(1, 1, 256), (7, 33, 3840), (128, 32, 65536), (3, 1000, 48128)])
def test_spectrogram_stream_workspace_bytes(B, T, nbytes):
    assert ds.get_lib().ds2_spectrogram_stream_workspace_bytes(B, T) == nbytes  # 16 bytes per frame, 256-aligned


def _pool_bytes(S, T, W, lm):
    """carve_pool + the list records of csrc/beam_decode.cu: every array rounded up to 256 bytes"""
    a = lambda x: (x + 255) // 256 * 256
    NP = T * W + 1
    HC = 1
    while HC < 2 * NP:
        HC <<= 1
    n, h = S * NP, S * HC
    pool = 4 * a(4 * n) + a(8 * n) + a(8 * h) + a(4 * h) + (a(8 * n) if lm else 0)
    rec = a(16 + W * (4 * 8 + 2 * 8 + 5 * 4) + W * 4 * 4)      # LM_CTX = 4 context words per slot
    return pool + a(S * rec)


@pytest.mark.parametrize("S,T,W", [(1, 1, 1), (3, 50, 8), (128, 30001, 100), (7, 333, 128)])
def test_beam_stream_state_bytes(S, T, W):
    lib = ds.get_lib()
    assert lib.ds2_beam_decode_stream_state_bytes(S, T, W) == _pool_bytes(S, T, W, False)
    assert lib.ds2_beam_decode_lm_stream_state_bytes(S, T, W) == _pool_bytes(S, T, W, True)
    assert lib.ds2_beam_decode_stream_state_bytes(0, T, W) == 0
