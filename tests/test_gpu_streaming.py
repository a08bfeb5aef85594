"""-m gpu: the streaming transcriber (deepspeech.pytorch_b200/streaming.py).

* spectrogram: streamed raw frames bit-identical to `ds2_spectrogram_batch(normalize=0)` of the whole stream over
  several chunkings; fixed normalisation against (x - mean) / std; running normalisation against the float64
  oracle (oracle/stream_oracle.py);
* model: the decided head outputs of 1, 7 and 48 sessions that start and finish at different steps against
  `model(x, lengths, logits=True)` of each whole utterance, normalised with the fixed statistics, in the fp32 mode
  and in precision 16, small and full size;
* decoding: the streamed greedy transcript against `GreedyDecoder.decode` of the concatenated output, and the same
  audio in two chunkings; the resumed beam search, with and without a language model, against one-shot
  `decode_beams` bit for bit (all W beams at the end, the best beam after every call);
* refusals of sessions."""
import random

import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import streaming as S
from gpu_helpers import make_model, rel, rel_l2
from oracle.stream_oracle import running_normalize
from test_gpu_beam_decode_lm import model_file, peaked_lm_probs

pytestmark = pytest.mark.gpu
SR, HOP = 16000, 160


def _audio(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    y = 0.05 * rng.standard_normal(n) + 0.3 * np.sin(2 * np.pi * (180 + 40 * seed) * t) * np.sin(2 * np.pi * 3 * t)
    return y.astype(np.float32)


def _raw_offline(y):
    return ds.ChunkSpectrogramParser(ds.SpectConfig(), normalize=False).spectrograms(y)[0]


def _feeds(n, kind, rng):
    if kind == "ones":
        return [1] * n
    if kind == "whole":
        return [n]
    if kind == "short":
        hi = HOP
    elif kind == "160ms":
        return [2560] * (n // 2560) + ([n % 2560] if n % 2560 else [])
    else:
        hi = 6000
    out, left = [], n
    while left > 0:
        c = min(left, rng.randrange(0, hi))
        out.append(c)
        left -= c
    return out


def _drive(step, audios, feeds, starts):
    """feed session i its chunks from step starts[i]; even sessions finish with their last feed, odd ones in a
    separate call with nothing new.  step(feeds {i: pcm}, finish [i]) -> {i: result}; returns the results per
    session in order"""
    pos = [0] * len(audios)
    off = [0] * len(audios)
    done = [False] * len(audios)
    res = [[] for _ in audios]
    t = 0
    while not all(done):
        fd, fin = {}, []
        for i in range(len(audios)):
            if done[i] or t < starts[i]:
                continue
            if pos[i] < len(feeds[i]):
                n = feeds[i][pos[i]]
                fd[i] = audios[i][off[i]:off[i] + n]
                off[i] += n
                pos[i] += 1
                if i % 2 == 0 and pos[i] == len(feeds[i]):
                    fin.append(i)
            else:
                fin.append(i)
        for i, r in step(fd, fin).items():
            res[i].append(r)
            if i in fin:
                done[i] = True
        t += 1
    return res


def _spect_stream(norm, audios, feeds, starts, stats=None):
    sp = S.StreamSpectrogram(ds.SpectConfig(), max_sessions=len(audios) + 2)
    slot = {i: len(audios) + 1 - i for i in range(len(audios))}       # slots out of order
    for i in range(len(audios)):
        m, s = stats[i] if stats else (0.0, 1.0)
        sp.reset(slot[i], norm, m, s)
    got = [[] for _ in audios]

    def step(fd, fin):
        ids = list(fd) + [i for i in fin if i not in fd]
        out, counts = sp.step([(slot[i], fd.get(i, np.zeros(0, np.float32)), i in fin) for i in ids])
        for j, i in enumerate(ids):
            if counts[j]:
                got[i].append(out[j, :, :counts[j]].clone())
        return {i: None for i in ids}

    _drive(step, audios, feeds, starts)
    return [torch.cat(g, 1) for g in got]


LENS = [1, 100, 159, 160, 4000, 16000, 23457]
KINDS = ["whole", "ones", "short", "whole", "short", "random", "160ms"]


def _spect_case(seed):
    rng = random.Random(seed)
    audios = [_audio(n, seed + i) for i, n in enumerate(LENS)]
    feeds = [_feeds(n, k if n < 5000 or k != "ones" else "short", rng) for n, k in zip(LENS, KINDS)]
    return audios, feeds, [rng.randrange(0, 3) for _ in LENS]


@pytest.mark.parametrize("seed", [0, 1])
def test_spectrogram_raw_frames_bit_identical(seed):
    audios, feeds, starts = _spect_case(seed)
    got = _spect_stream(S.NORM_NONE, audios, feeds, starts)
    for y, g in zip(audios, got):
        ref = _raw_offline(y)
        assert g.shape == ref.shape
        assert torch.equal(g, ref), float((g - ref).abs().max())


def test_spectrogram_fixed_and_running_normalisation():
    audios, feeds, starts = _spect_case(3)
    raw = [_raw_offline(y) for y in audios]
    # a 1-sample stream has one frame of 161 equal values: std 0, so it is normalised with std 1
    stats = [(float(r.double().mean()), float(r.double().std()) or 1.0) for r in raw]
    fixed = _spect_stream(S.NORM_FIXED, audios, feeds, starts, stats)
    for r, g, (m, s) in zip(raw, fixed, stats):
        ref = (r.double() - m) / s
        ulp = 2 ** -23 * (float(r.abs().max()) + abs(m)) / s
        assert float((g.double() - ref).abs().max()) <= 4 * ulp
    running = _spect_stream(S.NORM_RUNNING, audios, feeds, starts)
    for r, g in zip(raw, running):
        ref = torch.from_numpy(running_normalize(r.cpu().numpy()))
        # the one frame of a 1-sample stream holds 161 equal values: its std is 0 up to rounding, so it is left out
        ok = torch.isfinite(ref) & torch.isfinite(g.cpu())
        if r.shape[1] == 1:
            continue
        assert bool(ok.all())
        assert rel(g.cpu(), ref) < 1e-6
    # split independence: the same audio in another chunking gives the same bits
    rng = random.Random(9)
    other = _spect_stream(S.NORM_RUNNING, audios, [_feeds(len(y), "random", rng) for y in audios], [0] * len(LENS))
    for a, b in zip(running[1:], other[1:]):
        assert torch.equal(a, b)


def _model(rnn, H, layers, ctx, precision):
    m = make_model(rnn, False, H, layers, ctx=ctx).eval()
    m.precision = precision
    return m


def _offline_logits(model, y, m, s):
    raw = _raw_offline(y)
    x = (raw - torch.tensor(np.float32(m), device=raw.device)) * (1.0 / torch.tensor(np.float32(s), device=raw.device))
    with torch.no_grad():
        out, _, _ = model(x[None, None].contiguous(), torch.tensor([raw.shape[1]]), logits=True)
    return out[0]


def _stream_logits(model, audios, feeds, starts, stats, max_sessions=None):
    st = ds.StreamingTranscriber(model, ds.GreedyDecoder(ds.LABELS), max_sessions=max_sessions or len(audios),
                                 logits=True)
    sid = {}
    outs = [[] for _ in audios]

    def step(fd, fin):
        for i in list(fd) + list(fin):
            if i not in sid:
                sid[i] = st.open(*stats[i])
        res = st.step({sid[i]: p for i, p in fd.items()}, [sid[i] for i in fin], return_outputs=True)
        back = {v: k for k, v in sid.items()}
        out = {}
        for s_, r in res.items():
            i = back[s_]
            if r.outputs is not None and r.outputs.shape[0]:
                outs[i].append(r.outputs.clone())
            out[i] = r
        return out

    res = _drive(step, audios, feeds, starts)
    return [torch.cat(o) for o in outs], res


def _check_model(model, n_sessions, seed, tol, bit_equal=False):
    rng = random.Random(seed)
    lens = [rng.randrange(2000, 40000) for _ in range(n_sessions)]
    lens[0] = 1200                                           # shorter than the receptive field: 8 frames
    audios = [_audio(n, seed + i) for i, n in enumerate(lens)]
    kinds = ["160ms", "random", "short", "whole"]
    feeds = [_feeds(n, kinds[i % 4], rng) for i, n in enumerate(lens)]
    starts = [rng.randrange(0, 4) for _ in lens]
    raw = [_raw_offline(y) for y in audios]
    stats = [(float(r.double().mean()), float(r.double().std())) for r in raw]
    got, res = _stream_logits(model, audios, feeds, starts, stats)
    worst, equal = 0.0, True
    for i, y in enumerate(audios):
        ref = _offline_logits(model, y, *stats[i])
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        assert res[i][-1].final and res[i][-1].frames_decided == ref.shape[0]
        tol(got[i], ref)
        if bit_equal:
            assert torch.equal(got[i], ref), (i, rel(got[i], ref))
        worst = max(worst, rel(got[i], ref))
        equal = equal and torch.equal(got[i], ref)
    print(f"sessions={n_sessions} worst rel err={worst:.2e} bit-equal={equal}")
    return equal


def _fp32(a, b):
    assert rel(a, b) < 1e-5, rel(a, b)


def _fp16(a, b):
    assert rel(a, b) < 2e-2 and rel_l2(a, b) < 1e-2, (rel(a, b), rel_l2(a, b))


@pytest.mark.parametrize("rnn", ["lstm", "gru"])
@pytest.mark.parametrize("n_sessions", [1, 7, 48])
def test_model_outputs_equal_offline_fp32(rnn, n_sessions):
    saved = ds.get_precision()
    ds.set_precision("fp32")
    try:
        # the fp32 mode runs every output through the same products in the same order as the offline forward
        _check_model(_model(rnn, 64, 2, 5 if rnn == "gru" else 20, 32), n_sessions, 11 + n_sessions, _fp32,
                     bit_equal=True)
    finally:
        ds.set_precision(saved)


@pytest.mark.parametrize("rnn", ["lstm", "gru"])
@pytest.mark.parametrize("n_sessions", [1, 7, 48])
def test_model_outputs_full_size_precision_16(rnn, n_sessions):
    lib = ds.get_lib()
    model = _model(rnn, 1024, 5, 20, 16)
    lib.ds2_fallback_count(1)
    _check_model(model, n_sessions, 5 + n_sessions, _fp16)
    print(f"{rnn} sessions={n_sessions} fallbacks={lib.ds2_fallback_count(1)}")


def test_full_size_single_session_takes_no_fallback():
    lib = ds.get_lib()
    model = _model("lstm", 1024, 5, 20, 16)
    y = _audio(32000, 3)
    st = ds.StreamingTranscriber(model, ds.GreedyDecoder(ds.LABELS), max_sessions=1)
    sid = st.open()
    st.step({sid: y[:2560]})
    lib.ds2_fallback_count(1)
    for k in range(2560, len(y), 2560):
        st.step({sid: y[k:k + 2560]})
    st.step({}, finish=[sid])
    assert lib.ds2_fallback_count(1) == 0


def test_greedy_stream_equals_one_shot_decode():
    model = _model("gru", 64, 2, 20, 32)
    rng = random.Random(4)
    lens = [48000, 3000, 20000]
    audios = [_audio(n, 20 + i) for i, n in enumerate(lens)]
    feeds = [_feeds(n, k, rng) for n, k in zip(lens, ["160ms", "short", "random"])]
    dec = ds.GreedyDecoder(ds.LABELS)
    st = ds.StreamingTranscriber(model, dec, max_sessions=3)
    sid = {}
    outs = [[] for _ in lens]

    def step(fd, fin):
        for i in list(fd) + list(fin):
            if i not in sid:
                sid[i] = st.open()
        res = st.step({sid[i]: p for i, p in fd.items()}, [sid[i] for i in fin], return_outputs=True)
        back = {v: k for k, v in sid.items()}
        for s_, r in res.items():
            if r.outputs is not None:
                outs[back[s_]].append(r.outputs.clone())
        return {back[s_]: r for s_, r in res.items()}

    res = _drive(step, audios, feeds, [0, 1, 2])
    for i in range(len(lens)):
        probs = torch.cat(outs[i])[None]
        strings, offsets = dec.decode(probs)
        final = res[i][-1]
        assert final.final and final.text == strings[0][0]
        assert final.offsets == offsets[0][0].tolist()
        # partial results only ever grow
        for a, b in zip(res[i], res[i][1:]):
            assert b.text.startswith(a.text) and b.frames_decided >= a.frames_decided


def test_two_chunkings_give_the_same_transcript():
    model = _model("lstm", 64, 2, 20, 32)
    y = _audio(40000, 8)
    texts = []
    for feeds in ([2560] * 15 + [1600], _feeds(len(y), "random", random.Random(1))):
        st = ds.StreamingTranscriber(model, ds.GreedyDecoder(ds.LABELS), max_sessions=1)
        sid = st.open()
        off = 0
        for n in feeds:
            st.step({sid: y[off:off + n]})
            off += n
        r = st.step({}, finish=[sid])[sid]
        texts.append((r.text, r.offsets, r.frames_decided))
    assert texts[0] == texts[1]


def test_session_refusals():
    model = _model("gru", 32, 1, 5, 32)
    st = ds.StreamingTranscriber(model, ds.GreedyDecoder(ds.LABELS), max_sessions=2, max_seconds=1.0)
    a, b = st.open(), st.open()
    with pytest.raises(ds.Ds2Error, match="sessions are open"):
        st.open()
    with pytest.raises(ds.Ds2Error, match="unknown"):
        st.step({12345: np.zeros(10, np.float32)})
    with pytest.raises(ds.Ds2Error, match="max_seconds"):
        st.step({a: np.zeros(100, np.float32), b: np.zeros(SR + 1, np.float32)})
    assert st.spect.n[st._slot[a]] == 0                     # nothing was fed: the check runs before any launch
    st.step({a: np.zeros(SR, np.float32)}, finish=[a])
    with pytest.raises(ds.Ds2Error, match="finished"):
        st.step({a: np.zeros(10, np.float32)})
    c = st.open()                                            # the finished session's slot is free again
    assert c not in (a, b)
    with pytest.raises(ds.Ds2Error, match="1-D"):
        st.step({c: np.zeros((2, 10), np.float32)})


def _split(T, rng, kind):
    if kind == "ones":
        return [1] * T
    out, left = [], T
    while left > 0:
        c = min(left, rng.randrange(0, 13))
        out.append(c)
        left -= c
    return out


def _flat_probs(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(B, T, 29, generator=g) * 1.5, -1)


def _best_of(dec, probs_bt):
    labels, scores, timesteps, lengths, n_beams = dec.decode_beams(probs_bt[None].cuda())
    n = int(lengths[0, 0])
    return labels[0, 0, :n].numpy(), timesteps[0, 0, :n].numpy(), n, float(scores[0, 0]), int(n_beams[0])


@pytest.mark.parametrize("W", [1, 8, 100])
@pytest.mark.parametrize("prune", [False, True])
@pytest.mark.parametrize("lm_order", [0, 3])
def test_resumed_beam_search_equals_one_shot(tmp_path_factory, W, prune, lm_order):
    B, T = 3, 48
    seed = W + 2 * prune + lm_order
    probs = peaked_lm_probs(B, T, seed) if lm_order else _flat_probs(B, T, seed)
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=model_file(tmp_path_factory, lm_order, seed) if lm_order else None,
                            alpha=0.8, beta=1.5, beam_width=W, cutoff_top_n=5 if prune else 40,
                            cutoff_prob=0.95 if prune else 1.0)
    ref = dec.decode_beams(probs.cuda())
    bs = S.StreamBeamSearch(dec, max_sessions=4, max_frames=T)
    slots = [3, 0, 2]
    for s_ in slots:
        bs.reset(s_)
    rng = random.Random(seed)
    splits = [_split(T, rng, "ones"), _split(T, rng, "random"), _split(T, rng, "random")]
    pos, done = [0] * B, [0] * B
    while any(pos[b] < len(splits[b]) for b in range(B)):
        items, rows = [], []
        for b in range(B):
            if pos[b] < len(splits[b]):
                k = splits[b][pos[b]]
                items.append((b, k, pos[b] == len(splits[b]) - 1))
                rows.append(probs[b, done[b]:done[b] + k])
                pos[b] += 1
        packed = torch.cat(rows).cuda() if sum(r.shape[0] for r in rows) else None
        got = bs.step(packed, [(slots[b], k, f) for b, k, f in items])
        for (b, k, fin), (lab, ts, ln, sc, nb) in zip(items, got):
            done[b] += k
            if fin:
                assert done[b] == T
                labels, scores, timesteps, lengths, n_beams = ref
                assert nb == int(n_beams[b])
                assert np.array_equal(lab, labels[b].numpy()) and np.array_equal(ts, timesteps[b].numpy())
                assert np.array_equal(ln, lengths[b].numpy()) and np.array_equal(sc, scores[b].numpy())
            elif done[b] > 0 and (b == 1 or done[b] % 7 == 0):
                bl, bt, bn, bsc, bnb = _best_of(dec, probs[b, :done[b]])
                assert nb == bnb and int(ln[0]) == bn and float(sc[0]) == bsc
                assert np.array_equal(lab[0, :bn], bl) and np.array_equal(ts[0, :bn], bt)


@pytest.mark.parametrize("lm_order", [0, 2])
def test_transcriber_with_beam_decoder(tmp_path_factory, lm_order):
    model = _model("gru", 64, 2, 20, 32)
    dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=model_file(tmp_path_factory, lm_order, 4) if lm_order else None,
                            alpha=0.5, beta=1.0, beam_width=16)
    rng = random.Random(2)
    lens = [30000, 5000]
    audios = [_audio(n, 30 + i) for i, n in enumerate(lens)]
    feeds = [_feeds(n, k, rng) for n, k in zip(lens, ["160ms", "random"])]
    st = ds.StreamingTranscriber(model, dec, max_sessions=2, max_seconds=3.0)
    sid, outs = {}, [[] for _ in lens]

    def step(fd, fin):
        for i in list(fd) + list(fin):
            if i not in sid:
                sid[i] = st.open()
        res = st.step({sid[i]: p for i, p in fd.items()}, [sid[i] for i in fin], return_outputs=True)
        back = {v: k for k, v in sid.items()}
        for s_, r in res.items():
            if r.outputs is not None:
                outs[back[s_]].append(r.outputs.clone())
        return {back[s_]: r for s_, r in res.items()}

    res = _drive(step, audios, feeds, [0, 1])
    for i in range(len(lens)):
        probs = torch.cat(outs[i])[None]
        labels, scores, timesteps, lengths, n_beams = dec.decode_beams(probs)
        final = res[i][-1]
        assert final.final and len(final.beams) == int(n_beams[0])
        for r, (text, offs, score) in enumerate(final.beams):
            n = int(lengths[0, r])
            assert text == "".join(ds.LABELS[int(c)] for c in labels[0, r, :n])
            assert offs == timesteps[0, r, :n].tolist() and score == float(scores[0, r])
        assert final.text == final.beams[0][0] and final.offsets == final.beams[0][1]
