"""-m gpu: `ds2_ctc_align` bit for bit against the float64 oracle (oracle/align_oracle.py), the logits mode, the
argument errors, and the alignment front ends on golden models, generated WAV files and a manifest."""
import json

import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from conftest import Golden, golden_names
from gpu_helpers import make_model, model_from_golden
from oracle import align_oracle as A

pytestmark = pytest.mark.gpu
MAX_L = 6144   # DS2_CTC_ALIGN_MAX_TGT_LEN
SR = 16000


def _log_probs(T, B, C, seed, peak=3.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, B, C, generator=g) * peak
    return torch.log_softmax(x, dim=2)


def _targets(lens, C, seed, repeats=True):
    rng = np.random.default_rng(seed)
    out = []
    for L in lens:
        t = rng.integers(1, C, size=L)
        if repeats and L > 3:
            t[1] = t[0]                      # at least one adjacent repeat
        out.append([int(v) for v in t])
    return out


def _run(lp_tbc, tg, in_len, log_probs=True):
    """lp (T,B,C) CPU -> kernel outputs on the CPU"""
    em = lp_tbc.cuda().transpose(0, 1)      # the model's layout: a transpose view of (T,B,C)
    flat = torch.tensor([c for t in tg for c in t], dtype=torch.int64)
    labels, flp, spans, scores = ds.forced_align(em, torch.tensor(in_len), flat, torch.tensor([len(t) for t in tg]),
                                                 blank=0, log_probs=log_probs)
    torch.cuda.synchronize()
    return labels.cpu(), flp.cpu(), spans.cpu(), scores.cpu()


def _check_against_oracle(lp_tbc, tg, in_len, labels, flp, spans, scores):
    T, B, C = lp_tbc.shape
    max_l = max(len(t) for t in tg)
    for b in range(B):
        ref = A.ctc_align(lp_tbc[:in_len[b], b].numpy(), tg[b])
        assert float(scores[b]) == ref["score"] or (np.isinf(ref["score"]) and float(scores[b]) == ref["score"]), b
        exp_labels = np.full(T, -1)
        exp_labels[:in_len[b]] = ref["labels"]
        assert np.array_equal(labels[b].numpy(), exp_labels), b
        exp_spans = np.full((max_l, 2), -1)
        exp_spans[:len(tg[b])] = ref["spans"]
        assert np.array_equal(spans[b].numpy().reshape(max_l, 2), exp_spans), b
        exp_lp = np.zeros(T)
        exp_lp[:in_len[b]] = ref["frame_log_probs"]
        assert np.abs(flp[b].double().numpy() - exp_lp).max() <= 1e-6, b


@pytest.mark.parametrize("B,T,L", [(1, 1, 0), (1, 1, 1), (7, 500, 250), (64, 500, 1), (7, 5000, 2000),
                                   (64, 500, 0), (1, 5000, 250)])
def test_bit_exact_against_the_oracle(B, T, L):
    lp = _log_probs(T, B, 29, seed=T + B + L)
    lens = [max(0, L - (b % 3)) for b in range(B)]
    tg = _targets(lens, 29, seed=L)
    in_len = [max(1, T - 7 * b) for b in range(B)]
    for b in range(B):
        if b % 2 == 1:      # each odd row at its feasibility minimum
            reps = sum(1 for i in range(1, len(tg[b])) if tg[b][i] == tg[b][i - 1])
            in_len[b] = min(T, max(1, len(tg[b]) + reps))
    lp_nan = lp.clone()
    for b in range(B):
        lp_nan[in_len[b]:, b] = float("nan")          # padding frames are never read
    out = _run(lp_nan, tg, in_len)
    _check_against_oracle(lp, tg, in_len, *out)


def test_minus_inf_entries_and_infeasible_rows():
    T, B, C = 300, 8, 29
    lp = _log_probs(T, B, C, seed=11)
    tg = _targets([40] * B, C, seed=3)
    in_len = [T] * B
    in_len[1] = 20                                      # too few frames
    lp[:, 2, tg[2][5]] = float("-inf")                  # every path of row 2 runs through -inf
    lp[100:140, 3, 0] = float("-inf")                   # row 3: blanks forbidden for a while, still feasible
    lp[:, 4, 7] = float("-inf")
    tg[5] = []                                          # empty target: all-blank path
    in_len[6] = 0                                       # no frames, non-empty target
    out = _run(lp, tg, in_len)
    _check_against_oracle(lp, tg, in_len, *out)
    labels, flp, spans, scores = out
    assert float(scores[1]) == float("-inf") and float(scores[2]) == float("-inf")
    assert float(scores[6]) == float("-inf") and bool((labels[6] == -1).all())
    assert np.isfinite(float(scores[3])) and np.isfinite(float(scores[5]))
    assert bool((labels[1] == -1).all()) and bool((spans[1] == -1).all())


def test_empty_target_and_no_frames_scores_zero():
    lp = _log_probs(10, 2, 29, seed=1)
    labels, flp, spans, scores = _run(lp, [[], [3]], [0, 10])
    assert float(scores[0]) == 0.0 and bool((labels[0] == -1).all())
    assert A.ctc_align(lp[:10, 1].numpy(), [3])["score"] == float(scores[1])


def test_supported_maximum_length():
    T, B, C = 13000, 2, 29
    lp = _log_probs(T, B, C, seed=5, peak=1.0)
    tg = _targets([MAX_L, MAX_L - 1], C, seed=9)
    in_len = [T, T - 11]
    out = _run(lp, tg, in_len)
    _check_against_oracle(lp, tg, in_len, *out)


def test_over_the_limit_is_an_error_and_runs_repeat_bit_for_bit():
    lib = ds.get_lib()
    T, B, C = 50, 3, 29
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    x = torch.zeros(T, B, C, device="cuda")
    out = torch.empty(B, dtype=torch.float64, device="cuda")
    rc = lib.ds2_ctc_align(T, B, C, x.data_ptr(), 0, ws.data_ptr(), ws.data_ptr(), ws.data_ptr(), MAX_L + 1, 0,
                           None, None, ws.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), None)
    assert rc == -1 and b"DS2_CTC_ALIGN_MAX_TGT_LEN = 6144" in lib.ds2_last_error()
    assert lib.ds2_ctc_align_workspace_bytes(T, B, C, 10) > 0
    rc = lib.ds2_ctc_align(T, B, C, x.data_ptr(), 0, ws.data_ptr(), ws.data_ptr(), ws.data_ptr(), 10, 0, None, None,
                           ws.data_ptr(), out.data_ptr(), ws.data_ptr(), 16, None)
    assert rc == -1 and b"workspace" in lib.ds2_last_error()
    rc = lib.ds2_ctc_align(T, B, C, x.data_ptr(), 0, ws.data_ptr(), ws.data_ptr(), ws.data_ptr(), 10, C, None, None,
                           ws.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), None)
    assert rc == -1
    with pytest.raises(ds.Ds2Error):
        ds.forced_align(x.transpose(0, 1), [T] * B, torch.zeros(B, 2, dtype=torch.long), [2] * B)   # blank target
    lp = _log_probs(400, 16, 29, seed=2)
    tg = _targets([120] * 16, 29, seed=2)
    a = _run(lp, tg, [400] * 16)
    b = _run(lp, tg, [400] * 16)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_logits_mode():
    T, B, C = 400, 6, 29
    g = torch.Generator().manual_seed(7)
    x = torch.randn(T, B, C, generator=g) * 4
    tg = _targets([100, 80, 1, 0, 150, 60], C, seed=4)
    in_len = [T, T - 30, 50, 40, T - 5, 200]
    labels, flp, spans, scores = _run(x, tg, in_len, log_probs=False)
    lp = torch.log_softmax(x.cuda(), dim=2).cpu()
    compared = 0
    for b in range(B):
        ref = A.ctc_align(lp[:in_len[b], b].numpy(), tg[b])
        n = in_len[b]
        got_lp = flp[b, :n].double()
        idx = labels[b, :n].long()
        assert (got_lp - lp[torch.arange(n), b, idx].double()).abs().max() <= 1e-6
        last, second = ref["final"]
        if abs(last - second) > 1e-9:
            assert np.array_equal(labels[b, :n].numpy(), ref["labels"]), b
            compared += 1
    assert compared >= 4


# ---------------------------------------------------------------------------------------------- model level
@pytest.mark.parametrize("name", golden_names())
def test_golden_logits_softmax_equals_eval_output(name):
    g = Golden(name)
    model = model_from_golden(g).eval()
    ds.set_precision("fp32")
    x = g.x.cuda()
    with torch.no_grad():
        probs, osz, _ = model(x, g.input_sizes)
        logits, osz2, _ = model(x, g.input_sizes, logits=True)
    assert torch.equal(osz, osz2)
    assert (torch.softmax(logits, dim=2) - probs).abs().max() <= 1e-6
    # the greedy transcript of each utterance, aligned back, reproduces the argmax path where that path is unique
    lab, offs, counts = ds.GreedyDecoder(model.labels).decode_indices(probs, osz)
    greedy_tg = []
    for b in range(x.shape[0]):
        greedy_tg.append(lab[b, :int(counts[b])].tolist())
    flat = torch.tensor([c for t in greedy_tg for c in t], dtype=torch.int64)
    labels, flp, spans, scores = ds.forced_align(logits, osz, flat, [len(t) for t in greedy_tg])
    top2 = torch.log_softmax(logits, 2).topk(2, dim=2).values
    for b in range(x.shape[0]):
        n = int(osz[b])
        if float((top2[b, :n, 0] - top2[b, :n, 1]).min()) <= 1e-5:
            continue
        argmax = probs[b, :n].argmax(dim=1).cpu()
        assert torch.equal(labels[b, :n].cpu().long(), argmax), b


def _wav(path, seconds, seed):
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    t = np.arange(n) / SR
    y = 0.3 * np.sin(2 * np.pi * (300 + 200 * seed) * t) * np.sin(2 * np.pi * 1.3 * t) + 0.05 * rng.standard_normal(n)
    wavfile.write(str(path), SR, np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16))
    return n / SR


def _model():
    torch.manual_seed(0)
    return make_model("lstm", True, 64, 2).eval()


def test_align_audio(tmp_path):
    model = _model()
    ds.set_precision("fp32")
    dur = _wav(tmp_path / "a.wav", 2.3, seed=1)
    parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
    text = "HELLO THERE\n"
    rec = ds.align_audio(str(tmp_path / "a.wav"), text, parser, model, torch.device("cuda"), 32)
    assert rec["feasible"] and rec["transcript"] == "HELLO THERE" and np.isfinite(rec["score"])
    assert "".join(c["char"] for c in rec["chars"]) == "HELLO THERE"
    assert [w["word"] for w in rec["words"]] == ["HELLO", "THERE"]
    prev_end = 0.0
    for c in rec["chars"]:
        assert prev_end <= c["start"] <= c["end"] <= dur
        assert 0.0 < c["score"] <= 1.0
        prev_end = c["end"]
    assert (rec["frames"] - 1) * 0.02 <= dur + 1e-9      # the last output frame starts inside the file
    # too long a transcript for the audio
    bad = ds.align_audio(str(tmp_path / "a.wav"), "A" * 400, parser, model, torch.device("cuda"), 32)
    assert not bad["feasible"] and bad["score"] is None and bad["chars"] == []


def _manifest(tmp_path):
    texts = ["HI", "A LONGER ONE", "", "SOME WORDS HERE", "OK"]
    secs = [1.1, 3.0, 0.7, 2.2, 1.6]
    samples = []
    (tmp_path / "wav").mkdir()
    (tmp_path / "txt").mkdir()
    for i, (t, s) in enumerate(zip(texts, secs)):
        _wav(tmp_path / "wav" / f"{i}.wav", s, seed=i)
        (tmp_path / "txt" / f"{i}.txt").write_text(t + "\n")
        samples.append({"wav_path": f"wav/{i}.wav", "transcript_path": f"txt/{i}.txt"})
    path = tmp_path / "manifest.json"
    path.write_text(json.dumps({"root_path": str(tmp_path), "samples": samples}))
    return str(path), texts


def test_align_manifest(tmp_path):
    model = _model()
    ckpt = tmp_path / "m.ckpt"
    torch.save({"state_dict": model.state_dict(),
                "hyper_parameters": {"labels": model.labels, "model_cfg": model.model_cfg, "precision": 32,
                                     "optim_cfg": model.optim_cfg, "spect_cfg": model.spect_cfg}}, str(ckpt))
    manifest, texts = _manifest(tmp_path)
    ds.set_precision("fp32")
    parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
    singles = [ds.align_audio(str(tmp_path / "wav" / f"{i}.wav"), t, parser, model, torch.device("cuda"), 32)
               for i, t in enumerate(texts)]
    out1 = tmp_path / "out1.jsonl"
    cfg = ds.AlignConfig(model=ds.ModelConfig(model_path=str(ckpt)), manifest_path=manifest, output_path=str(out1),
                         batch_size=1, num_workers=0)
    recs1 = ds.align_manifest(cfg)
    lines = [json.loads(l) for l in out1.read_text().splitlines()]
    assert len(lines) == len(texts) == len(recs1)
    for i, (r, line, single) in enumerate(zip(recs1, lines, singles)):
        assert r["wav_path"].endswith(f"wav/{i}.wav") and r["transcript_path"].endswith(f"txt/{i}.txt")
        assert line == r
        r = {k: v for k, v in r.items() if k not in ("wav_path", "transcript_path")}
        assert r == single, i
    cfg.batch_size, cfg.output_path = 3, ""
    recs3 = ds.align_manifest(cfg)
    assert [r["transcript"] for r in recs3] == [r["transcript"] for r in recs1] == texts
    for a, b in zip(recs3, recs1):
        assert a["feasible"] == b["feasible"] and a["frames"] == b["frames"]
        assert abs(a["score"] - b["score"]) <= 1e-3 * abs(b["score"])
        for ca, cb in zip(a["chars"], b["chars"]):
            assert abs(ca["start"] - cb["start"]) <= 0.02 + 1e-9 and abs(ca["end"] - cb["end"]) <= 0.02 + 1e-9
