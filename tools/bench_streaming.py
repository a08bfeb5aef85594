"""Streaming transcription throughput: `StreamingTranscriber.step` for 1, 8, 32 and 128 live sessions fed 160 ms or
320 ms of audio per step, against the same audio through `run_transcribe` with chunks of the same length, one
session at a time.

Model: uni-LSTM, 5 x 1024, lookahead context 20, precision 16, random weights (the time does not depend on them).
Reports per-step device time (CUDA events; each step ends in a synchronising copy of its labels), library launches
per step, the real-time factor across sessions (wall time / audio seconds of all sessions), and the algorithmic
latency the frame rules give.  Prints the card name and power limit of the run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import deepspeech_pytorch_b200 as ds  # noqa: E402
from deepspeech_pytorch_b200.streaming import conv_outputs_ready, head_outputs_ready  # noqa: E402

SR = 16000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        q = f"unknown ({e})"
    return name, q


def latency_frames(ctx):
    """spectrogram frames between frame 2u (head output u's centre) and the frame that decides it"""
    e = next(e for e in range(1, 10000) if head_outputs_ready(conv_outputs_ready(e, False), ctx, False) > 0)
    return e - 1


def run_stream(model, n_sess, feed, seconds, warmup):
    lib = ds.get_lib()
    st = ds.StreamingTranscriber(model, ds.GreedyDecoder(ds.LABELS), max_sessions=n_sess, max_seconds=seconds + 1)
    rng = np.random.default_rng(0)
    audio = [(0.1 * rng.standard_normal(int(seconds * SR))).astype(np.float32) for _ in range(n_sess)]
    sids = [st.open() for _ in range(n_sess)]
    n_steps = int(seconds * SR) // feed
    times, launches = [], []
    t0 = time.perf_counter()
    for k in range(n_steps):
        fd = {s: a[k * feed:(k + 1) * feed] for s, a in zip(sids, audio)}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        lib.ds2_launch_count(1)
        ev0.record()
        st.step(fd)
        ev1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            times.append(ev0.elapsed_time(ev1))
            launches.append(lib.ds2_launch_count(1))
    st.step({}, finish=sids)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return dict(sessions=n_sess, feed_ms=1000 * feed / SR, steps=n_steps, step_ms_mean=float(np.mean(times)),
                step_ms_p90=float(np.percentile(times, 90)), launches_per_step=float(np.mean(launches)),
                rtf=wall / (n_sess * n_steps * feed / SR))


def run_baseline(model, feed, seconds):
    from scipy.io import wavfile
    rng = np.random.default_rng(0)
    y = (0.1 * rng.standard_normal(int(seconds * SR))).astype(np.float32)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "a.wav")
        wavfile.write(p, SR, y)
        parser = ds.ChunkSpectrogramParser(ds.SpectConfig(), normalize=True)
        dec = ds.GreedyDecoder(ds.LABELS)
        ds.run_transcribe(p, parser, model, dec, "cuda", 16, feed / SR)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ds.run_transcribe(p, parser, model, dec, "cuda", 16, feed / SR)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    return dict(feed_ms=1000 * feed / SR, rtf_one_session=wall / seconds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,8,32,128")
    ap.add_argument("--feeds-ms", default="160,320")
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_streaming: needs a GPU")
    name, limit = card()
    print(f"# {name}, power.limit, clocks.max.sm: {limit}")
    torch.manual_seed(0)
    cfg = ds.UniDirectionalConfig(rnn_type=ds.RNNType.lstm, hidden_size=1024, hidden_layers=5, lookahead_context=20)
    model = ds.DeepSpeech(ds.LABELS, cfg, 16, ds.AdamConfig(), ds.SpectConfig()).cuda().eval()
    lf = latency_frames(20)
    print(json.dumps(dict(latency_spect_frames=lf, latency_s=(lf * 160 + 160) / SR)))
    for fm in [int(x) for x in a.feeds_ms.split(",")]:
        feed = fm * SR // 1000
        print(json.dumps(dict(baseline="run_transcribe", **run_baseline(model, feed, a.seconds))), flush=True)
        for n in [int(x) for x in a.sessions.split(",")]:
            print(json.dumps(run_stream(model, n, feed, a.seconds, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
