"""Chunked transcription (`run_transcribe`) of the headline model on one GPU.

The headline model (5 x bi-LSTM-1024, seeded weights, eval mode) in precision 16 transcribes a seeded 60 s waveform
(int16 WAV in a temporary directory) in chunks of 10 s: T' = 500 output frames per chunk, each chunk's forward given
the previous chunk's final states `hs`.  Reported:
  * device time of one chunk's forward without a state (the first chunk) and with one (the later chunks), CUDA events
    around warmed-up calls, median of --iters;
  * the same stateful forward on the per-step FFMA kernels, the path every stateful forward took before the wgmma
    sweeps accepted an initial state (forced here with DS2_NO_RESIDENT=1, under which the sweeps decline a state);
  * whole-file `run_transcribe` wall time (host clock, the decode ends in a device-to-host copy) with the greedy
    decoder and with the beam decoder at W = 10, median of --reps;
  * `ds2_fallback_count()` over the wgmma runs (0 expected).
The card name, power limit and maximum SM clock are read in the same run.  Needs a GPU; prints one JSON line.

    python tools/bench_transcribe.py [--seconds 60] [--chunk 10] [--iters 10] [--reps 3]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch
from scipy.io import wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import deepspeech_pytorch_b200 as ds  # noqa: E402
from bench_beam_decode import card_info  # noqa: E402  (tools/ is on sys.path when run as a script)


def event_ms(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--chunk", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_transcribe: needs a GPU")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = ds.DeepSpeech(ds.LABELS, ds.BiDirectionalConfig(), 16, ds.AdamConfig(), ds.SpectConfig()).to(dev).eval()
    sr = model.spect_cfg.sample_rate
    rng = np.random.default_rng(0)
    n = int(args.seconds * sr)
    t = np.arange(n) / sr
    y = 0.3 * np.sin(2 * np.pi * 220 * t) * np.sin(2 * np.pi * 0.7 * t) + 0.05 * rng.standard_normal(n)
    lib = ds.get_lib()
    res = {"card": card_info(), "model": "5x bi-LSTM-1024, precision 16, eval", "seconds": args.seconds,
           "chunk_seconds": args.chunk}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "audio.wav")
        wavfile.write(path, sr, np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16))
        parser = ds.ChunkSpectrogramParser(model.spect_cfg, normalize=True)
        spects = [s.contiguous().view(1, 1, *s.shape) for s in parser.parse_audio(path, args.chunk)]
        sizes = torch.tensor([spects[0].shape[3]], dtype=torch.int32)
        res["chunks"] = len(spects)
        with torch.no_grad():
            _, osz, hs = model(spects[0], sizes)
        res["frames_per_chunk"] = int(osz[0])

        def fwd(state):
            with torch.no_grad():
                model(spects[1], sizes, hs if state else None)
        lib.ds2_fallback_count(1)
        for state in (False, True):
            fwd(state)
        res["fwd_no_state_ms"] = round(event_ms(lambda: fwd(False), args.iters), 3)
        res["fwd_with_state_ms"] = round(event_ms(lambda: fwd(True), args.iters), 3)

        greedy = ds.GreedyDecoder(model.labels)
        beam = ds.BeamCTCDecoder(model.labels, beam_width=10, blank_index=model.labels.index("_"))
        for name, dec in (("greedy", greedy), ("beam_w10", beam)):
            ds.run_transcribe(path, parser, model, dec, dev, 16, args.chunk)          # warm-up
            walls = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                out, _ = ds.run_transcribe(path, parser, model, dec, dev, 16, args.chunk)
                walls.append((time.perf_counter() - t0) * 1e3)
            res[f"run_transcribe_{name}_ms"] = round(statistics.median(walls), 1)
            res[f"transcript_{name}_chars"] = len(out[0][0])
        res["fallback_count"] = int(lib.ds2_fallback_count(1))

        os.environ["DS2_NO_RESIDENT"] = "1"
        try:
            fwd(True)
            res["fwd_with_state_ffma_ms"] = round(event_ms(lambda: fwd(True), max(3, args.iters // 3)), 3)
        finally:
            del os.environ["DS2_NO_RESIDENT"]
        lib.ds2_fallback_count(1)
    res["ffma_over_wgmma"] = round(res["fwd_with_state_ffma_ms"] / res["fwd_with_state_ms"], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
