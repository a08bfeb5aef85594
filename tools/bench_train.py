"""`train` on the BASELINE model (5 x bi-LSTM-1024, precision 16, gradient clip 400) over a seeded synthetic WAV set,
against back-to-back steps of the same model on the same batches already on the device.

Writes 20+ training batches of 32 utterances of ~10 s and a 64-utterance validation set as 16-bit WAV files with JSON
manifests into --out, runs `train` for --epochs epochs (the first one warms up: module loads, workspaces), then
decodes the same training batches once, keeps them on the device and times --steps steps of the same step loop on
them with CUDA events.  The epoch rate can reach the back-to-back rate only if reading the WAV files, the spectrogram
batches and the host side of the loop hide behind the GPU.  Prints one JSON line, with the card's name and power
limit read in the same run.

    python tools/bench_train.py --out /tmp/bench_train"""
import argparse
import itertools
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR = 16000
WORDS = ["THE", "SPEECH", "MODEL", "TRAINS", "ON", "AUDIO", "WITH", "CHARACTER", "TARGETS", "AND", "CTC", "LOSS"]


def write_set(root, name, n, rng, seconds=(9.5, 10.5)):
    from scipy.io import wavfile
    samples = []
    for k in range(n):
        m = int(rng.uniform(*seconds) * SR)
        t = np.arange(m) / SR
        y = 0.2 * np.sin(2 * np.pi * rng.uniform(100, 400) * t) + 0.05 * rng.standard_normal(m)
        wavfile.write(os.path.join(root, f"{name}{k}.wav"), SR,
                      np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16))
        with open(os.path.join(root, f"{name}{k}.txt"), "w") as f:
            f.write(' '.join(rng.choice(WORDS, int(rng.integers(15, 30))).tolist()))
        samples.append({"wav_path": f"{name}{k}.wav", "transcript_path": f"{name}{k}.txt"})
    path = os.path.join(root, f"{name}.json")
    with open(path, "w") as f:
        json.dump({"root_path": root, "samples": samples}, f)
    return path


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the WAV set and checkpoints (default: a temp dir)")
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()

    import torch
    import deepspeech_pytorch_b200 as ds
    from deepspeech_pytorch_b200.evaluation import AudioDataLoader, SpectrogramDataset
    from deepspeech_pytorch_b200.optim import FlatParams, FusedOptimizer
    assert torch.cuda.is_available(), "bench_train needs a GPU"

    out = args.out or tempfile.mkdtemp(prefix="bench_train_")
    os.makedirs(out, exist_ok=True)
    rng = np.random.default_rng(2024)
    t0 = time.perf_counter()
    train_path = write_set(out, "tr", args.batches * args.batch_size, rng)
    val_path = write_set(out, "va", 64, rng)
    labels = os.path.join(out, "labels.json")
    with open(labels, "w") as f:
        json.dump(list(ds.LABELS), f)
    print(f"wrote the WAV set in {time.perf_counter() - t0:.1f} s", file=sys.stderr)

    workers = min(args.workers, os.cpu_count() or 1)
    cfg = ds.DeepSpeechConfig(seed=123456)
    cfg.data = ds.DataConfig(train_path=train_path, val_path=val_path, batch_size=args.batch_size,
                             num_workers=workers, labels_path=labels)
    cfg.trainer.max_epochs, cfg.trainer.precision, cfg.trainer.gradient_clip_val = args.epochs, 16, 400
    cfg.checkpoint.dirpath = os.path.join(out, "checkpoints")
    recs = ds.train(cfg)

    # the input pipeline alone: WAV reading in the workers + spectrogram batches on the GPU, no model
    loader = AudioDataLoader(SpectrogramDataset(cfg.data.spect, train_path, list(ds.LABELS), normalize=True),
                             batch_size=args.batch_size, num_workers=workers)
    loader_s = []
    for _ in range(2):
        t0 = time.perf_counter()
        batches = [(x, t, p.clone(), s) for x, t, p, s in loader]
        torch.cuda.synchronize()
        loader_s.append(time.perf_counter() - t0)

    # the same batches, kept on the device, through the same step on the same streams
    dev = torch.device("cuda")
    ds.seed_everything(cfg.seed)
    model = ds.DeepSpeech(list(ds.LABELS), cfg.model, 16, cfg.optim, cfg.data.spect).to(dev).train()
    flat = FlatParams(model, direct_grads=True)
    opt = FusedOptimizer(flat, cfg.optim, max_norm=400.0)
    main_stream = torch.cuda.Stream(device=dev, priority=-1)
    main_stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(main_stream):
        ds.ops.enable_deferred_weight_grads(dev)

        def step(b):
            x, t, p, s = b
            loss = model.training_step((x, t, p.clone(), s), 0)
            loss.backward()
            opt.step()
        for b in batches[:3]:
            step(b)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for b in itertools.islice(itertools.cycle(batches), args.steps):
            step(b)
        e1.record()
        torch.cuda.synchronize()
        ds.ops.enable_deferred_weight_grads(enable=False)
    step_ms = e0.elapsed_time(e1) / args.steps

    steady = recs[1:] or recs
    epoch_s = float(np.mean([r["train_s"] for r in steady]))
    n_steps = recs[0]["global_step"]
    n_utt = n_steps * args.batch_size
    res = {"gpu": gpu_info(), "model": "5x bi-LSTM-1024, precision 16, clip 400", "batch": args.batch_size,
           "train_batches": n_steps, "utterance_s": "9.5-10.5", "loader_workers": workers,
           "epoch_s": [round(r["train_s"], 3) for r in recs], "val_s": [round(r["val_s"], 3) for r in recs],
           "val_utterances": 64,
           "steady_epoch_s": round(epoch_s, 3), "utt_per_s": round(n_utt / epoch_s, 1),
           "epoch_ms_per_step": round(1e3 * epoch_s / n_steps, 2), "back_to_back_ms_per_step": round(step_ms, 2),
           "back_to_back_utt_per_s": round(1e3 * args.batch_size / step_ms, 1),
           "loader_only_s": [round(x, 3) for x in loader_s],
           "epoch_over_back_to_back": round(1e3 * epoch_s / n_steps / step_ms, 4),
           "losses": [round(r["loss"], 3) for r in recs]}
    print(json.dumps(res))
    with open(os.path.join(out, "bench_train.json"), "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main()
