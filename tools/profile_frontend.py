#!/usr/bin/env python
"""Per-kernel device time of one block of the benchmarked train step: the conv front-end or the recurrent layers.

    python tools/profile_frontend.py [--block conv|rnn] [--workload librispeech] [--steps 3] [--warmup 3]
                                     [--precision fp16] [--json OUT.json]

Builds the model, batch, precision mode and side stream exactly as `bench.py` does, warms up, then runs a few steps
under `torch.profiler` (CUDA activities).  Every kernel / memset launched from inside the block's library calls
(`ds2_conv_frontend_fwd` / `_bwd`, or `ds2_rnn_layer_fwd` / `_bwd` for all layers) is attributed to that call
through the launch's correlation id, and its device time and launch count are summed per step and per stream (the
main stream and the side stream the weight gradients run on are shown separately).  The card name and power limit are read in the same run.  Times under the profiler include its own
overhead per launch; step times come from `bench.py`, not from here.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, synth_batch  # noqa: E402

BLOCKS = {"conv": {"ds2_conv_frontend_fwd": "conv_fwd", "ds2_conv_frontend_bwd": "conv_bwd"},
          "rnn": {"ds2_rnn_layer_fwd": "rnn_fwd", "ds2_rnn_layer_bwd": "rnn_bwd"}}


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": clk}
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", default="conv", choices=sorted(BLOCKS))
    ap.add_argument("--workload", default="librispeech", choices=sorted(WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp16", choices=["tf32", "fp32", "fp16"])
    ap.add_argument("--json", default="", help="also write the table as JSON to this file")
    ap.add_argument("--trace", default="", help="also keep the profiler's chrome trace at this path")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    import deepspeech_pytorch_b200 as ds
    from deepspeech_pytorch_b200.optim import FlatParams, FusedOptimizer

    assert torch.cuda.is_available(), "profile_frontend.py needs a GPU"
    tags = BLOCKS[args.block]
    fwd_tag = next(iter(tags.values()))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = ds.get_lib()
    ds.set_precision(args.precision)
    rnn, bidir, H, layers, ctx, B, T, L = WORKLOADS[args.workload]
    rt = getattr(ds.RNNType, rnn)
    mcfg = (ds.BiDirectionalConfig(rnn_type=rt, hidden_size=H, hidden_layers=layers) if bidir else
            ds.UniDirectionalConfig(rnn_type=rt, hidden_size=H, hidden_layers=layers, lookahead_context=ctx))
    torch.manual_seed(123456)
    model = ds.DeepSpeech(ds.LABELS, mcfg, 32, ds.AdamConfig(), ds.SpectConfig()).to(dev).train()
    flat = FlatParams(model, direct_grads=True)
    main_stream = torch.cuda.Stream(device=dev, priority=-1)
    main_stream.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.set_stream(main_stream)
    ds.ops.enable_deferred_weight_grads(dev)
    opt = FusedOptimizer(flat, model.optim_cfg, max_norm=400.0)
    x, targets, pct, tsz = synth_batch(B, T, L, seed=1234)
    x_dev = x.to(dev)
    targets_pinned = targets.pin_memory()

    # mark the block's library calls with profiler ranges (the ctypes attributes are looked up at call time)
    for sym, tag in tags.items():
        fn = getattr(lib, sym)

        def wrapped(*a, _fn=fn, _tag=tag):
            with record_function(_tag):
                return _fn(*a)
        setattr(lib, sym, wrapped)

    def train_step():
        loss = model.training_step((x_dev, targets_pinned, pct.clone(), tsz), 0)
        loss.backward()
        opt.step(grad_scale=1.0)
        flat.zero_grad()
        return loss

    for _ in range(args.warmup):
        train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            train_step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
        if args.trace:
            os.makedirs(os.path.dirname(os.path.abspath(args.trace)), exist_ok=True)
            json.dump(trace, open(args.trace, "w"))
    card = card_info()

    ev = trace["traceEvents"] if isinstance(trace, dict) else trace
    ranges = [(e["ts"], e["ts"] + e["dur"], e["tid"], e["name"]) for e in ev
              if e.get("ph") == "X" and e.get("cat") == "user_annotation" and e.get("name") in tags.values()]
    corr_tag = {}
    for e in ev:
        if e.get("ph") != "X" or e.get("cat") not in ("cuda_runtime", "cuda_driver"):
            continue
        c = e.get("args", {}).get("correlation")
        for t0, t1, tid, tag in ranges:
            if e["tid"] == tid and t0 <= e["ts"] <= t1:
                corr_tag[c] = tag
                break
    table = defaultdict(lambda: [0.0, 0])     # (tag, stream, name) -> [us, count]
    for e in ev:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        tag = corr_tag.get(e.get("args", {}).get("correlation"))
        if tag is None:
            continue
        name = e["name"] if e["cat"] == "kernel" else e["cat"]
        key = (tag, e.get("args", {}).get("stream"), name.split("(")[0])
        table[key][0] += e["dur"]
        table[key][1] += 1
    fwd_streams = defaultdict(float)
    for (tag, stream, _), (us, _) in table.items():
        if tag == fwd_tag:
            fwd_streams[stream] += us
    main_id = max(fwd_streams, key=fwd_streams.get) if fwd_streams else None

    rows = []
    for (tag, stream, name), (us, cnt) in sorted(table.items(), key=lambda kv: (kv[0][0] != fwd_tag,
                                                                                 kv[0][1] != main_id, -kv[1][0])):
        rows.append({"block": tag, "stream": "main" if stream == main_id else f"side({stream})", "kernel": name,
                     "ms_per_step": us / 1e3 / args.steps, "launches_per_step": cnt / args.steps})
    print(f"card: {card}")
    print(f"block {args.block}, workload {args.workload}, precision {args.precision}, {args.steps} profiled steps (device time per step, "
          f"under the profiler)")
    print(f"{'block':9s} {'stream':10s} {'ms/step':>8s} {'launches':>8s}  kernel")
    totals = defaultdict(float)
    for r in rows:
        totals[(r["block"], r["stream"])] += r["ms_per_step"]
        print(f"{r['block']:9s} {r['stream']:10s} {r['ms_per_step']:8.3f} {r['launches_per_step']:8.1f}  {r['kernel']}")
    for (blk, stream), ms in sorted(totals.items()):
        print(f"total {blk} on {stream}: {ms:.3f} ms/step")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump({"card": card, "block": args.block, "workload": args.workload, "precision": args.precision, "steps": args.steps,
                   "rows": rows}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
