#!/usr/bin/env python
"""Where a step of the forward recurrent sweep goes: per-phase medians from the kernel's own clock stamps.

    python tools/sweep_trace.py [--rnn lstm|gru] [--bidir 1] [--H 1024] [--B 32] [--T 500] [--json OUT.json]

Runs one layer forward (training mode, precision 16, every utterance full length) with `DS2_TRACE_FWD` pointing at
a device buffer, so that the split-K forward sweep (`rnn_fwd_splitk_kernel`) writes 16 stamps per (CTA, time step),
and prints the medians over CTAs and steps 2 .. T-2 of the phases between them, in SM cycles.  Slots (set by
`trace_stamp` in csrc/rnn_persistent_tc.cu):
    0  producer passed the grid barrier          1  producer issued the h_{t-1} TMA loads
    2  first K group of h_{t-1} landed           3  last K group landed
    4  all MMAs of the step done (a kernel with an accumulator image: image written)
    5  epilogue warps woke on the accumulator image (only a kernel with one)
    6  partial rows pushed to the peer CTA       7  the peer's partial rows landed
    8  cell update done, h_t (fp16) stored       9  step barrier among the finishing warps passed
    10 fence.proxy.async done                   11 red.release on the step counter done
    12 %globaltimer (ns) at the release          13 deferred fp32 stores issued
Phases are differences of stamps of one CTA (one SM clock); the step period is the median difference of slot 0
between consecutive steps, and the arrival skew the median over steps of (latest - earliest) slot 12 over the CTAs
of a direction.  Needs a GPU; the card name and power limit are printed with the table."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = 16

# (name, end slot, start slot or tuple of fallbacks: the first start slot that was stamped is used)
PHASES = [
    ("barrier_to_tma_issued", 1, (0,)),
    ("barrier_to_first_h_group", 2, (0,)),
    ("first_to_last_h_group", 3, (2,)),
    ("mma_chain", 4, (2,)),
    ("accum_image_handoff", 5, (4,)),
    ("push_partials", 6, (5, 4)),
    ("wait_peer_partials", 7, (6,)),
    ("cell_update", 8, (7,)),
    ("step_barrier_fence_release", 11, (8,)),
    ("release_to_next_barrier_pass", None, None),   # slot 0 of step s+1 minus slot 11 of step s
    ("deferred_stores", 13, (11,)),
]


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": clk}
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def phase_table(tr, T, ctas_per_dir):
    """tr: int64 [CTAs, T, SLOTS] -> {phase: median cycles}, period (cycles, ns), arrival skew (ns)"""
    steps = np.arange(2, T - 1)
    s = tr[:, steps, :].astype(np.float64)
    res = {}
    for name, end, starts in PHASES:
        if end is None:
            v = tr[:, steps + 1, 0].astype(np.float64) - tr[:, steps, 11]
        else:
            start = next((a for a in starts if np.all(s[:, :, a] != 0)), None)
            if start is None or not np.all(s[:, :, end] != 0):
                continue
            v = s[:, :, end] - s[:, :, start]
        res[name] = float(np.median(v))
    period = tr[:, steps + 1, 0].astype(np.float64) - tr[:, steps, 0]
    period_ns = tr[:, steps + 1, 12].astype(np.float64) - tr[:, steps, 12]
    ns = tr[:, steps, 12].astype(np.float64)
    skew = [float(np.median(ns[d0:d0 + ctas_per_dir].max(0) - ns[d0:d0 + ctas_per_dir].min(0)))
            for d0 in range(0, tr.shape[0], ctas_per_dir)]
    return {"phases_cycles": res, "step_period_cycles": float(np.median(period)),
            "step_period_ns": float(np.median(period_ns)), "arrival_skew_ns": skew}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rnn", default="lstm", choices=["lstm", "gru"])
    ap.add_argument("--bidir", type=int, default=1)
    ap.add_argument("--H", type=int, default=1024)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=500)
    ap.add_argument("--In", type=int, default=2048, help="input width of the layer (the projection is not traced)")
    ap.add_argument("--json", default="", help="also write the result as JSON to this file")
    args = ap.parse_args()

    import torch
    import deepspeech_pytorch_b200 as ds
    from deepspeech_pytorch_b200 import _lib

    assert torch.cuda.is_available(), "sweep_trace.py needs a GPU"
    torch.cuda.set_device(0)
    ds.set_precision("fp16")
    code, G = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3)}[args.rnn]
    T, B, H, D = args.T, args.B, args.H, 2 if args.bidir else 1
    g = torch.Generator().manual_seed(7)
    x = torch.randn(T, B, args.In, generator=g).cuda()
    lens = torch.full((B,), T, dtype=torch.int32).cuda()
    k = 1.0 / H ** 0.5
    ws = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda() for s in
          [(G * H, args.In), (G * H, H), (G * H,), (G * H,)] * D]

    def layer():
        with torch.no_grad():
            return ds.ops.RnnLayer.apply(x, lens, code, bool(args.bidir), True, 0.1, 1e-5, None, None, None, None,
                                         None, None, *ws)

    layer()                                              # warm-up: module load, weight copies
    ctas = D * (H // 32) * 2
    trace = torch.zeros(ctas * T * SLOTS, dtype=torch.int64, device="cuda")
    lib = ds.get_lib()
    lib.ds2_fallback_count(1)
    os.environ["DS2_TRACE_FWD"] = str(trace.data_ptr())
    try:
        layer()
        torch.cuda.synchronize()
    finally:
        del os.environ["DS2_TRACE_FWD"]
    assert lib.ds2_fallback_count(1) == 0, "the forward sweep fell back to the per-step FFMA kernels"
    tr = trace.view(ctas, T, SLOTS).cpu().numpy()
    assert np.all(tr[:, 2:T - 1, 0] != 0), "no split-K forward sweep stamps: another forward kernel ran"
    out = {"card": card_info(), "rnn": args.rnn, "D": D, "H": H, "B": B, "T": T, "root": ROOT}
    out.update(phase_table(tr, T, ctas // D))
    print(json.dumps(out))
    print(f"{'phase':32s} {'cycles (median)':>16s}")
    for name, v in out["phases_cycles"].items():
        print(f"{name:32s} {v:16.0f}")
    print(f"{'step period':32s} {out['step_period_cycles']:16.0f}  ({out['step_period_ns']:.0f} ns)")
    print(f"{'arrival skew (ns, per direction)':32s} {', '.join(f'{v:.0f}' for v in out['arrival_skew_ns'])}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
