"""Device time of CTC forced alignment (`ds2_ctc_align`) per batch.

Two shapes: B = 32 utterances of T' = 500 output frames (10 s of audio, the eval batch of the README) with targets of
about 200 characters, and a long case, B = 4 of T' = 30 000 frames (10 minutes) with about 6 000 characters.  C = 29.
The rows are peaked and alignment-like: each utterance's frame path walks its own target (runs of 1-3 frames per
character, blanks between some) and the logits are noise + 6 on the path's label, as tools/bench_beam_decode.py builds
its peaked rows.  The call takes logits (apply_log_softmax = 1): log-softmax, target offsets and the alignment kernel,
three launches.  Times are device times between CUDA events around warmed-up, back-to-back calls.  Where torchaudio
is importable, `torchaudio.functional.forced_align` on CUDA, one utterance per call as it takes them, is timed on the
same log-probabilities and its frame labels are compared with ours.  The card name and power limit are read in the
same run.  Needs a GPU; prints one JSON line.

    python tools/bench_align.py [--iters 10] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import deepspeech_pytorch_b200 as ds  # noqa: E402
from deepspeech_pytorch_b200._lib import check, ptr  # noqa: E402


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": clk}
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def time_events(fn, iters, reps):
    """device ms per call: events around `reps` back-to-back calls, median and min over `iters` windows"""
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / reps)
    return float(np.median(ts)), float(np.min(ts))


def alignment_rows(B, T, C, L, seed=0):
    """(T,B,C) fp32 logits whose argmax path spells each row's target, and the targets (B, ~L)"""
    rng = np.random.default_rng(seed)
    lab = np.zeros((B, T), np.int64)
    targets = []
    for b in range(B):
        tg = []
        t = 0
        while t < T and len(tg) < L:
            c = int(rng.integers(1, C))
            if tg and c == tg[-1] or rng.random() < 0.3:
                t += int(rng.integers(1, 3))                 # a blank run (required between repeats)
            tg.append(c)
            n = int(rng.integers(1, 4))
            lab[b, t:t + n] = c
            t += n
        targets.append(tg)
    lg = rng.standard_normal((T, B, C)).astype(np.float32) * 0.5
    lg[np.arange(T)[:, None], np.arange(B)[None, :], lab.T] += 6.0
    return torch.from_numpy(lg), targets


class Call:
    """prepared buffers for back-to-back `ds2_ctc_align` launches on logits (T,B,C)"""

    def __init__(self, logits, targets):
        dev = logits.device
        self.x = logits.contiguous()
        T, B, Cn = self.x.shape
        self.shape = (T, B, Cn)
        self.max_l = max(len(t) for t in targets)
        self.targets = torch.tensor([c for t in targets for c in t], dtype=torch.int64, device=dev)
        self.in_len = torch.full((B,), T, dtype=torch.int32, device=dev)
        self.tgt_len = torch.tensor([len(t) for t in targets], dtype=torch.int32, device=dev)
        lib = ds.get_lib()
        self.nws = lib.ds2_ctc_align_workspace_bytes(T, B, Cn, self.max_l)
        self.ws = torch.empty(self.nws, dtype=torch.uint8, device=dev)
        self.labels = torch.empty(B, T, dtype=torch.int32, device=dev)
        self.flp = torch.empty(B, T, dtype=torch.float32, device=dev)
        self.spans = torch.empty(B, self.max_l, 2, dtype=torch.int32, device=dev)
        self.scores = torch.empty(B, dtype=torch.float64, device=dev)

    def __call__(self):
        T, B, Cn = self.shape
        check(ds.get_lib().ds2_ctc_align(T, B, Cn, ptr(self.x), 1, ptr(self.targets), ptr(self.in_len),
                                         ptr(self.tgt_len), self.max_l, 0, ptr(self.labels), ptr(self.flp),
                                         ptr(self.spans), ptr(self.scores), ptr(self.ws), self.nws,
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)), "ds2_ctc_align")


def torchaudio_case(call, targets, iters):
    try:
        import torchaudio.functional as TAF
    except Exception as e:  # pragma: no cover
        return {"torchaudio": f"not importable ({type(e).__name__})"}
    lp = torch.log_softmax(call.x, dim=2).transpose(0, 1).contiguous()      # (B,T,C)
    B, T, _ = lp.shape
    tgs = [torch.tensor([t], dtype=torch.int32, device=lp.device) for t in targets]
    Tl = torch.tensor([T], dtype=torch.int32, device=lp.device)

    def run():
        return [TAF.forced_align(lp[b:b + 1], tgs[b], Tl, torch.tensor([len(targets[b])], dtype=torch.int32,
                                                                      device=lp.device), blank=0)[0]
                for b in range(B)]
    try:
        paths = run()
    except Exception as e:  # pragma: no cover
        return {"torchaudio": f"forced_align failed ({type(e).__name__}: {str(e)[:120]})"}
    torch.cuda.synchronize()
    med, mn = time_events(run, iters, 1)
    call()
    same = sum(int(torch.equal(paths[b][0].long().cpu(), call.labels[b].long().cpu())) for b in range(B))
    return {"torchaudio_ms": round(med, 3), "torchaudio_min_ms": round(mn, 3), "torchaudio_same_paths": f"{same}/{B}"}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_align: needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    row = {"bench": "ctc_align", "card": card_info()}
    for name, (B, T, L, iters, reps) in {"b32_t500": (32, 500, 200, args.iters, args.reps),
                                         "b4_t30000": (4, 30000, 6000, 3, 1)}.items():
        logits, targets = alignment_rows(B, T, 29, L, seed=B)
        call = Call(logits.to(dev), targets)
        call()
        torch.cuda.synchronize()
        res = [time_events(call, iters, reps) for _ in range(2)]
        feasible = int(torch.isfinite(call.scores).sum())
        r = {"B": B, "T": T, "L_mean": round(float(np.mean([len(t) for t in targets])), 1), "max_l": call.max_l,
             "ms": round(float(np.median([x[0] for x in res])), 3), "min_ms": round(min(x[1] for x in res), 3),
             "us_per_frame": round(1e3 * float(np.median([x[0] for x in res])) / T, 3),
             "workspace_bytes": call.nws, "feasible": f"{feasible}/{B}"}
        r.update(torchaudio_case(call, targets, 3 if T > 1000 else args.iters))
        row[name] = r
    print(json.dumps(row))


if __name__ == "__main__":
    main()
