"""Device time and TFLOP/s of the dense GEMM (`gemm_tc_kernel`) at the shapes of the benchmarked step.

The shapes are those of the 5 x bi-LSTM-1024 training step (B = 32, T' = 500, so TB = 16000 rows; D*G*H = 8192;
In = 1312 for layer 0 and 1024 for the other layers) in precision-16 mode, through `ds2_gemm_f16`:

    proj    gates = x16 . W16^T             TB x 8192 x In
    dX      dG16 . W16^T                    TB x In x 8192
    dW_ih   dG16^T . x16^T  (per direction)  4096 x In x TB
    dW_hh   dG16^T . h16^T  (per direction)  4096 x 1024 x (TB - B), one operand offset by B columns

plus the fc head's logits GEMM (TB x 29 x 1024, TF32) through `ds2_gemm`.  Each shape is timed with CUDA events
around single calls after warm-up; the median of `--iters` calls (at least 50) is reported with TFLOP/s and the share
of the data sheet's dense rate (989 TFLOP/s fp16, 495 TF32, H100 SXM at 700 W).  The card name, power limit and SM
clocks are read in the same run.

`--lib PATH` (repeatable) times other builds of the library in the same process, round-robin with this tree's, so
that two versions are compared under the same conditions.  Needs a GPU; prints a table and one JSON line.

    python tools/bench_gemm.py [--lib other/libds2_b200.so] [--rounds 3] [--iters 50]
"""
import argparse
import ctypes as C
import json
import os
import subprocess

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THIS_LIB = os.path.join(ROOT, "deepspeech.pytorch_b200", "libds2_b200.so")
PEAK_TFLOPS = {"f16": 989.0, "tf32": 495.0}
PREC_F16 = 2
TB, B, DGH, H = 16000, 32, 8192, 1024


def card_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=" + q,
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def load(path):
    lib = C.CDLL(os.path.abspath(path), mode=C.RTLD_LOCAL)
    vp, i32, f32, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    lib.ds2_gemm_f16.restype = i32
    lib.ds2_gemm_f16.argtypes = [i32] * 3 + [f32, vp, i32, vp, i32, f32, vp, i32, vp]
    lib.ds2_gemm.restype = i32
    lib.ds2_gemm.argtypes = [i32] * 5 + [f32, vp, i32, vp, i32, f32, vp, i32, vp, sz, vp]
    lib.ds2_gemm_workspace_bytes.restype = sz
    lib.ds2_gemm_workspace_bytes.argtypes = [i32] * 5
    lib.ds2_set_precision.restype = i32
    lib.ds2_set_precision.argtypes = [i32]
    lib.ds2_last_error.restype = C.c_char_p
    if lib.ds2_set_precision(PREC_F16) != 0:
        raise SystemExit(f"{path}: ds2_set_precision failed: {lib.ds2_last_error()}")
    return lib


def shapes():
    """(name, kind, M, N, K, lda, ldb, a_off, b_off): operands are K-major; offsets in elements"""
    out = []
    for In in (1312, 1024):
        out.append((f"proj In={In}", "f16", TB, DGH, In, In, In, 0, 0))
        out.append((f"dX In={In}", "f16", TB, In, DGH, DGH, DGH, 0, 0))
        out.append((f"dW_ih In={In}", "f16", DGH // 2, In, TB, TB, TB, 0, 0))
    out.append(("dW_hh fwd", "f16", DGH // 2, H, TB - B, TB, TB, B, 0))
    out.append(("dW_hh rev", "f16", DGH // 2, H, TB - B, TB, TB, 0, B))
    out.append(("fc head", "tf32", TB, 29, H, H, H, 0, 0))
    return out


class Case:
    def __init__(self, spec, g):
        self.name, self.kind, self.M, self.N, self.K, self.lda, self.ldb, self.a_off, self.b_off = spec
        dt = torch.float16 if self.kind == "f16" else torch.float32
        self.a = torch.randn(self.M, self.lda, generator=g, device="cuda").to(dt)
        self.b = torch.randn(self.N, self.ldb, generator=g, device="cuda").to(dt)
        self.c = torch.empty(self.M, self.N, device="cuda")
        self.flop = 2.0 * self.M * self.N * self.K

    def call(self, lib, ws, stream):
        es = self.a.element_size()
        pa = C.c_void_p(self.a.data_ptr() + es * self.a_off)
        pb = C.c_void_p(self.b.data_ptr() + es * self.b_off)
        pc = C.c_void_p(self.c.data_ptr())
        if self.kind == "f16":
            rc = lib.ds2_gemm_f16(self.M, self.N, self.K, 1.0, pa, self.lda, pb, self.ldb, 0.0, pc, self.N, stream)
        else:
            rc = lib.ds2_gemm(0, 1, self.M, self.N, self.K, 1.0, pa, self.lda, pb, self.ldb, 0.0, pc, self.N,
                              C.c_void_p(ws.data_ptr()), ws.numel(), stream)
        if rc != 0:
            raise SystemExit(f"{self.name}: rc={rc}: {lib.ds2_last_error()}")


def time_calls(case, lib, ws, stream, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        case.call(lib, ws, stream)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", action="append", default=[], help="another build of libds2_b200.so to time alongside")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.iters < 50:
        raise SystemExit("bench_gemm: --iters must be at least 50")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm: needs a CUDA device")
    torch.cuda.set_device(0)
    paths = [THIS_LIB] + args.lib
    libs = [load(p) for p in paths]
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(0)
    cases = [Case(s, g) for s in shapes()]
    ws_bytes = max(lib.ds2_gemm_workspace_bytes(0, 1, c.M, c.N, c.K) for lib in libs for c in cases)
    ws = torch.empty(max(256, ws_bytes), dtype=torch.uint8, device="cuda")
    for case in cases:
        for lib in libs:
            for _ in range(args.warmup):
                case.call(lib, ws, stream)
    torch.cuda.synchronize()
    card_before = card_info()

    times = {(c.name, p): [] for c in cases for p in paths}
    rounds = {(c.name, p): [] for c in cases for p in paths}
    for _ in range(args.rounds):
        for case in cases:
            for lib, p in zip(libs, paths):
                ts = time_calls(case, lib, ws, stream, args.iters)
                times[(case.name, p)] += ts
                rounds[(case.name, p)].append(float(np.median(ts)))
    card_after = card_info()

    rows = []
    hdr = f"{'shape':<16} {'M x N x K':<20} " + " ".join(f"{'lib%d ms' % i:>9} {'TFLOP/s':>8} {'%peak':>6}"
                                                        for i in range(len(paths)))
    print(hdr)
    for case in cases:
        line = f"{case.name:<16} {'%dx%dx%d' % (case.M, case.N, case.K):<20} "
        row = {"shape": case.name, "kind": case.kind, "M": case.M, "N": case.N, "K": case.K, "libs": []}
        for p in paths:
            ms = float(np.median(times[(case.name, p)]))
            tf = case.flop / (ms * 1e-3) / 1e12
            pk = 100.0 * tf / PEAK_TFLOPS[case.kind]
            line += f"{ms:9.4f} {tf:8.1f} {pk:6.1f} "
            row["libs"].append({"lib": p, "median_ms": round(ms, 5), "tflops": round(tf, 1),
                                "pct_of_datasheet": round(pk, 1),
                                "round_medians_ms": [round(r, 5) for r in rounds[(case.name, p)]]})
        print(line)
        rows.append(row)
    for i, p in enumerate(paths):
        print(f"lib{i} = {p}")
    print(json.dumps({"card_before": card_before, "card_after": card_after, "iters": args.iters,
                      "rounds": args.rounds, "libs": paths, "shapes": rows}))


if __name__ == "__main__":
    main()
