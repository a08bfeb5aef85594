"""Device time of the GPU beam-search decoder (`ds2_beam_decode`, row N5) per batch, next to the eval forward that
produces its input.

One batch of B = 32 utterances, T' = 500 output frames (10 s of audio), C = 29 characters is decoded with
cutoff_top_n = 40, cutoff_prob = 1.0 (the `BeamCTCDecoder` defaults) at W = 10 (the `LMConfig` default) and W = 100
(the `BeamCTCDecoder` default), on two inputs: peaked, alignment-like rows (a label run plus noise), and the softmax
output of the headline model (5 x bi-LSTM-1024, seeded weights, eval mode), which is near-uniform: the worst case,
where every prefix branches into every character.  For comparison the same model's eval forward on the same batch
is timed in the library's precision-16 mode (the reference's `precision: 16`).  Times are device times between CUDA
events around warmed-up, back-to-back calls; per frame = per batch / T' (the utterances are decoded side by side,
one CTA each).  Two utterances of the timed W = 100 configuration on the model output are checked against
`oracle/beam_oracle.py` in the same run.  The card name and power limit are read in the same run.  Needs a GPU;
prints one JSON line.

With --lm, the same probabilities are also decoded with a language model (`ds2_beam_decode_lm`, row N6, alpha = 0.8,
beta = 1.0): a seeded synthetic ARPA 3-gram at the scale of LibriSpeech's pruned 3-gram (200 000 words, 1.5 M 2-grams,
1.5 M 3-grams; written to a temporary directory).  The row then adds the host parse + trie time, the device build
time, the table bytes, the decode times with the model, and two utterances of the W = 100 model-output decode checked
against `oracle/lm_oracle.py`.

    python tools/bench_beam_decode.py [--batch 32] [--frames 500] [--iters 10] [--reps 5] [--lm]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import deepspeech_pytorch_b200 as ds  # noqa: E402
from deepspeech_pytorch_b200._lib import check, ptr  # noqa: E402
from oracle import beam_oracle as BO  # noqa: E402
from oracle import lm_oracle as LO  # noqa: E402


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": clk}
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)[:200]}


def time_events(fn, iters, reps):
    """device ms per call: events around `reps` back-to-back calls, median over `iters` windows"""
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


def peaked_probs(B, T, C, seed=0):
    rng = np.random.default_rng(seed)
    lab = np.zeros((B, T), np.int64)
    for b in range(B):
        t = 0
        while t < T:
            c = 0 if rng.random() < 0.3 else int(rng.integers(0, C))
            n = int(rng.integers(1, 5))
            lab[b, t:t + n] = c
            t += n
    lg = rng.standard_normal((B, T, C)) * 0.5 + 6.0 * np.eye(C)[lab]
    e = np.exp(lg - lg.max(-1, keepdims=True))
    return torch.from_numpy((e / e.sum(-1, keepdims=True)).astype(np.float32))


LM_ALPHA, LM_BETA = 0.8, 1.0


class Call:
    """prepared buffers for back-to-back `ds2_beam_decode` (or, with `lm`, `ds2_beam_decode_lm`) launches"""

    def __init__(self, probs, W, lm=None):
        self.probs = probs.contiguous()
        B, T, Cn = self.probs.shape
        self.shape, self.W, self.lm = (B, T, Cn), W, lm
        lib = ds.get_lib()
        self.nws = (lib.ds2_beam_decode_workspace_bytes if lm is None else lib.ds2_beam_decode_lm_workspace_bytes)(
            B, T, Cn, W)
        dev = self.probs.device
        self.ws = torch.empty(self.nws, dtype=torch.uint8, device=dev)
        self.labels = torch.empty(B, W, T, dtype=torch.int32, device=dev)
        self.timesteps = torch.empty_like(self.labels)
        self.lengths = torch.empty(B, W, dtype=torch.int32, device=dev)
        self.scores = torch.empty(B, W, dtype=torch.float64, device=dev)
        self.n_beams = torch.empty(B, dtype=torch.int32, device=dev)

    def __call__(self):
        B, T, Cn = self.shape
        if self.lm is not None:
            lm = self.lm
            check(ds.get_lib().ds2_beam_decode_lm(B, T, Cn, ptr(self.probs), None, 0, self.W, 40, 1.0,
                                                  ptr(lm.device_tables(self.probs.device)), lm.order, LM_ALPHA,
                                                  LM_BETA, lm.space, ptr(self.labels), ptr(self.timesteps),
                                                  ptr(self.lengths), ptr(self.scores), ptr(self.n_beams),
                                                  ptr(self.ws), self.nws,
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  "ds2_beam_decode_lm")
            return
        check(ds.get_lib().ds2_beam_decode(B, T, Cn, ptr(self.probs), None, 0, self.W, 40, 1.0, ptr(self.labels),
                                           ptr(self.timesteps), ptr(self.lengths), ptr(self.scores),
                                           ptr(self.n_beams), ptr(self.ws), self.nws,
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)), "ds2_beam_decode")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--lm", action="store_true", help="also decode with a LibriSpeech-pruned-3-gram-sized ARPA model")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_beam_decode: needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    ds.get_lib()
    B, Tp, Cn = args.batch, args.frames, len(ds.LABELS)

    # the headline model's eval output on an N(0,1) spectrogram batch of 2 T' input frames
    torch.manual_seed(0)
    model = ds.DeepSpeech(ds.LABELS, ds.BiDirectionalConfig(), 16, ds.AdamConfig(), ds.SpectConfig()).to(dev).eval()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 1, 161, 2 * Tp, generator=g).to(dev)
    lengths = torch.full((B,), 2 * Tp, dtype=torch.int32)

    def forward():
        with torch.no_grad():
            return model(x, lengths)

    out, out_sizes, _ = forward()
    assert tuple(out.shape) == (B, Tp, Cn), out.shape
    model_probs = out.contiguous()
    pmax = float(model_probs.max())
    inputs = {"peaked": peaked_probs(B, Tp, Cn).to(dev), "model": model_probs}

    calls = {(k, W): Call(p, W) for k, p in inputs.items() for W in (10, 100)}
    lm_row = {}
    if args.lm:
        tmp = tempfile.mkdtemp(prefix="ds2_bench_lm_")
        path = os.path.join(tmp, "synthetic_3gram.arpa.gz")
        LO.synthetic_arpa(path, 200000, 3, [1500000, 1500000], seed=7, alphabet="ABCDEFGHIJKLMNOPQRSTUVWXYZ'",
                          max_len=10, gz=True)
        from deepspeech_pytorch_b200.lm import LanguageModel
        t0 = time.perf_counter()
        lm = LanguageModel(path, ds.LABELS, 0)
        lm_row["lm_host_parse_and_trie_s"] = round(time.perf_counter() - t0, 2)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        lm.device_tables(dev)
        b.record()
        b.synchronize()
        lm_row["lm_device_build_ms"] = round(a.elapsed_time(b), 2)
        lm_row["lm_device_build_wall_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
        lm_row["lm_table_bytes"] = lm.table_bytes
        lm_row["lm_ngrams"] = [len(x) for x in lm.model.logp]
        lm_row["lm_trie_nodes"] = len(lm.trie.mask)
        lm_row["lm_alpha_beta"] = [LM_ALPHA, LM_BETA]
        calls.update({("lm_" + k, W): Call(p, W, lm) for k, p in inputs.items() for W in (10, 100)})
    for c in calls.values():
        c()
    forward()
    torch.cuda.synchronize()
    res = {}
    for _ in range(2):                                   # alternate the configurations
        for key, c in calls.items():
            res.setdefault(key, []).append(time_events(c, args.iters, args.reps))
        res.setdefault("forward", []).append(time_events(forward, args.iters, 1))
    med = {k: float(np.median([r[0] for r in v])) for k, v in res.items()}

    # oracle check of the timed W = 100 configuration on the model output, two utterances
    c = calls[("model", 100)]
    c()
    torch.cuda.synchronize()
    ref = BO.beam_decode(model_probs[:2].cpu(), None, blank=0, beam_width=100, cutoff_top_n=40, cutoff_prob=1.0)
    ok = (c.n_beams[:2].cpu().numpy().tolist() == ref["n_beams"].tolist()
          and np.array_equal(c.lengths[:2].cpu().numpy(), ref["lengths"])
          and np.array_equal(c.labels[:2].cpu().numpy(), ref["labels"])
          and np.array_equal(c.timesteps[:2].cpu().numpy(), ref["timesteps"]))
    s, r = c.scores[:2].cpu().numpy(), ref["scores"]
    f = np.isfinite(r)
    ok = ok and bool(np.all(np.abs(s[f] - r[f]) <= 1e-10 * np.maximum(1.0, np.abs(r[f]))))

    row = {"card": card_info(), "batch": B, "frames": Tp, "C": Cn, "cutoff_top_n": 40, "cutoff_prob": 1.0,
           "model_probs_max": round(pmax, 4),
           "eval_forward_ms": round(med["forward"], 3), "forward_precision": "16"}
    for (k, W) in calls:
        ms = med[(k, W)]
        row[f"decode_{k}_W{W}_ms"] = round(ms, 3)
        row[f"decode_{k}_W{W}_us_per_frame"] = round(1e3 * ms / Tp, 2)
    row["decode_model_W100_over_forward"] = round(med[("model", 100)] / med["forward"], 3)
    row["oracle_check_W100_model_2utts"] = "equal" if ok else "MISMATCH"
    row["oracle_margin"] = float(f"{ref['margin']:.3g}")
    if args.lm:
        row.update(lm_row)
        row["decode_lm_model_W100_over_forward"] = round(med[("lm_model", 100)] / med["forward"], 3)
        c = calls[("lm_model", 100)]
        c()
        torch.cuda.synchronize()
        ref = LO.beam_decode_lm(model_probs[:2].cpu(), None, ds.LABELS, LO.read_arpa(path), LM_ALPHA, LM_BETA,
                                blank=0, beam_width=100, cutoff_top_n=40, cutoff_prob=1.0)
        lm_ok = (c.n_beams[:2].cpu().numpy().tolist() == ref["n_beams"].tolist()
                 and np.array_equal(c.lengths[:2].cpu().numpy(), ref["lengths"])
                 and np.array_equal(c.labels[:2].cpu().numpy(), ref["labels"])
                 and np.array_equal(c.timesteps[:2].cpu().numpy(), ref["timesteps"]))
        s, r = c.scores[:2].cpu().numpy(), ref["scores"]
        f = np.isfinite(r)
        lm_ok = lm_ok and bool(np.all(np.abs(s[f] - r[f]) <= 1e-10 * np.maximum(1.0, np.abs(r[f]))))
        row["lm_oracle_check_W100_model_2utts"] = "equal" if lm_ok else "MISMATCH"
        row["lm_oracle_margin"] = float(f"{ref['margin']:.3g}")
        row["lm_top_beam_utt0"] = ''.join(ds.LABELS[int(x)] for x in c.labels[0, 0, :int(c.lengths[0, 0])])[:80]
        ok = ok and lm_ok
    print(json.dumps(row))
    if not ok:
        raise SystemExit("bench_beam_decode: GPU result differs from the oracle")


if __name__ == "__main__":
    main()
