"""Device time of the language-model weight search (`ds2_beam_decode_lm_grid` + `ds2_error_counts`) against the way
the reference's search_lm_params.py does it: one full evaluation per (alpha, beta) pair.

Input: N = 256 utterances of T' = 500 output frames (10 s of audio), the softmax output of the headline model
(5 x bi-LSTM-1024, seeded weights, eval mode, precision 16) on N(0,1) spectrograms, in batches of 32 as in
tools/bench_beam_decode.py; reference transcripts are seeded word sequences over the language model's vocabulary.  The
language model is the same seeded synthetic ARPA 3-gram at LibriSpeech-pruned scale (200 000 words, 1.5 M 2-grams,
1.5 M 3-grams, written to a temporary directory).  cutoff_top_n = 40, cutoff_prob = 1.0.

Rows, for W = 100 and W = 10:
  * grid_K{K}: device time of one `decode_best_grid` launch over all N utterances for K pairs plus the
    `ds2_error_counts` launch, per (pair, utterance), K in {1, 4, 16, 64}; median and spread (min, max) over
    --windows windows after a warm-up of every shape;
  * current_K{K}, K in {1, 4}: wall clock to the (wer, cer) of K pairs the current way: per pair,
    `BeamCTCDecoder.decode` per batch of 32 (every beam converted to strings on the host) plus the metrics.py classes;
    one run (it is orders of magnitude slower);
  * the check that both ways give identical (wer, cer) for those pairs.
Also `ds2_error_counts` alone on the K = 64 rows against metrics.edit_distance on the K = 1 rows (per row), with the
per-row counts checked, and, with --parent-lib, `ds2_beam_decode_lm` (B = 32, W = 100, the model output, the case of
tools/bench_beam_decode.py --lm) timed with this library and with the given one alternately in the same process.
The card name and power limit are read in the same run.  Needs a GPU; prints one JSON line.

    python tools/bench_lm_search.py [--windows 3] [--parent-lib path/to/libds2_b200.so]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import deepspeech_pytorch_b200 as ds  # noqa: E402
from deepspeech_pytorch_b200 import _lib  # noqa: E402
from deepspeech_pytorch_b200._lib import check, ptr  # noqa: E402
from deepspeech_pytorch_b200.evaluation import error_counts, rates  # noqa: E402
from deepspeech_pytorch_b200.metrics import CharErrorRate, WordErrorRate, edit_distance  # noqa: E402
from oracle import lm_oracle as LO  # noqa: E402
from bench_beam_decode import card_info, time_events  # noqa: E402

N, TP, BATCH = 256, 500, 32
KS, KS_CURRENT = (1, 4, 16, 64), (1, 4)


def model_outputs(dev):
    torch.manual_seed(0)
    model = ds.DeepSpeech(ds.LABELS, ds.BiDirectionalConfig(), 16, ds.AdamConfig(), ds.SpectConfig()).to(dev).eval()
    outs = []
    with torch.no_grad():
        for b in range(N // BATCH):
            g = torch.Generator().manual_seed(1 + b)
            x = torch.randn(BATCH, 1, 161, 2 * TP, generator=g).to(dev)
            out, _, _ = model(x, torch.full((BATCH,), 2 * TP, dtype=torch.int32))
            outs.append(out.float().contiguous())
    del model
    return torch.cat(outs)


def references(lm, seed=3):
    """seeded transcripts: 15-25 words of the model's spellable vocabulary"""
    rng = np.random.default_rng(seed)
    words = [w.decode() if isinstance(w, bytes) else w for w in lm.model.words]
    words = [w for w in words if w and w[0] != '<' and all(c in ds.LABELS[1:-1] for c in w)]
    out = []
    for _ in range(N):
        s = ' '.join(words[int(i)] for i in rng.integers(0, len(words), int(rng.integers(15, 26))))
        out.append([ds.LABELS.index(c) for c in s])
    return out


def spread(ts):
    return {"median": round(float(np.median(ts)), 4), "min": round(float(np.min(ts)), 4),
            "max": round(float(np.max(ts)), 4)}


def parent_ab(lm, probs, windows, parent_path):
    """ds2_beam_decode_lm, B = 32, W = 100, with this library and the parent's, alternately"""
    libs = {"new": ds.get_lib(), "parent": C.CDLL(os.path.abspath(parent_path))}
    for name in ("ds2_beam_decode_lm_workspace_bytes", "ds2_beam_decode_lm"):
        fn = getattr(libs["parent"], name)
        fn.restype, fn.argtypes = _lib.PROTOTYPES[name]
    p = probs[:BATCH].contiguous()
    B, T, Cn = p.shape
    W = 100
    dev = p.device
    tables = lm.device_tables(dev)
    bufs = {}
    for k, lib in libs.items():
        nws = lib.ds2_beam_decode_lm_workspace_bytes(B, T, Cn, W)
        bufs[k] = dict(nws=nws, ws=torch.empty(nws, dtype=torch.uint8, device=dev),
                       labels=torch.empty(B, W, T, dtype=torch.int32, device=dev),
                       ts=torch.empty(B, W, T, dtype=torch.int32, device=dev),
                       lengths=torch.empty(B, W, dtype=torch.int32, device=dev),
                       scores=torch.empty(B, W, dtype=torch.float64, device=dev),
                       n=torch.empty(B, dtype=torch.int32, device=dev))

    def call(k):
        lib, b = libs[k], bufs[k]
        rc = lib.ds2_beam_decode_lm(B, T, Cn, ptr(p), None, 0, W, 40, 1.0, ptr(tables), lm.order, 0.8, 1.0, lm.space,
                                    ptr(b["labels"]), ptr(b["ts"]), ptr(b["lengths"]), ptr(b["scores"]), ptr(b["n"]),
                                    ptr(b["ws"]), b["nws"], C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, k
    for k in libs:
        call(k)
    torch.cuda.synchronize()
    same = all(torch.equal(bufs["new"][x], bufs["parent"][x]) for x in ("labels", "ts", "lengths", "scores", "n"))
    res = {k: [] for k in libs}
    for _ in range(windows):
        for k in libs:
            res[k].append(time_events(lambda: call(k), 5, 2)[0])
    return {"ms_new": spread(res["new"]), "ms_parent": spread(res["parent"]), "outputs_equal": same}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--parent-lib", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lm_search: needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    row = {"card": card_info(), "utterances": N, "frames": TP}
    probs = model_outputs(dev)
    sizes = torch.full((N,), TP, dtype=torch.int32, device=dev)

    tmp = tempfile.mkdtemp(prefix="ds2_bench_lm_search_")
    path = os.path.join(tmp, "synthetic_3gram.arpa.gz")
    LO.synthetic_arpa(path, 200000, 3, [1500000, 1500000], seed=7, alphabet="ABCDEFGHIJKLMNOPQRSTUVWXYZ'",
                      max_len=10, gz=True)
    from deepspeech_pytorch_b200.lm import LanguageModel
    lm = LanguageModel(path, ds.LABELS, 0)
    refs = references(lm)
    targets = torch.tensor([x for r in refs for x in r], dtype=torch.int64)
    tsz = torch.tensor([len(r) for r in refs], dtype=torch.int32)
    targets_d = targets.to(dev)
    target_dec = ds.GreedyDecoder(ds.LABELS)
    space = ds.LABELS.index(' ')
    rng = np.random.default_rng(5)
    all_pairs = [(float(a), float(b)) for a, b in zip(rng.uniform(0, 3, max(KS)), rng.uniform(0, 1, max(KS)))]
    ok = True

    for W in (100, 10):
        dec = ds.BeamCTCDecoder(ds.LABELS, lm_path=path, beam_width=W)
        grid_out = {}

        def grid(K):
            counts = torch.zeros(K, 4, dtype=torch.int64, device=dev)
            labels, lengths = dec.decode_best_grid(probs, sizes, all_pairs[:K])
            error_counts(labels, lengths, targets_d, tsz, 0, space, pair_counts=counts, rows=False)
            grid_out[K] = (labels, lengths, counts)

        for K in KS:                                        # warm-up of every shape
            grid(K)
        torch.cuda.synchronize()
        times = {K: [] for K in KS}
        for _ in range(args.windows):
            for K in KS:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                grid(K)
                b.record()
                b.synchronize()
                times[K].append(1e3 * a.elapsed_time(b) / (K * N))     # us per (pair, utterance)
        for K in KS:
            row[f"W{W}_grid_K{K}_us_per_pair_utt"] = spread(times[K])
        res_grid = {K: [rates(c) for c in grid_out[K][2].cpu().tolist()] for K in KS}

        # the current way: one evaluation per pair, decode per batch of 32 + metrics.py
        for K in KS_CURRENT:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cur = []
            for a, b in all_pairs[:K]:
                dec.reset_params(a, b)
                wer, cer = WordErrorRate(dec, target_dec), CharErrorRate(dec, target_dec)
                for s in range(0, N, BATCH):
                    off = int(tsz[:s].sum())
                    n = int(tsz[s:s + BATCH].sum())
                    for m in (wer, cer):
                        m.update(probs[s:s + BATCH], sizes[s:s + BATCH].cpu(), targets[off:off + n],
                                 tsz[s:s + BATCH])
                cur.append((wer.compute(), cer.compute()))
            dt = time.perf_counter() - t0
            row[f"W{W}_current_K{K}_us_per_pair_utt"] = round(1e6 * dt / (K * N), 1)
            same = cur == res_grid[K]
            row[f"W{W}_current_K{K}_equal_to_grid"] = same
            ok = ok and same
        row[f"W{W}_wer_cer_pair0"] = [round(x, 3) for x in res_grid[1][0]]

        if W == 100:
            # ds2_error_counts alone (K = 64 rows) against metrics.edit_distance (K = 1 rows), per row
            labels, lengths, _ = grid_out[64]
            ts = []
            for _ in range(args.windows):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                rows = error_counts(labels, lengths, targets_d, tsz, 0, space)
                b.record()
                b.synchronize()
                ts.append(1e3 * a.elapsed_time(b) / (64 * N))
            row["counts_alone_us_per_row"] = spread(ts)
            L1, n1 = grid_out[1][0][0].cpu(), grid_out[1][1][0].cpu()
            rows1 = error_counts(grid_out[1][0], grid_out[1][1], targets_d, tsz, 0, space)[0].cpu()
            t0 = time.perf_counter()
            py = []
            off = 0
            for u in range(N):
                h = ''.join(ds.LABELS[int(x)] for x in L1[u, :int(n1[u])])
                r = ''.join(ds.LABELS[x] for x in refs[u])
                py.append([edit_distance(h.replace(' ', ''), r.replace(' ', '')), len(r.replace(' ', '')),
                           edit_distance(h.split(), r.split()), len(r.split())])
            row["python_edit_distance_us_per_row"] = round(1e6 * (time.perf_counter() - t0) / N, 1)
            same = py == rows1.tolist()
            row["counts_equal_to_python"] = same
            ok = ok and same
            row["W100_mean_hyp_len"] = round(float(n1.float().mean()), 1)
            row["mean_ref_len"] = round(float(tsz.float().mean()), 1)

    if args.parent_lib:
        row["beam_decode_lm_B32_W100_ab"] = parent_ab(lm, probs, args.windows, args.parent_lib)
        ok = ok and row["beam_decode_lm_B32_W100_ab"]["outputs_equal"]
    print(json.dumps(row))
    if not ok:
        raise SystemExit("bench_lm_search: the two ways differ")


if __name__ == "__main__":
    main()
