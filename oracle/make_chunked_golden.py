"""TEST INFRASTRUCTURE — generates tests/golden/chunked/*.npz by EXECUTING THE REFERENCE.

Runs only in the dev container (needs /root/reference).  Chunked transcription (reference inference.py:86-97) feeds
the chunks of a file through `DeepSpeech.forward(x, lengths, hs)` one after the other and hands each chunk's final
recurrent states to the next.  For a small bi-LSTM and a small uni-GRU with Lookahead, this runs the reference's
own, unmodified `DeepSpeech` (imported through oracle/ref_shim.py) in eval mode on CPU over 3 seeded chunks of a
2-utterance batch with ragged lengths, carrying `hs`, and stores the chunks, every chunk's output and every chunk's
final states.  The parameters are the default initialisation under torch.manual_seed(123456) plus seeded BatchNorm
statistics, which the package's `DeepSpeech` reproduces draw for draw; the fixture keeps only their float64 sums and
absolute sums (`psum/`, `pabs/`), so that a test can check that it rebuilt the same parameters.

    python oracle/make_chunked_golden.py      # rewrites tests/golden/chunked/*.npz
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden import build  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "chunked")

CASES = {
    # name: (rnn_type, bidirectional, H, layers, ctx, chunk frames, per-chunk lengths)
    # H = 128: the split-K forward sweeps (no state in chunk 0, the state kernel after it); H = 64: the 16-unit ones
    "bilstm_h128_l2": ("lstm", True, 128, 2, 0, 64, [[64, 47], [64, 64], [64, 21]]),
    "unigru_h64_l2_la5": ("gru", False, 64, 2, 5, 64, [[64, 64], [64, 37], [64, 64]]),
}


def main():
    ns = ref_shim.load_reference()
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(1)
    for name, (rnn_type, bidir, H, layers, ctx, T, chunk_lens) in CASES.items():
        torch.manual_seed(123456)
        model = build(ns, rnn_type, bidir, H, layers, ctx)
        g = torch.Generator().manual_seed(11)
        with torch.no_grad():   # non-trivial BatchNorm statistics and affine parameters
            for k, v in model.state_dict().items():
                if k.endswith("running_mean"):
                    v.copy_(0.05 * torch.randn(v.shape, generator=g))
                elif k.endswith("running_var"):
                    v.copy_(1.0 + 0.2 * torch.rand(v.shape, generator=g))
        model.eval()
        blob = {"meta": np.array(json.dumps(dict(rnn_type=rnn_type, bidirectional=bidir, hidden_size=H,
                                                  hidden_layers=layers, lookahead_context=ctx, T=T,
                                                  chunks=len(chunk_lens), torch=torch.__version__)))}
        for k, v in model.state_dict().items():
            blob["psum/" + k] = np.array(float(v.double().sum()))
            blob["pabs/" + k] = np.array(float(v.double().abs().sum()))
        hs = None
        for c, lens in enumerate(chunk_lens):
            x = torch.randn(len(lens), 1, 161, T, generator=g)
            for b, l in enumerate(lens):
                x[b, :, :, l:] = 0
            sizes = torch.tensor(lens, dtype=torch.int32)
            with torch.no_grad():
                out, out_sizes, hs = model(x, sizes, hs)
            blob[f"x/{c}"] = x.numpy()
            blob[f"sizes/{c}"] = sizes.numpy()
            blob[f"out_sizes/{c}"] = out_sizes.numpy()
            blob[f"out/{c}"] = out.numpy()
            for i, h in enumerate(hs):
                if isinstance(h, tuple):
                    blob[f"hn/{c}/{i}"] = h[0].numpy()
                    blob[f"cn/{c}/{i}"] = h[1].numpy()
                else:
                    blob[f"hn/{c}/{i}"] = h.numpy()
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **blob)
        print(f"{name}: {len(chunk_lens)} chunks -> {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
