import glob
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def golden_names():
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


class Golden:
    """One fixture written by oracle/make_golden.py (outputs of the reference itself)."""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
        self.name = name
        self.meta = json.loads(str(z["meta"]))
        self.z = z
        self.params = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("p/")}
        self.grads = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("g/")}
        self.buffers_after = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("b1/")}
        self.taps = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("tap/")}
        self.x = torch.from_numpy(z["x"])
        self.targets = torch.from_numpy(z["targets"])
        self.input_percentages = torch.from_numpy(z["input_percentages"])
        self.target_sizes = torch.from_numpy(z["target_sizes"])
        self.input_sizes = torch.from_numpy(z["input_sizes"])
        self.output_sizes = torch.from_numpy(z["output_sizes"])
        self.logits = torch.from_numpy(z["logits"])
        self.loss = float(z["loss"])
        self.eval_out = torch.from_numpy(z["eval_out"])

    def oracle_cfg(self):
        from oracle.ds2_oracle import OracleConfig
        m = self.meta
        return OracleConfig(rnn_type=m["rnn_type"], hidden_size=m["hidden_size"], hidden_layers=m["hidden_layers"],
                            bidirectional=m["bidirectional"], lookahead_context=m["lookahead_context"] or 20)


@pytest.fixture(params=golden_names())
def golden(request):
    return Golden(request.param)


def rel_err(a, b):
    """max |a-b| / max |b|  — the 'rel' of the north_star tolerance (1e-3 rel, fp32)."""
    a = torch.as_tensor(a, dtype=torch.float64)
    b = torch.as_tensor(b, dtype=torch.float64)
    denom = float(b.abs().max())
    return float((a - b).abs().max()) / (denom if denom > 0 else 1.0)
