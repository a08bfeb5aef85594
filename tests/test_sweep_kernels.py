"""Resource usage of the recurrent sweep kernels, read from the built library (no GPU needed).

The sweeps keep one CTA per SM resident for a whole layer, so local memory (spills or stack) sits on the per-step
critical path, and the register counts of the benchmarked instantiations decide whether one CTA of 288 threads
still fits an SM.  DESIGN §5.1 states these figures; this test keeps them true while the sweep file is edited."""
import os
import re
import shutil
import subprocess

import pytest

from deepspeech_pytorch_b200 import _lib

# (mangled name, demangled form for messages, most registers allowed)
BENCHMARKED = [
    ("_ZN3ds221rnn_fwd_splitk_kernelILi0ELi8EEEvNS_13PersistParamsE",
     "rnn_fwd_splitk_kernel<LSTM, 8>", 134),
    ("_ZN3ds221rnn_bwd_splitk_kernelILi0ELb1ELi4ELi16ELb1EEEvNS_13PersistParamsE",
     "rnn_bwd_splitk_kernel<LSTM, true, 4, 16, true>", 136),
    ("_ZN3ds221rnn_bwd_splitk_kernelILi0ELb1ELi4ELi16ELb0EEEvNS_13PersistParamsE",
     "rnn_bwd_splitk_kernel<LSTM, true, 4, 16, false>", 128),
]


def _resource_usage():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    usage = {}
    lines = txt.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S+):", line)
        if m:
            usage[m.group(1)] = dict(re.findall(r"(\w+):(\d+)", lines[i + 1]))
    return usage


def test_sweep_kernels_do_not_spill():
    usage = _resource_usage()
    sweeps = {name: u for name, u in usage.items() if re.search(r"rnn_\w+_kernel", name)}
    assert any("rnn_bwd_splitk_kernel" in name for name in sweeps)
    for name, u in sweeps.items():
        assert u["LOCAL"] == "0", (name, u)


def test_benchmarked_sweeps_keep_their_registers():
    usage = _resource_usage()
    for mangled, pretty, max_regs in BENCHMARKED:
        assert mangled in usage, pretty
        u = usage[mangled]
        assert u["STACK"] == "0", (pretty, u)
        assert int(u["REG"]) <= max_regs, (pretty, u)
