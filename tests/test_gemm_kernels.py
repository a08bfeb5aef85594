"""Resource usage and mainloop shape of the dense GEMM kernels, read from the built library (no GPU needed).

`gemm_tc_kernel` runs one CTA of 384 threads per SM: 168 registers per thread at launch, which the producer warpgroup
trims to 40 so that each MMA warpgroup can hold its 128 fp32 accumulators (128 x 256 tile) in up to 232.  A spill
or a stack frame would put local memory into the epilogue or the mainloop, and the MMA warpgroups must keep one wgmma
group in flight across stages (DESIGN §5.2)."""
import os
import re
import shutil
import subprocess

import pytest

from deepspeech_pytorch_b200 import _lib

# (F16, BN) -> mangled name
INSTANTIATIONS = {(f16, bn): "_ZN3ds214gemm_tc_kernelILb%dELi%dEEEv14CUtensorMap_stS1_iiiffPfiPKf" % (f16, bn)
                  for f16 in (0, 1) for bn in (128, 256)}
# registers per thread at launch: exactly what `setmaxnreg` hands over, 128 x 40 (producer) + 256 x 232 (MMA) =
# 384 x 168.  With fewer at launch the MMA warpgroups' `setmaxnreg.inc 232` could never be granted.
PRODUCER_REGS, MMA_REGS = 40, 232
LAUNCH_REGS = (128 * PRODUCER_REGS + 256 * MMA_REGS) // 384


def _cuobjdump(*args):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return subprocess.run([tool, *args, _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def test_gemm_kernels_have_no_local_memory_and_launch_with_the_handed_over_registers():
    lines = _cuobjdump("--dump-resource-usage").splitlines()
    usage = {}
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S+):", line)
        if m:
            usage[m.group(1)] = dict(re.findall(r"(\w+):(\d+)", lines[i + 1]))
    gemms = {name for name in usage if "gemm_tc_kernel" in name}
    assert gemms == set(INSTANTIATIONS.values()), sorted(gemms)
    for name in gemms:
        u = usage[name]
        assert u["LOCAL"] == "0" and u["STACK"] == "0", (name, u)
        assert int(u["REG"]) == LAUNCH_REGS, (name, u)


def test_gemm_mainloop_keeps_one_wgmma_group_in_flight():
    for (f16, bn), name in INSTANTIATIONS.items():
        sass = _cuobjdump("-sass", "-fun", name)
        shape = "HGMMA.64x%dx%d" % (bn, 16 if f16 else 8)
        assert shape in sass, (name, shape)
        assert re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", sass), name
        assert "USETMAXREG.DEALLOC.CTAPOOL 0x%x" % PRODUCER_REGS in sass and "0x%x" % MMA_REGS in sass, name
        assert "USETMAXREG.TRY_ALLOC.CTAPOOL" in sass, name
