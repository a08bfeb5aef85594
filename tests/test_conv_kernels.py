"""Resource usage, warp roles and tile schedule of the conv2 tap-in-N kernel, read from the built library (no GPU
needed).

`conv_tc_kernel` is persistent, one CTA of 384 threads per SM: a producer warpgroup trims its registers to 40 so that
each of the two MMA warpgroups can hold a whole tile's 64 x 352 fp32 accumulator (176 registers per thread) in up to
232, which is 168 per thread at launch.  A spill or a stack frame would put local memory into the mainloop or the
epilogue that the other warpgroup's MMAs are meant to hide (DESIGN §5.3)."""
import os
import re
import shutil
import subprocess

import pytest

from deepspeech_pytorch_b200 import _lib

KERNEL = "_ZN3ds214conv_tc_kernelENS_12ConvTcParamsE"
PRODUCER_REGS, MMA_REGS = 40, 232
LAUNCH_REGS = (128 * PRODUCER_REGS + 256 * MMA_REGS) // 384
TO = 54                                   # outputs per 64-position tile


def _cuobjdump(*args):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return subprocess.run([tool, *args, _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def test_conv_tc_kernel_has_no_local_memory_and_launches_with_the_handed_over_registers():
    lines = _cuobjdump("--dump-resource-usage").splitlines()
    usage = {}
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S+):", line)
        if m:
            usage[m.group(1)] = dict(re.findall(r"(\w+):(\d+)", lines[i + 1]))
    assert {name for name in usage if "conv_tc_kernel" in name} == {KERNEL}, sorted(usage)
    u = usage[KERNEL]
    assert u["LOCAL"] == "0" and u["STACK"] == "0", u
    assert int(u["REG"]) == LAUNCH_REGS, u


def test_conv_tc_kernel_mma_warpgroups_hold_the_whole_tile():
    sass = _cuobjdump("-sass", "-fun", KERNEL)
    assert "USETMAXREG.DEALLOC.CTAPOOL 0x%x" % PRODUCER_REGS in sass
    assert re.search(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \w+, 0x%x" % MMA_REGS, sass)
    # two m64n176k8 (both N halves) per k-step, four k-steps per stage; one wgmma group kept in flight
    assert sass.count("HGMMA.64x176x8.F32.TF32") == 8
    assert re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", sass)


def _tile_stages(B, Tp, R_in, classes, row_mul, row_step):
    """stages (vertical taps with an input row) of every tile, in the kernel's tile order: class, b, d, time tile"""
    ntt = -(-Tp // TO)
    stages = []
    for R_out, J, row_off in classes:
        for b in range(B):
            for d in range(R_out):
                r0 = row_mul * d + row_off
                nj = sum(1 for j in range(J) if 0 <= r0 + j * row_step < R_in)
                stages += [nj] * ntt
    return stages


@pytest.mark.parametrize("name,args", [
    ("forward", (32, 500, 81, [(41, 21, -10)], 2, 1)),
    ("data gradient", (32, 500, 41, [(41, 11, 5), (40, 10, 5)], 1, -1)),
])
def test_static_tile_stride_balances_the_stages_per_cta(name, args):
    """At the benchmark shape (B = 32, T' = 500) on 132 SMs, CTA c takes tiles c, c + 132, ...: the edge rows' shorter
    tap ranges average out, every CTA streams within 1 % of the mean number of stages."""
    stages = _tile_stages(*args)
    grid = min(len(stages), 132)
    per_cta = [sum(stages[c::grid]) for c in range(grid)]
    mean = sum(per_cta) / grid
    print(f"{name}: {len(stages)} tiles, per-CTA stages min {min(per_cta)} max {max(per_cta)} mean {mean:.1f}")
    assert max(per_cta) <= 1.01 * mean and min(per_cta) >= 0.99 * mean, (min(per_cta), max(per_cta), mean)
