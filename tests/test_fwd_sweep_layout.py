"""CPU checks of the register layout the split-K forward sweep finishes its step in (rnn_persistent_tc.cu:
rnn_fwd_splitk_kernel, quad_transpose, fwd_cell_unit / fwd_cell_col), restated here from the .cu source.

An m-block of the weight tile holds 16 units x 4 gate rows, row = 4 * unit + gate (GRU: gate row 3 is zero fill).
Thread tid of the MMA warpgroup (warp w = tid / 32, lane l) holds accumulator value 4 i + 2 hh + e of each 32-column
chunk at row 16 w + l / 4 + 8 hh, column 8 i + 2 (l & 3) + e (the wgmma m64nNk16 fp32 fragment).  After the
four-lane transpose, block g of a thread must hold gate g of its four cells k = 2 hh + e."""
import itertools
from pathlib import Path

import pytest

from conftest import ROOT

SRC = Path(ROOT) / "deepspeech.pytorch_b200" / "csrc"


def fragment(tid, idx):
    """(row in the 64-row m-block, column in the 32-column chunk) of accumulator value idx of thread tid"""
    w, l = tid // 32, tid % 32
    i, hh, e = idx // 4, (idx // 2) % 2, idx % 2
    return 16 * w + l // 4 + 8 * hh, 8 * i + 2 * (l & 3) + e


def fwd_cell_unit(tid, k):
    return 4 * (tid >> 5) + ((tid >> 4) & 1) + 2 * (k >> 1)


def fwd_cell_col(tid, k):
    return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + (k & 1)


def fwd_store_col(tid):
    return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + ((tid >> 4) & 1)


def fwd_units4(vals):
    """vals[tid] = the 4 values of the thread's cells k; the kernel's shfl.xor(16) round"""
    out = []
    for tid in range(128):
        ub = (tid >> 4) & 1
        pv = vals[tid ^ 16]
        r0, r1 = (pv[0], pv[2]) if not ub else (pv[1], pv[3])   # what the partner (ub ^ 1) sends
        v = vals[tid]
        out.append([r0 if ub else v[0], v[1] if ub else r0, r1 if ub else v[2], v[3] if ub else r1])
    return out


def quad_transpose(regs):
    """regs[tid] = 16 values; the kernel's two shfl.xor rounds, lane by lane (a shuffle reads the partner's value
    from before the instruction)"""
    regs = [list(r) for r in regs]
    for bit in range(2):
        for i in range(4):
            if i & (1 << bit):
                continue
            i1 = i | (1 << bit)
            for k in range(4):
                sent = []
                for tid in range(128):
                    hi = ((tid >> 2) & 3) >> bit & 1
                    sent.append(regs[tid][4 * i + k] if hi else regs[tid][4 * i1 + k])
                for tid in range(128):
                    hi = ((tid >> 2) & 3) >> bit & 1
                    r = sent[(tid & ~31) | ((tid & 31) ^ (4 << bit))]
                    if hi:
                        regs[tid][4 * i + k] = r
                    else:
                        regs[tid][4 * i1 + k] = r
    return regs


def test_layout_formulas_match_the_source():
    src = (SRC / "rnn_persistent_tc.cu").read_text()
    assert "return 4 * (tid >> 5) + ((tid >> 4) & 1) + 2 * (k >> 1);" in src
    assert "return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + (k & 1);" in src
    assert "hi ? v[4 * i + k] : v[4 * i1 + k], 4 << bit);" in src
    assert "return 8 * ((tid >> 2) & 3) + 2 * (tid & 3) + ((tid >> 4) & 1);" in src
    assert "__shfl_xor_sync(0xffffffffu, ub ? v[0] : v[1], 16);" in src
    assert "__shfl_xor_sync(0xffffffffu, ub ? v[2] : v[3], 16);" in src
    # (k, gate, unit) weight map with a box of 4 gate rows x 16 units
    assert "3, a.H, G, a.H, (size_t)a.H * a.H, (size_t)a.H, 64, 4, UT)" in src


@pytest.mark.parametrize("G,nch", [(4, 1), (4, 2), (3, 1), (3, 2)])
def test_every_cell_is_finished_by_exactly_one_thread(G, nch):
    seen = {}
    for c in range(nch):
        # what each accumulator value is: (unit, gate, column), from row = 4 * unit + gate
        regs = []
        for tid in range(128):
            vals = []
            for idx in range(16):
                row, col = fragment(tid, idx)
                vals.append((row // 4, row % 4, 32 * c + col))
            regs.append(vals)
        regs = quad_transpose(regs)
        for tid, k in itertools.product(range(128), range(4)):
            cell = (fwd_cell_unit(tid, k), 32 * c + fwd_cell_col(tid, k))
            for g in range(4):
                unit, gate, col = regs[tid][4 * g + k]
                assert (unit, col) == cell and gate == g, (tid, k, g, regs[tid][4 * g + k], cell)
            assert cell not in seen, (cell, seen[cell], (tid, k))
            seen[cell] = (tid, k)
    # 16 units x 32 * nch columns, each with all G real gates (and the GRU's zero row) in one thread
    assert set(seen) == set(itertools.product(range(16), range(32 * nch)))
    assert G in (3, 4)


def test_peer_tile_is_read_back_in_the_order_it_was_pushed():
    """thread tid pushes its 16 values of the peer's m-block to float4 slots (4 c + j) * 128 + tid of the peer's
    tile; the peer's thread tid, whose fragment covers the same rows and columns of its own m-block, reads the same
    slots: one writer per slot, and a warp's 32 lanes touch 32 consecutive 16-byte slots (no bank conflicts)"""
    for nch in (1, 2):
        slots = {}
        for c, j, tid in itertools.product(range(nch), range(4), range(128)):
            s = (4 * c + j) * 128 + tid
            assert s not in slots
            slots[s] = (c, j, tid)
        assert sorted(slots) == list(range(nch * 512))
        for c, j, w in itertools.product(range(nch), range(4), range(4)):
            warp = [(4 * c + j) * 128 + 32 * w + l for l in range(32)]
            assert warp == list(range(warp[0], warp[0] + 32))


def test_stores_take_four_consecutive_units_of_one_column():
    """after fwd_units4 value j of thread tid is unit 4 w + j at column fwd_store_col(tid): each (unit, column) of
    the 16 x 32 cells of a chunk is stored by exactly one thread, as part of one 16-byte vector"""
    vals = [[(fwd_cell_unit(tid, k), fwd_cell_col(tid, k)) for k in range(4)] for tid in range(128)]
    out = fwd_units4(vals)
    seen = set()
    for tid in range(128):
        for j in range(4):
            assert out[tid][j] == (4 * (tid >> 5) + j, fwd_store_col(tid)), (tid, j, out[tid][j])
            assert out[tid][j] not in seen
            seen.add(out[tid][j])
    assert seen == set(itertools.product(range(16), range(32)))
