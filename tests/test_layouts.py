"""CPU checks of index arithmetic that the CUDA kernels rely on (restated here from the .cu sources; the -m gpu
tests exercise the kernels themselves)."""
import itertools
import re
from pathlib import Path

import pytest

from conftest import ROOT

SRC = Path(ROOT) / "deepspeech.pytorch_b200" / "csrc"


# ---- exchange-tile layout of the cluster split-K sweeps (rnn_persistent_tc.cu: xt_cgs / xt_slice / xt_off) ----
def xt_cgs(rows):
    return (rows + rows // 8) * 4 + 4


def xt_slice(rows, nb):
    return (nb // 4) * xt_cgs(rows)


def xt_off(rows, row, col):
    return (col >> 2) * xt_cgs(rows) + (row + (row >> 3)) * 4 + (col & 3)


def test_exchange_tile_formulas_match_the_source():
    src = (SRC / "rnn_persistent_tc.cu").read_text()
    assert "return (rows + rows / 8) * 4 + 4;" in src
    assert "return (nb / 4) * xt_cgs(rows);" in src
    assert "return (col >> 2) * xt_cgs(rows) + (row + (row >> 3)) * 4 + (col & 3);" in src


@pytest.mark.parametrize("rows,nb", [(16, 8), (16, 24), (16, 32), (16, 40), (16, 256), (64, 16), (64, 32), (64, 48)])
def test_exchange_tile_layout_is_injective_and_aligned(rows, nb):
    offs = {}
    for r, c in itertools.product(range(rows), range(nb)):
        o = xt_off(rows, r, c)
        assert 0 <= o < xt_slice(rows, nb)
        assert o not in offs, (r, c, offs[o])
        offs[o] = (r, c)
    # 16-byte st.async targets: the first column of a group of 4 lands on a multiple of 4 floats, groups stay together
    for r, c in itertools.product(range(rows), range(0, nb, 4)):
        assert xt_off(rows, r, c) % 4 == 0
        assert [xt_off(rows, r, c + i) for i in range(4)] == list(range(xt_off(rows, r, c), xt_off(rows, r, c) + 4))
    # reader pattern of a warp: rows base + {0, 4, 8, 12}, eight batch columns: at most 2-way bank conflicts
    # (a column-group pitch = 8 mod 32 floats would make it conflict-free: noted in DESIGN.md section 7)
    for base in range(0, min(rows, 16) - 12):
        for b0 in range(0, nb - 7, 8):
            banks = [xt_off(rows, base + 4 * q, b0 + bb) % 32 for q in range(4) for bb in range(8)]
            assert max(banks.count(v) for v in set(banks)) <= 2, (base, b0)


# ---- grouping of K chunks in the resident sweeps (grp_begin / grp_count) ----------------------------------
@pytest.mark.parametrize("nkr", [1, 2, 4, 5, 8, 16, 24, 32, 120])
def test_chunk_groups_cover_every_chunk_once(nkr):
    ng = (nkr + 3) // 4
    chunks = []
    for g in range(ng):
        c0, c1 = 4 * g, min(nkr, 4 * (g + 1))
        assert c0 < c1
        chunks += list(range(c0, c1))
    assert chunks == list(range(nkr)) and ng <= 32


# ---- conv2 weight gradient: which delayed copy / box coordinate serves tap kw (conv_tc.cu: KW_OF_BLOCK) ----
def test_conv2_wgrad_tap_order_matches_the_box_plan():
    src = (SRC / "conv_tc.cu").read_text()
    m = re.search(r"KW_OF_BLOCK\[11\] = \{([0-9, ]+)\}", src)
    order = [int(v) for v in m.group(1).split(",")]
    plan = []                                     # (box coordinate offset, first copy, number of copies)
    for coord, first, n in [(-4, 0, 2), (0, 0, 4), (4, 0, 4), (8, 3, 1)]:
        for copy in range(first, first + n):
            plan.append((coord, copy))
    assert len(plan) == 11 and sorted(order) == list(range(11))
    for blk, kw in enumerate(order):
        coord, copy = plan[blk]
        sh = kw - 5                               # a1[t + sh] = copy[t + sh + copy]  (copy delayed by `copy` steps)
        assert coord == sh + copy and coord % 4 == 0


# ---- conv1 weight gradient: de-interleaved, delayed copies of the stride-2 time axis (conv_tc.cu: KW1_OF_GROUP) ----
def test_conv1_wgrad_tap_columns_match_the_box_plan():
    """xs[s][q][u'] = x[2 (u' - s) + q]; box 1 at coordinate t0 spans s = 0..3, q = 0..1, box 2 at t0 + 4 spans
    s = 2..3: group g of 8 shared-memory rows must hold x[2 t + kw - 5] for kw = KW1_OF_GROUP[g], and the six classes
    of (4 output rows) x (8 input rows) must reach every vertical tap exactly once per output row."""
    src = (SRC / "conv_tc.cu").read_text()
    m = re.search(r"KW1_OF_GROUP\[12\] = \{([-0-9, ]+)\}", src)
    table = [int(v) for v in m.group(1).split(",")]
    groups = [(0, s, q) for s in range(4) for q in range(2)] + [(4, s, q) for s in (2, 3) for q in range(2)]
    assert len(groups) == len(table) == 12
    seen = set()
    for g, (coord, s, q) in enumerate(groups):
        # row element k of the box is xs[s][q][t0 + coord + k] = x[2 (t0 + coord + k - s) + q]: for output step
        # t = t0 + k that is x[2 t + 2 (coord - s) + q], i.e. tap column kw = 5 + 2 (coord - s) + q
        kw = 5 + 2 * (coord - s) + q
        if 0 <= kw <= 10:
            assert table[g] == kw
            seen.add(kw)
        else:
            assert table[g] == -1
    assert seen == set(range(11))
    # vertical taps: kh = 8 c + j - 2 i for class c, input row j of 8, output row i of 4
    for i in range(4):
        hits = sorted(8 * c + j - 2 * i for c in range(6) for j in range(8) if 0 <= 8 * c + j - 2 * i < 41)
        assert hits == list(range(41))


# ---- conv2 weight gradient: taps stacked in M (conv_tc.cu: wg::KH_PER, wg::GROUPS) ----
def test_conv2_wgrad_tap_groups_cover_every_vertical_tap_once():
    """CTA class (parity, group) owns taps kh = parity + 2 (KH_PER group + i), i < KH_PER (a class whose first tap is past
    kh = 20 has no work); the dz2 row of tap i for input row r is d = (r + 10 - kh) / 2.  Every (d, kh) pair of the
    41 x 21 products must be produced by exactly one (r, class, i)."""
    src = (SRC / "conv_tc.cu").read_text()
    kh_per = int(re.search(r"constexpr int KH_PER = (\d+);", src).group(1))
    groups = int(re.search(r"constexpr int GROUPS = (\d+);", src).group(1))
    seen = {}
    for parity in range(2):
        for g in range(groups):
            kh0 = parity + 2 * kh_per * g
            if kh0 >= 21:
                continue
            nkh = min(kh_per, (21 - 1 - kh0) // 2 + 1)
            assert nkh >= 1
            for r in range(parity, 81, 2):
                for i in range(nkh):
                    kh = kh0 + 2 * i
                    assert (r + 10 - kh) % 2 == 0
                    d = (r + 10 - kh0) // 2 - i
                    if 0 <= d < 41:
                        assert 2 * d + kh - 10 == r
                        seen[(d, kh)] = seen.get((d, kh), 0) + 1
    want = {(d, kh) for d in range(41) for kh in range(21) if 0 <= 2 * d + kh - 10 < 81}
    assert set(seen) == want and all(v == 1 for v in seen.values())
