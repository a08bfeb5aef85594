"""The persistent conv2 tap-in-N kernel at the shapes its tile schedule treats specially, against float64 ATen: fewer
tiles than SMs (a grid below one CTA per SM, every second MMA warpgroup without a tile), and tile counts that leave
one MMA warpgroup of some CTAs a tile fewer than the other."""
import pytest
import torch

from test_gpu_conv_frontend import _check

pytestmark = pytest.mark.gpu

TO = 54   # outputs per time tile


def _tiles(B, T):
    """tiles of the forward (41 output rows) and of the data gradient (41 even + 40 odd rows)"""
    ntt = -(-((T - 1) // 2 + 1) // TO)
    return ntt * 41 * B, ntt * 81 * B


@pytest.mark.parametrize("T,B", [(100, 1), (200, 2), (331, 3)])
def test_conv_tile_schedule_edge_shapes_vs_float64(T, B):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fwd, dgrad = _tiles(B, T)
    if (T, B) == (100, 1):
        assert fwd < sms and dgrad < sms          # one tile per CTA: warpgroup 1 idles in every CTA
    else:
        assert fwd % sms and dgrad % sms          # some CTAs take one tile more than others
    lens = sorted([max(40, T - (T // (B + 1)) * i) for i in range(B)], reverse=True)
    _check(T, B, lens)
