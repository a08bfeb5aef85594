"""CPU check of the workspace sizes the library reports: each entry point lays its buffers out in one carve function
that both sizes the workspace and places the buffers, and the sizes below were recorded before those layouts were
merged with their separate size formulas.  The shapes are those the benchmark configs run (T' = 500 or 2000 frames
after the convolutions, 29 labels, targets of 200 / 400), the GEMMs of the recurrent layer and the fc head, and the
edges of each formula.  Every GEMM shape here needs at least as much room for gemm_tc's operand copies as for
gemm_simt's split-K slabs on a 132-SM H100, so the table holds with and without a GPU."""
import pytest

import deepspeech_pytorch_b200 as ds

CTC = [  # (T, B, C, max_tgt_len) -> bytes
    ((500, 32, 29, 200), 53440512),     # librispeech, unigru_lookahead
    ((500, 4, 29, 200), 6681344),       # an4
    ((2000, 8, 29, 400), 104640512),    # stress
    ((500, 32, 29, 0), 2240512),        # empty targets
    ((1, 1, 2, 0), 1792),
    ((37, 3, 29, 5), 25856),
    ((250, 7, 1000, 61), 8751104),
]
FC_HEAD = [  # (rows, H, C) -> bytes
    ((16000, 1024, 29), 132964864),     # librispeech, unigru_lookahead
    ((2000, 256, 29), 4340480),         # an4
    ((16000, 1536, 29), 198517248),     # stress
    ((1, 1, 2), 5120),
    ((1, 1024, 29), 172032),            # 57856 before the dX GEMM's workspace was counted (more labels than rows)
    ((37, 200, 29), 77056),
    ((1000, 2048, 29), 16569856),
]
BEAM = [  # (B, T, C, beam_width) -> (bytes without, with a language model)
    ((20, 500, 29, 10), (6332928, 7133184)),
    ((1, 1, 2, 1), (1792, 2048)),
    ((1, 1, 2, 128), (10496, 11776)),     # the largest beam width
    ((32, 500, 29, 128), (99484928, 115869184)),
    ((3, 120, 29, 1), (18432, 21504)),
    ((7, 333, 64, 100), (16605440, 18470400)),
    ((0, 10, 29, 10), (0, 0)),
    ((3, 0, 29, 10), (0, 0)),
    ((3, 10, 29, 0), (0, 0)),
]
ERROR_COUNTS = [  # (K, B, n_targets, max_target_size) -> bytes
    ((1, 20, 4000, 200), 97280),
    ((40, 20, 4000, 200), 97280),
    ((3, 5, 0, 0), 1536),               # no targets
    ((2, 3, 10, 4096), 1536),           # the longest reference the shared-memory blocks hold
    ((2, 3, 5000, 4097), 127744),       # one 64-symbol block more: the Myers vectors go to the workspace
    ((4, 6, 9000, 10000), 277248),
    ((0, 3, 10, 10), 0),
    ((2, 0, 10, 10), 0),
    ((2, 3, -1, 10), 0),
]
GEMM = [  # (transA, transB, M, N, K) -> bytes
    ((0, 1, 16000, 4096, 1312), 0),             # librispeech layer 1: input projection
    ((1, 0, 4096, 1312, 16000), 346112000),     # dW_ih
    ((1, 0, 4096, 1024, 15968), 327024640),     # dW_hh
    ((1, 0, 1024, 1024, 15968), 130809856),     # GRU dW_hn
    ((0, 0, 16000, 1312, 4096), 21495808),      # dX
    ((0, 1, 2000, 768, 1312), 0),               # an4
    ((1, 0, 512, 256, 1996), 6131712),
    ((0, 0, 2000, 1312, 768), 4030464),
    ((0, 1, 16000, 29, 1024), 0),               # fc head: logits
    ((1, 0, 29, 1024, 16000), 67392000),        # dW
    ((0, 0, 16000, 1024, 29), 131072),          # dX, K not a multiple of 4
    ((1, 1, 512, 512, 1001), 2056192),
    ((1, 0, 64, 96, 1001), 642560),
    ((0, 0, 100, 200, 37), 32000),
    ((1, 1, 33, 17, 3), 768),
    ((0, 1, 5, 7, 1), 0),
]
CONV = [  # (B, T) -> bytes
    ((32, 1000), 1102076672),
    ((4, 1000), 152477952),
    ((8, 4000), 1098092288),
    ((1, 1), 17054976),
    ((3, 7), 18128896),
    ((0, 5), 0),
    ((5, 0), 0),
]


@pytest.mark.parametrize("shape,want", CTC)
def test_ctc_workspace_bytes(shape, want):
    assert ds.get_lib().ds2_ctc_workspace_bytes(*shape) == want


@pytest.mark.parametrize("shape,want", FC_HEAD)
def test_fc_head_workspace_bytes(shape, want):
    assert ds.get_lib().ds2_fc_head_workspace_bytes(*shape) == want


@pytest.mark.parametrize("shape,want", BEAM)
def test_beam_decode_workspace_bytes(shape, want):
    lib = ds.get_lib()
    assert (lib.ds2_beam_decode_workspace_bytes(*shape), lib.ds2_beam_decode_lm_workspace_bytes(*shape)) == want


@pytest.mark.parametrize("shape,want", ERROR_COUNTS)
def test_error_counts_workspace_bytes(shape, want):
    assert ds.get_lib().ds2_error_counts_workspace_bytes(*shape) == want


@pytest.mark.parametrize("shape,want", GEMM)
def test_gemm_workspace_bytes(shape, want):
    assert ds.get_lib().ds2_gemm_workspace_bytes(*shape) == want


@pytest.mark.parametrize("shape,want", CONV)
def test_conv_frontend_workspace_bytes(shape, want):
    assert ds.get_lib().ds2_conv_frontend_workspace_bytes(*shape) == want


@pytest.mark.parametrize("shape", [(0, 1, 0, 7, 3000), (0, 1, 5, 0, 4096), (0, 1, 0, 0, 2048)])
def test_gemm_workspace_bytes_of_an_empty_product(shape):
    """M = 0 or N = 0 with a long K: no output tiles to split K over (this used to divide by zero)"""
    assert ds.get_lib().ds2_gemm_workspace_bytes(*shape) == 0


def al(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("rows,H,C", [
    (16000, 1024, 29), (2000, 256, 29), (16000, 1536, 29),   # the benchmark heads
    (32, 1024, 64), (40, 256, 500), (64, 1024, 256),         # more labels than rows: the dX GEMM needs the most
    (37, 200, 4096),
])
def test_fc_head_gemms_have_their_workspace_after_the_pass_buffers(rows, H, C):
    """After the buffers a pass lays out (fc_ws_carve in misc_ops.cu, restated here: the BatchNorm output and its
    sums, 4*H doubles forward and 2*H backward), the rest of the workspace holds what each of the head's ds2_gemm
    calls needs.  When it did not, gemm_tc declined the dX GEMM for want of room for its operand copy and the FFMA
    kernel ran instead."""
    lib = ds.get_lib()
    ws = lib.ds2_fc_head_workspace_bytes(rows, H, C)
    need = {"logits": lib.ds2_gemm_workspace_bytes(0, 1, rows, C, H),
            "dW": lib.ds2_gemm_workspace_bytes(1, 0, C, H, rows), "dX": lib.ds2_gemm_workspace_bytes(0, 0, rows, H, C)}
    for bwd, names in ((False, ["logits"]), (True, ["dW", "dX"])):
        rest = ws - al(rows * H * 4) - al((2 if bwd else 4) * H * 8)
        for k in names:
            assert rest >= need[k], f"{'bwd' if bwd else 'fwd'}: {k} needs {need[k]} bytes, {rest} left"
