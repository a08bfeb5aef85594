"""CPU check of ds2_rnn_workspace_bytes: after the buffers a pass lays out (layer_ws_carve in rnn_layer.cu, restated
here), the rest of the workspace holds what every fp32 / TF32 GEMM of the layer needs (ds2_gemm_workspace_bytes).
When it did not, gemm_tc declined for want of room for its operand transposes and the FFMA gemm_simt ran instead:
other bits and a much slower GEMM.  The shapes include ones without the fp16 operand copies in the precision-16 mode
(B % 8 != 0, T*B < 128), where the dX GEMM falls back to ds2_gemm."""
import ctypes as C

import pytest

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3), "tanh": (_lib.RNN_TANH, 1)}
PRECS = {"fp32": _lib.PREC_FP32, "tf32": _lib.PREC_TF32, "fp16": _lib.PREC_F16}


def al(n):
    return (n + 255) // 256 * 256


def carve_bytes(rnn, bidir, T, B, In, H, bwd, prec):
    """bytes of the buffers of one pass, in the order layer_ws_carve lays them out"""
    D, G = (2 if bidir else 1), CODES[rnn][1]
    TB, GH = T * B, G * H
    n = al(TB * In * 4) * (3 if bwd else 1) + al((2 if bwd else 4) * In * 8)   # BN: xbn [xhat, dxbn], sums
    if bwd:
        n += D * al(GH * H * 4) + al(D * B * H * 4)                             # W_hh^T per direction, carry
    if prec == "fp16" and B % 8 == 0 and In % 8 == 0 and H % 8 == 0 and (not bwd or TB >= 128):
        if bwd:
            n += (2 * al(TB * D * GH * 2) + al(TB * In * 2) + al(D * H * TB * 2) * (2 if rnn == "gru" else 1) +
                  al(In * D * GH * 2) + al(16 * 4))
        else:
            n += al(TB * In * 2) + al(D * GH * In * 2)
    return n


@pytest.mark.parametrize("prec", sorted(PRECS))
@pytest.mark.parametrize("rnn,bidir,T,B,In,H", [
    ("gru", False, 50, 1, 1312, 1024),     # precision 16 without fp16 copies (B % 8 != 0)
    ("lstm", True, 100, 5, 1312, 1024),
    ("lstm", True, 10, 8, 1024, 1024),     # T*B < 128: no fp16 copies in the backward
    ("gru", True, 500, 4, 1312, 256),      # an4
    ("lstm", True, 500, 32, 1312, 1024),   # librispeech, first layer
    ("gru", False, 500, 32, 1024, 1024),   # unigru_lookahead, later layers
    ("tanh", True, 37, 3, 200, 72),
])
def test_the_gemms_have_their_workspace_after_the_pass_buffers(rnn, bidir, T, B, In, H, prec):
    lib = ds.get_lib()
    code, G = CODES[rnn]
    TB, Kr, GH = T * B, (T - 1) * B, G * H
    rows_x = 2 * H if rnn == "gru" else GH
    was = lib.ds2_get_precision()
    lib.ds2_set_precision(PRECS[prec])
    try:
        desc = _lib.RnnDesc(code, int(bidir), T, B, In, H, 1, 0.1, 1e-5, 0)
        ws = lib.ds2_rnn_workspace_bytes(C.byref(desc))
        gemm = {"projection": (0, 1, TB, GH, In), "dW_ih": (1, 0, GH, In, TB), "dW_hh": (1, 0, rows_x, H, Kr),
                "dW_hn": (1, 0, H, H, Kr), "dX": (0, 0, TB, In, GH)}
        need = {k: lib.ds2_gemm_workspace_bytes(*v) for k, v in gemm.items()}
    finally:
        lib.ds2_set_precision(was)
    for bwd, names in ((False, ["projection"]), (True, ["dW_ih", "dW_hh", "dW_hn", "dX"])):
        rest = ws - carve_bytes(rnn, bidir, T, B, In, H, bwd, prec)
        for k in names:
            assert rest >= need[k], f"{'bwd' if bwd else 'fwd'}: {k} needs {need[k]} bytes, {rest} left"
