"""-m gpu: a backward on a reserve that no forward of this process filled.

A training forward in a tensor-core mode leaves an fp16 W_hh^T in its reserve for the backward sweep; a backward on a
reserve the library did not see filled converts the weights itself (include/ds2_b200.h).  The forward's copy is
f32_to_f16_transpose(W_hh) and the backward's own is the same call on the same W_hh: the same fp16 values, so both
backwards must give the same bits.  One shape per backward sweep variant (tests/test_gpu_sweep_selection.py) and one
that falls back to the FFMA step kernels.  Only the resident split-K variants read the fp16 W_hh^T; the streaming,
16-unit and FFMA backwards make the fp32 transpose either way, so for those shapes the two backwards take the same
path and the test checks that a backward gives the same bits when it runs again."""
import ctypes as C

import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib
from deepspeech_pytorch_b200._lib import RnnDesc, check, ptr, ptr_array

pytestmark = pytest.mark.gpu

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3)}

# case: (rnn, H, B, bidirectional)
CASES = {
    "bilstm1024_b32": ("lstm", 1024, 32, True),   # resident 4-CTA split-K, L2 exchange
    "unigru1024_b32": ("gru", 1024, 32, False),   # resident 8-CTA split-K
    "bilstm1536_b8": ("lstm", 1536, 8, True),     # streaming 4-CTA split-K, one launch per direction
    "bilstm160_b16": ("lstm", 160, 16, True),     # 16-unit kernel
    "bilstm72_b8": ("lstm", 72, 8, True),         # FFMA step kernels (H % 32 != 0)
}


@pytest.mark.parametrize("precision", ["tf32", "fp16"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_backward_on_an_unfilled_reserve_gives_the_same_bits(case, precision):
    rnn, H, B, bidir = CASES[case]
    code, G = CODES[rnn]
    D = 2 if bidir else 1
    T, In = 24, 96
    g = torch.Generator().manual_seed(11)
    lens = torch.tensor(sorted([max(1, T - 2 * i) for i in range(B)], reverse=True), dtype=torch.int32)
    x = torch.randn(T, B, In, generator=g)
    dy = torch.randn(T, B, H, generator=g)
    for b in range(B):
        x[int(lens[b]):, b] = 0
        dy[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    w = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda() for s in [(G * H, In), (G * H, H), (G * H,), (G * H,)] * D]
    x, dy, lens = x.cuda(), dy.cuda(), lens.cuda()
    w_ih, w_hh, b_ih, b_hh = (ptr_array(w[i::4]) for i in range(4))

    lib = ds.get_lib()
    desc = RnnDesc(code, int(bidir), T, B, In, H, 1, 0.1, 1e-5, 0)
    n = lib.ds2_rnn_reserve_floats(C.byref(desc))
    reserve = torch.empty(n, device="cuda")
    # 64 bytes into an allocation: no allocation starts there, so no earlier forward can have registered it
    copy = torch.empty(n + 16, device="cuda")[16:]
    y = torch.empty(T, B, H, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def backward(res):
        dx = torch.empty_like(x)
        grads = [torch.empty_like(t) for t in w]
        check(lib.ds2_rnn_layer_bwd(C.byref(desc), ptr(x), ptr(lens), None, None, w_ih, w_hh, b_ih, b_hh, ptr(dy),
                                    ptr(res), ptr(dx), None, None, *(ptr_array(grads[i::4]) for i in range(4)),
                                    ptr(ws), ws.numel(), stream), "ds2_rnn_layer_bwd")
        return [dx] + grads

    ds.set_precision(precision)
    try:
        ws = torch.empty(lib.ds2_rnn_workspace_bytes(C.byref(desc)), dtype=torch.uint8, device="cuda")   # per mode
        check(lib.ds2_rnn_layer_fwd(C.byref(desc), ptr(x), ptr(lens), None, None, None, None, w_ih, w_hh, b_ih, b_hh,
                                    None, None, ptr(y), None, None, ptr(reserve), ptr(ws), ws.numel(), stream),
              "ds2_rnn_layer_fwd")
        copy.copy_(reserve)   # the backward turns the reserve's gate activations into gate gradients in place
        on_forward_copy = backward(reserve)
        converted_here = backward(copy)
        torch.cuda.synchronize()
    finally:
        ds.set_precision("fp32")
    names = ["dx"] + [f"{p}[{d}]" for d in range(D) for p in ("dw_ih", "dw_hh", "db_ih", "db_hh")]
    for name, a, b in zip(names, on_forward_copy, converted_here):
        assert torch.isfinite(a).all(), name
        assert torch.equal(a, b), f"{name}: max |diff| {float((a - b).abs().max())}"
