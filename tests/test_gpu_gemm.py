"""The dense GEMM (`gemm_tc_kernel`) at the shapes of the benchmarked step, against fp64 products of the same operands.

The recurrent stack of the 5 x bi-LSTM-1024 step (B = 32, T' = 500: TB = 16000 rows, D*G*H = 8192, In = 1312 for
layer 0 and 1024 after it) runs four GEMM families in precision-16 mode: the input projection, dX, and per direction
dW_ih and dW_hh, whose K = TB - B operands start B columns into the transposed copies.  They take the 128 x 256 tile;
N <= 128 (the fc head) keeps the 128 x 128 one.  Partial tiles in M and N, beta, the device-side alpha factor and the
TF32 instantiations are checked here too, and repeated calls must give identical bits."""
import ctypes as C

import pytest
import torch

from gpu_helpers import rel_l2

import deepspeech_pytorch_b200 as ds

pytestmark = pytest.mark.gpu

TB, B, DGH, H = 16000, 32, 8192, 1024
F16_BOUND = 1e-5      # the bound of test_gemm_f16_tile_configurations_vs_fp64


def _p(t, off=0):
    return C.c_void_p(t.data_ptr() + t.element_size() * off)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gemm_f16(M, N, K, a, lda, b, ldb, out, alpha=1.0, beta=0.0, a_off=0, b_off=0, alpha_dev=None):
    lib = ds.get_lib()
    rc = lib.ds2_gemm_f16_scaled(M, N, K, alpha, _p(a, a_off), lda, _p(b, b_off), ldb, beta, _p(out), out.shape[1],
                                 _p(alpha_dev) if alpha_dev is not None else None, _stream())
    assert rc == 0, lib.ds2_last_error()
    return out


def ref64(M, N, K, a, lda, b, ldb, alpha=1.0, a_off=0, b_off=0):
    a64 = a.reshape(-1)[a_off:a_off + (M - 1) * lda + K].as_strided((M, K), (lda, 1)).double()
    b64 = b.reshape(-1)[b_off:b_off + (N - 1) * ldb + K].as_strided((N, K), (ldb, 1)).double()
    return alpha * (a64 @ b64.t())


def _randn(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).half()


# (name, M, N, K, lda, ldb, a_off, b_off): every GEMM of the benchmarked layer
STEP_SHAPES = []
for _In in (1312, 1024):
    STEP_SHAPES += [(f"proj-In{_In}", TB, DGH, _In, _In, _In, 0, 0),
                    (f"dX-In{_In}", TB, _In, DGH, DGH, DGH, 0, 0),
                    (f"dWih-In{_In}", DGH // 2, _In, TB, TB, TB, 0, 0)]
STEP_SHAPES += [("dWhh-fwd", DGH // 2, H, TB - B, TB, TB, B, 0),
                ("dWhh-rev", DGH // 2, H, TB - B, TB, TB, 0, B)]


@pytest.mark.parametrize("shape", STEP_SHAPES, ids=[s[0] for s in STEP_SHAPES])
def test_gemm_f16_step_shapes_vs_fp64(shape):
    """every shape of the table, with the power-of-two alpha factor the layers pass on the device (the scaled
    operand is multiplied by 2^s, alpha_dev = 2^-s); two calls give identical bits.

    Small integer operands make every product and partial sum exact in fp32, so any lost, repeated or misplaced
    k-step or tile shows as an inexact result.  With normal data the fp32 accumulation error grows with K: the
    bound of the K <= 4104 shapes, 1e-5, is scaled by K / 4096 (the K = 16000 shapes measure about 1.9e-5)."""
    name, M, N, K, lda, ldb, a_off, b_off = shape
    g = torch.Generator(device="cuda").manual_seed(11)
    s = 6.0
    alpha_dev = torch.tensor([2.0 ** -s], device="cuda")
    ints = (torch.randint(-3, 4, (M, lda), generator=g, device="cuda") * 2.0 ** s).half(), \
        torch.randint(-3, 4, (N, ldb), generator=g, device="cuda").half()
    normal = _randn((M, lda), g, 2.0 ** s), _randn((N, ldb), g)
    for exact, (a, b) in ((True, ints), (False, normal)):
        out = torch.empty(M, N, device="cuda")
        gemm_f16(M, N, K, a, lda, b, ldb, out, a_off=a_off, b_off=b_off, alpha_dev=alpha_dev)
        again = torch.empty_like(out)
        gemm_f16(M, N, K, a, lda, b, ldb, again, a_off=a_off, b_off=b_off, alpha_dev=alpha_dev)
        torch.cuda.synchronize()
        assert torch.equal(out, again), name
        ref = ref64(M, N, K, a, lda, b, ldb, 2.0 ** -s, a_off, b_off)
        if exact:
            assert torch.equal(out.double(), ref), name
        else:
            assert rel_l2(out, ref) < F16_BOUND * max(1.0, K / 4096), name
        del out, again, ref


@pytest.mark.parametrize("M,N,K", [(300, 520, 1000), (257, 200, 136), (130, 129, 72), (384, 1000, 1312),
                                   (200, 96, 200)])
@pytest.mark.parametrize("ldc_pad", [0, 1])
def test_gemm_f16_partial_tiles_and_beta(M, N, K, ldc_pad):
    """partial tiles in M and N for both tile widths, a K tail, beta = 1 and 0.5; an odd output pitch takes the
    scalar stores"""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a, b = _randn((M, K), g), _randn((N, K), g)
    c0 = torch.randn(M, N + ldc_pad, generator=g, device="cuda")
    for alpha, beta in ((1.0, 1.0), (0.5, 0.5), (1.0, 0.0)):
        out = c0.clone()
        lib = ds.get_lib()
        rc = lib.ds2_gemm_f16(M, N, K, alpha, _p(a), K, _p(b), K, beta, _p(out), N + ldc_pad, _stream())
        assert rc == 0, lib.ds2_last_error()
        ref = ref64(M, N, K, a, K, b, K, alpha) + beta * c0[:, :N].double()
        assert rel_l2(out[:, :N], ref) < F16_BOUND, (M, N, K, alpha, beta)
        if ldc_pad:
            assert torch.equal(out[:, N:], c0[:, N:])          # the pitch padding is not written


@pytest.mark.parametrize("M,N,K", [(TB, 29, H), (2048, 1024, 1024), (300, 300, 100)])
def test_gemm_tf32_vs_fp64(M, N, K):
    """TF32 instantiations: the fc head's logits shape (128 x 128 tile) and larger N (128 x 256 tile).  The TF32
    operand rounding must show (the FFMA kernel would be ~1e-7 off) and stay within its bound."""
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(M, K, generator=g, device="cuda")
    b = torch.randn(N, K, generator=g, device="cuda")
    try:
        ds.set_precision("tf32")
        out = ds.ops.gemm(a, b, trans_b=True)
        again = ds.ops.gemm(a, b, trans_b=True)
        torch.cuda.synchronize()
    finally:
        ds.set_precision("fp32")
    assert torch.equal(out, again)
    err = rel_l2(out, a.double() @ b.double().t())
    assert 1e-5 < err < 2e-3, (M, N, K, err)
