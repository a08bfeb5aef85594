"""The tensor-core conv front-end (conv2 forward / data gradient / weight gradient and the conv1 weight gradient on
wgmma) against float64 ATen at the benchmark shape and at odd, ragged shapes, and its bitwise repeatability."""
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from gpu_helpers import make_model, rel, rel_l2
from oracle import ds2_oracle as O

pytestmark = pytest.mark.gpu


def _frontend(T, B, lens, seed=0):
    """front-end module with seeded weights, input x (zero beyond each length), output lengths"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, 161, T, generator=g)
    for b, l in enumerate(lens):
        x[b, :, :, l:] = 0
    model = make_model("gru", True, 8, 1).train()
    sm = model.conv.seq_module
    with torch.no_grad():
        for m in (sm[0], sm[3]):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g).cuda() * 0.05)
            m.bias.copy_(torch.randn(m.bias.shape, generator=g).cuda() * 0.1)
    out_len = model.get_seq_lens(torch.tensor(lens)).cuda()
    return model, x.cuda(), out_len


def _run(model, x, out_len, dy_seed=9):
    sm = model.conv.seq_module
    params = [sm[i].weight for i in (0, 1, 3, 4)] + [sm[i].bias for i in (0, 1, 3, 4)]
    y = ds.ops.ConvFrontend.apply(x, out_len, sm[0].weight, sm[0].bias, sm[1].weight, sm[1].bias,
                                  sm[1].running_mean, sm[1].running_var, sm[3].weight, sm[3].bias, sm[4].weight,
                                  sm[4].bias, sm[4].running_mean, sm[4].running_var, True, 0.1, 1e-5)
    dy = torch.randn(y.shape, generator=torch.Generator().manual_seed(dy_seed)).cuda()
    for p in params:
        p.grad = None
    (y * dy).sum().backward()
    torch.cuda.synchronize()
    return y.detach().clone(), dy, [p.grad.detach().clone() for p in params]


def _reference(model, x, out_len, dy):
    """float64 ATen: conv2d / batch_norm / clamp with the mask after every module (oracle.conv_frontend)"""
    sm = model.conv.seq_module
    P = {f"conv.seq_module.{k}": v.detach().double().clone() for k, v in sm.state_dict().items()
         if v.dtype.is_floating_point}
    leaves = [P[f"conv.seq_module.{i}.weight"] for i in (0, 1, 3, 4)] + [P[f"conv.seq_module.{i}.bias"]
                                                                       for i in (0, 1, 3, 4)]
    for t in leaves:
        t.requires_grad_(True)
    z = O.conv_frontend(x.double(), out_len, P, True, {})
    B, C, D, Tp = z.shape
    y = z.reshape(B, C * D, Tp).permute(2, 0, 1)
    (y * dy.double()).sum().backward()
    return y.detach(), [t.grad.detach() for t in leaves]


def _check(T, B, lens):
    ds.set_precision("tf32")
    model, x, out_len = _frontend(T, B, lens)
    y, dy, grads = _run(model, x, out_len)
    y_ref, g_ref = _reference(model, x, out_len, dy)
    assert rel(y, y_ref) < 3e-3 and rel_l2(y, y_ref) < 1e-3, (rel(y, y_ref), rel_l2(y, y_ref))
    # weights of conv1, BN1, conv2, BN2, then their biases; the conv biases are ~0 after the BatchNorm (pure rounding)
    for i, (ga, gr) in enumerate(zip(grads[:4] + grads[5:6] + grads[7:8], g_ref[:4] + g_ref[5:6] + g_ref[7:8])):
        assert torch.isfinite(ga).all() and rel_l2(ga, gr) < 3e-2, (i, rel_l2(ga, gr))
    ol = out_len.cpu()
    for b in range(B):
        if int(ol[b]) < y.shape[0]:
            assert float(y[int(ol[b]):, b].abs().max()) == 0.0


def test_tensor_core_frontend_benchmark_shape_vs_float64():
    """B = 32, T = 1000 (the benchmarked shape), every utterance full length"""
    _check(1000, 32, [1000] * 32)


@pytest.mark.parametrize("T,B", [(301, 5), (640, 17), (1000, 1)])
def test_tensor_core_frontend_odd_ragged_shapes_vs_float64(T, B):
    """odd batches (B = 1, 5, 17), a partially filled last time tile, ragged lengths with fully masked tiles; T = 301
    (T' = 151) takes the FFMA conv2 weight gradient, the others the tensor-core one"""
    lens = sorted([max(40, T - (T // (B + 1)) * i) for i in range(B)], reverse=True)
    _check(T, B, lens)


def test_tensor_core_frontend_is_bit_repeatable():
    """two forward + backward runs from the same state: identical outputs and gradients"""
    ds.set_precision("tf32")
    model, x, out_len = _frontend(1000, 32, [1000 - 7 * i for i in range(32)], seed=3)
    sm = model.conv.seq_module
    state = {k: v.clone() for k, v in sm.state_dict().items()}
    y1, _, g1 = _run(model, x, out_len)
    sm.load_state_dict(state)
    y2, _, g2 = _run(model, x, out_len)
    assert torch.equal(y1, y2)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)
