"""-m gpu: the split-K forward sweep (`rnn_fwd_splitk_kernel`) at the edges of the shapes it takes, against the fp32
path: LSTM and GRU, one and two 32-column accumulator chunks (B <= 32 and 32 < B <= 64, with padded columns),
H = 1024 (compile-time chunk count) and H = 256 / 640 (runtime chunk count, a partial last group of K chunks),
uni- and bidirectional, ragged lengths with fully masked utterances.  The backward pass reads the gate values and
cell states the forward sweep saves, so the gradients check those too."""
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200 import _lib
from gpu_helpers import rel, rel_l2

pytestmark = pytest.mark.gpu

CODES = {"lstm": (_lib.RNN_LSTM, 4), "gru": (_lib.RNN_GRU, 3)}


def _layer(rnn, T, B, In, H, bidir, seed):
    code, G = CODES[rnn]
    g = torch.Generator().manual_seed(seed)
    lens = sorted([max(0, T - 3 * i) for i in range(B)], reverse=True)
    lens[0] = T
    lens[-2:] = [0, 0]
    lens = torch.tensor(lens, dtype=torch.int32)
    x = torch.randn(T, B, In, generator=g).cuda()
    dy = torch.randn(T, B, H, generator=g).cuda()
    for b in range(B):
        x[int(lens[b]):, b] = 0
        dy[int(lens[b]):, b] = 0
    k = 1.0 / H ** 0.5
    ws = [((torch.rand(s, generator=g) * 2 - 1) * k).cuda().requires_grad_(True) for s in
          [(G * H, In), (G * H, H), (G * H,), (G * H,)] * (2 if bidir else 1)]
    lens_dev = lens.cuda()

    def run():
        for w in ws:
            w.grad = None
        xx = x.clone().requires_grad_(True)
        y, hn, _ = ds.ops.RnnLayer.apply(xx, lens_dev, code, bidir, True, 0.1, 1e-5, None, None, None, None, None,
                                         None, *ws)
        y.backward(dy)
        torch.cuda.synchronize()
        return [y.detach(), hn.detach(), xx.grad.clone()] + [w.grad.clone() for w in ws]
    return run, lens


@pytest.mark.parametrize("rnn,B,H,bidir", [
    ("lstm", 32, 1024, True), ("gru", 32, 1024, False), ("lstm", 20, 1024, False), ("gru", 64, 1024, True),
    ("lstm", 48, 256, True), ("gru", 20, 256, True), ("lstm", 32, 640, False), ("gru", 40, 640, True)])
def test_split_k_forward_sweep_agrees_with_the_fp32_path(rnn, B, H, bidir):
    run, lens = _layer(rnn, T=29, B=B, In=96, H=H, bidir=bidir, seed=31)
    ds.set_precision("fp32")
    ref = run()
    ds.set_precision("fp16")
    lib = ds.get_lib()
    lib.ds2_fallback_count(1)
    got = run()
    again = run()
    assert lib.ds2_fallback_count(1) == 0, "a sweep fell back to the per-step FFMA kernels"
    for b in range(B):
        L = int(lens[b])
        if L < got[0].shape[0]:
            assert float(got[0][L:, b].abs().max()) == 0.0, b
    assert rel(got[0], ref[0]) < 5e-3 and rel(got[1], ref[1]) < 5e-3
    for a, r in zip(got[2:], ref[2:]):
        assert rel_l2(a, r) < 1e-2
    # bit-repeatable: the outputs and every gradient that is not a bias gradient (where the backward sweep does not
    # reduce the bias gradients itself, e.g. GRU with B > 32, a column sum with float atomics does)
    biases = {3 + 4 * d + j for d in range(2) for j in (2, 3)}
    for i, (a, b_) in enumerate(zip(got, again)):
        if i not in biases:
            assert torch.equal(a, b_), f"output {i} is not bit-repeatable"
