"""torch.autograd.Function wrappers: tensors -> raw device pointers + current stream -> C-ABI.

One Function per block of the reference's hot path (SURVEY.md §8a):
  ConvFrontend  model.py:53-69,157-164,219-221   RnnLayer  model.py:80-102
  Lookahead     model.py:105-130,189-193         FcHead    model.py:195-201 (+72-77)
  CtcLoss       model.py:203,245-248
All inputs must be fp32 CUDA tensors; anything else raises (no eager fallback).
"""
import ctypes as C
import functools
import weakref

import torch

from . import _lib
from ._lib import RnnDesc, check, get_lib, ptr, ptr_array

_workspaces = {}
# Gradient sinks: parameter storage address -> the tensor its gradient must be WRITTEN into (a view of the flat
# gradient buffer, optim.FlatParams).  The C-ABI writes parameter gradients through output pointers anyway; with a
# sink registered the backward of a block hands it that view instead of a fresh tensor and returns None to autograd,
# so there is no AccumulateGrad `add` launch per parameter (59 per step at cfg-L) and no temporary.  Semantics with
# sinks: gradients are overwritten by every backward (one backward per optimizer step), not accumulated.
_SINKS = {}


def register_grad_sinks(params_and_grads):
    for p, g in params_and_grads:
        _SINKS[p.data_ptr()] = (weakref.ref(p), g)


def clear_grad_sinks():
    _SINKS.clear()


def _sink(t):
    """the registered gradient view of parameter `t`, or None (also when the entry is stale: the parameter that
    registered it is gone and the address now belongs to another tensor)"""
    e = _SINKS.get(t.data_ptr()) if t is not None else None
    if e is None:
        return None
    owner, g = e
    o = owner()
    if o is None or o.data_ptr() != t.data_ptr() or g.shape != t.shape or g.device != t.device:
        if o is None:
            _SINKS.pop(t.data_ptr(), None)
        return None
    return g


def _out(sink, like):
    """(buffer the C call writes the gradient into, value handed back to autograd)"""
    if sink is not None:
        return sink, None
    t = torch.empty_like(like)
    return t, t


def _stream():
    """current stream of the CURRENT device — every op runs under `_on_device`, which makes the tensors' device
    current first (kernels, TMA descriptors and the per-device shared-memory opt-ins all bind to it)"""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_device(fn):
    """run a Function.forward/backward with the device of its first CUDA tensor argument made current: the C
    library launches on the current device, so a model on cuda:1 in a process whose current device is cuda:0
    must not issue device-0 launches with device-1 pointers"""
    @functools.wraps(fn)
    def wrapped(ctx, *args):
        dev = next((a.device for a in args if isinstance(a, torch.Tensor) and a.is_cuda), None)
        if dev is None:
            raise _lib.Ds2Error(f"{fn.__qualname__}: no CUDA tensor among the arguments (the CUDA path has no CPU "
                                "fallback)")
        with torch.cuda.device(dev):
            lib = get_lib()
            if fn.__name__ == "forward":
                ctx.ds2_prec = lib.ds2_get_precision()
                return fn(ctx, *args)
            # backward: same arithmetic mode as the forward that recorded the graph (the switch is process-global
            # and a precision-16 model sets it only for the duration of its own forward)
            cur = lib.ds2_get_precision()
            want = getattr(ctx, "ds2_prec", cur)
            if want == cur:
                return fn(ctx, *args)
            lib.ds2_set_precision(want)
            try:
                return fn(ctx, *args)
            finally:
                lib.ds2_set_precision(cur)
    return wrapped


def workspace(nbytes, device, slot=0):
    """grow-only per-device scratch shared by all ops (they are stream-ordered).  Slots 1 and 2 alternate between
    consecutive RnnLayer backwards while deferred weight-gradient GEMMs may still read the previous layer's operand
    copies (the library orders the reuse of a slot after the side work that read it)."""
    key = (device.index if device.index is not None else torch.cuda.current_device(), slot)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = None
        _workspaces.pop(key, None)
        ws = torch.empty(int(nbytes * 1.05) + 1024, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


# ---- deferred weight-gradient GEMMs (side stream) -------------------------------------------------------------------
_side = {"stream": None, "slot": 0}


def enable_deferred_weight_grads(device=None, enable=True):
    """Let RnnLayer.backward queue dW_ih / dW_hh on a side stream so that they run in the shadow of the next layer's
    latency-bound sweep (whose pipes are mostly idle; DESIGN.md §5.6).  Effective only for parameters with registered gradient
    sinks (FlatParams(direct_grads=True)): their memory is persistent, and whoever reads the gradients
    (FusedOptimizer.step, OverlappedGradAllReduce) calls `join_deferred()` first.  Run the training loop on a stream
    of higher priority than the side stream (`torch.cuda.Stream(priority=-1)`), otherwise a queued GEMM grid keeps the
    next sweep from becoming resident and nothing overlaps."""
    lib = get_lib()
    if not enable:
        _side["stream"] = None
        check(lib.ds2_set_side_stream(None), "ds2_set_side_stream")
        return None
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    with torch.cuda.device(dev):
        _side["stream"] = torch.cuda.Stream(device=dev, priority=0)
    check(lib.ds2_set_side_stream(C.c_void_p(_side["stream"].cuda_stream)), "ds2_set_side_stream")
    return _side["stream"]


def side_stream():
    return _side["stream"]


def join_deferred():
    """order the current stream after every deferred weight-gradient GEMM queued so far"""
    if _side["stream"] is not None:
        check(get_lib().ds2_join_side_stream(_stream()), "ds2_join_side_stream")


def _req(t, name):
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == torch.float32):
        raise _lib.Ds2Error(f"{name}: expected a float32 CUDA tensor, got {t.dtype} on {t.device} "
                            "(the CUDA path has no CPU fallback)")
    return t if t.is_contiguous() else t.contiguous()


class ConvFrontend(torch.autograd.Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, out_len, w1, b1, g1, be1, rm1, rv1, w2, b2, g2, be2, rm2, rv2, training, momentum, eps):
        lib = get_lib()
        x = _req(x, "x")
        B, _, F, T = x.shape
        assert F == 161 and x.shape[1] == 1, "front-end geometry is fixed to (B,1,161,T)"
        Tp = (T - 1) // 2 + 1
        dev = x.device
        y = torch.empty(Tp, B, 1312, device=dev)
        z1 = torch.empty(B, 32, 81, Tp, device=dev)
        a1 = torch.empty(B, 32, 81, Tp, device=dev)
        z2 = torch.empty(B, 32, 41, Tp, device=dev)
        stats = torch.empty(128, device=dev)
        nws = lib.ds2_conv_frontend_workspace_bytes(B, T)
        ws = workspace(nws, dev)
        params = [_req(t, "conv param") for t in (w1, b1, g1, be1, rm1, rv1, w2, b2, g2, be2, rm2, rv2)]
        check(lib.ds2_conv_frontend_fwd(B, T, ptr(x), ptr(out_len), *[ptr(t) for t in params], int(training),
                                        float(momentum), float(eps), ptr(y), ptr(z1), ptr(a1), ptr(z2), ptr(stats),
                                        ptr(ws), ws.numel(), _stream()), "ds2_conv_frontend_fwd")
        ctx.save_for_backward(x, out_len, params[0], params[2], params[3], params[6], params[8], params[9],
                              z1, a1, z2, stats)
        ctx.dims = (B, T)
        ctx.eval_mode = not training
        ctx.sinks = [_sink(t) for t in (w1, b1, g1, be1, w2, b2, g2, be2)]
        return y

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        lib = get_lib()
        if ctx.eval_mode:
            raise _lib.Ds2Error("ConvFrontend.backward: forward ran with training=False; the BatchNorm backward "
                                "implements the batch-statistics formula only")
        x, out_len, w1, g1, be1, w2, g2, be2, z1, a1, z2, stats = ctx.saved_tensors
        B, T = ctx.dims
        dy = _req(dy, "dy")
        dev = x.device
        outs = [_out(sk, like) for sk, like in zip(ctx.sinks, (w1, g1, g1, g1, w2, g2, g2, g2))]
        (dw1, db1, dg1, dbe1, dw2, db2, dg2, dbe2), rets = zip(*outs)
        ws = workspace(lib.ds2_conv_frontend_workspace_bytes(B, T), dev)
        check(lib.ds2_conv_frontend_bwd(B, T, ptr(x), ptr(out_len), ptr(w1), ptr(g1), ptr(be1), ptr(w2), ptr(g2),
                                        ptr(be2), ptr(z1), ptr(a1), ptr(z2), ptr(stats), ptr(dy), ptr(dw1), ptr(db1),
                                        ptr(dg1), ptr(dbe1), ptr(dw2), ptr(db2), ptr(dg2), ptr(dbe2), ptr(ws),
                                        ws.numel(), _stream()), "ds2_conv_frontend_bwd")
        return (None, None, rets[0], rets[1], rets[2], rets[3], None, None, rets[4], rets[5], rets[6], rets[7], None,
                None, None, None, None)


class RnnLayer(torch.autograd.Function):
    """args: x, len_dev, rnn_type, bidirectional, training, momentum, eps, bn_gamma, bn_beta, bn_rmean, bn_rvar,
    h0, c0, then per direction (w_ih, w_hh, b_ih, b_hh)."""

    @staticmethod
    @_on_device
    def forward(ctx, x, len_dev, rnn_type, bidirectional, training, momentum, eps, bn_g, bn_b, bn_rm, bn_rv, h0, c0,
                *weights):
        lib = get_lib()
        x = _req(x, "x")
        T, B, In = x.shape
        D = 2 if bidirectional else 1
        assert len(weights) == 4 * D
        weights = [_req(w, "rnn weight") for w in weights]
        H = weights[1].shape[1]
        desc = RnnDesc(rnn_type, int(bidirectional), T, B, In, H, int(training), float(momentum), float(eps))
        dev = x.device
        y = torch.empty(T, B, H, device=dev)
        hn = torch.empty(D, B, H, device=dev)
        cn = torch.empty(D, B, H, device=dev) if rnn_type == _lib.RNN_LSTM else None
        reserve = torch.empty(lib.ds2_rnn_reserve_floats(C.byref(desc)), device=dev)
        ws = workspace(lib.ds2_rnn_workspace_bytes(C.byref(desc)), dev)
        w_ih, w_hh = ptr_array(weights[0::4]), ptr_array(weights[1::4])
        b_ih, b_hh = ptr_array(weights[2::4]), ptr_array(weights[3::4])
        bn_g, bn_b, bn_rm, bn_rv = (_req(t, "bn") for t in (bn_g, bn_b, bn_rm, bn_rv))
        h0, c0 = _req(h0, "h0"), _req(c0, "c0")
        check(lib.ds2_rnn_layer_fwd(C.byref(desc), ptr(x), ptr(len_dev), ptr(bn_g), ptr(bn_b), ptr(bn_rm), ptr(bn_rv),
                                    w_ih, w_hh, b_ih, b_hh, ptr(h0), ptr(c0), ptr(y), ptr(hn), ptr(cn), ptr(reserve),
                                    ptr(ws), ws.numel(), _stream()), "ds2_rnn_layer_fwd")
        if training and _side["stream"] is not None:
            # a tensor-core-mode training forward writes the fp16 W_hh^T of the backward sweep into `reserve` on the
            # side stream: if the graph is dropped early, the block must not be handed out before that copy has run
            reserve.record_stream(_side["stream"])
        ctx.desc = desc
        ctx.has_bn = bn_g is not None
        ctx.sinks = [_sink(bn_g), _sink(bn_b)] + [_sink(w) for w in weights]
        # the C backward assumes zero initial state and batch-statistics BatchNorm, and it turns the saved gate
        # activations into gate gradients in place: anything else must fail loudly instead of returning garbage
        ctx.no_backward = ("forward ran with training=False (no saved gate activations, running-statistics "
                           "BatchNorm)" if not training else
                           "forward was given an initial state h0/c0 (the backward sweep assumes a zero initial "
                           "state)" if (h0 is not None or c0 is not None) else None)
        ctx.consumed = False
        ctx.save_for_backward(x, len_dev, bn_g, bn_b, reserve, *weights)
        ctx.mark_non_differentiable(hn)
        if cn is not None:
            ctx.mark_non_differentiable(cn)
            return y, hn, cn
        return y, hn, None

    @staticmethod
    @_on_device
    def backward(ctx, dy, _dhn, _dcn):
        lib = get_lib()
        if ctx.no_backward:
            raise _lib.Ds2Error("RnnLayer.backward is not available: " + ctx.no_backward)
        if ctx.consumed:
            raise _lib.Ds2Error("RnnLayer.backward ran twice on the same graph: the saved gate activations were "
                                "overwritten by the gate gradients of the first pass (retain_graph is not supported)")
        ctx.consumed = True
        x, len_dev, bn_g, bn_b, reserve = ctx.saved_tensors[:5]
        weights = ctx.saved_tensors[5:]
        desc = ctx.desc
        D = 2 if desc.bidirectional else 1
        dy = _req(dy, "dy")
        dev = x.device
        dx = torch.empty_like(x)
        dg, rdg = _out(ctx.sinks[0], bn_g) if ctx.has_bn else (None, None)
        db, rdb = _out(ctx.sinks[1], bn_b) if ctx.has_bn else (None, None)
        grads, rgrads = zip(*[_out(sk, w) for sk, w in zip(ctx.sinks[2:], weights)])
        slot = 0
        desc.deferred_dw = 0
        if _side["stream"] is not None and all(sk is not None for sk in ctx.sinks[2:]):
            _side["slot"] ^= 1
            slot = 1 + _side["slot"]
            desc.deferred_dw = 1
        ws = workspace(lib.ds2_rnn_workspace_bytes(C.byref(desc)), dev, slot)
        check(lib.ds2_rnn_layer_bwd(C.byref(desc), ptr(x), ptr(len_dev), ptr(bn_g), ptr(bn_b),
                                    ptr_array(weights[0::4]), ptr_array(weights[1::4]), ptr_array(weights[2::4]),
                                    ptr_array(weights[3::4]), ptr(dy), ptr(reserve), ptr(dx), ptr(dg), ptr(db),
                                    ptr_array(grads[0::4]), ptr_array(grads[1::4]), ptr_array(grads[2::4]),
                                    ptr_array(grads[3::4]), ptr(ws), ws.numel(), _stream()), "ds2_rnn_layer_bwd")
        assert len(grads) == 4 * D
        if desc.deferred_dw:
            # the side stream still reads the layer input and the saved sequences (operand copies of the deferred
            # weight-gradient GEMMs): keep the caching allocator from handing them out before that work has run
            for t in (x, reserve):
                t.record_stream(_side["stream"])
        return (dx, None, None, None, None, None, None, rdg, rdb, None, None, None, None, *rgrads)


class Lookahead(torch.autograd.Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, w):
        lib = get_lib()
        x, w = _req(x, "x"), _req(w, "w")
        T, B, H = x.shape
        ctxlen = w.shape[-1]
        y = torch.empty_like(x)
        check(lib.ds2_lookahead_fwd(T, B, H, ctxlen, ptr(x), ptr(w), ptr(y), _stream()), "ds2_lookahead_fwd")
        ctx.save_for_backward(x, w)
        ctx.sink = _sink(w)
        return y

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        lib = get_lib()
        x, w = ctx.saved_tensors
        T, B, H = x.shape
        dy = _req(dy, "dy")
        dz, dx = torch.empty_like(x), torch.empty_like(x)
        dw, rdw = _out(ctx.sink, w)
        check(lib.ds2_lookahead_bwd(T, B, H, w.shape[-1], ptr(x), ptr(w), ptr(dy), ptr(dz), ptr(dx), ptr(dw),
                                    _stream()), "ds2_lookahead_bwd")
        return dx, rdw


class FcHead(torch.autograd.Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, g, b, rm, rv, w, training, momentum, eps, softmax):
        lib = get_lib()
        x, g, b, rm, rv, w = (_req(t, "fc") for t in (x, g, b, rm, rv, w))
        T, B, H = x.shape
        Cn = w.shape[0]
        rows = T * B
        dev = x.device
        logits = torch.empty(T, B, Cn, device=dev)
        xhat = torch.empty(rows, H, device=dev)
        stats = torch.empty(2 * H, device=dev)
        ws = workspace(lib.ds2_fc_head_workspace_bytes(rows, H, Cn), dev)
        check(lib.ds2_fc_head_fwd(rows, H, Cn, ptr(x), ptr(g), ptr(b), ptr(rm), ptr(rv), ptr(w), int(training),
                                  float(momentum), float(eps), int(softmax), ptr(logits), ptr(xhat), ptr(stats),
                                  ptr(ws), ws.numel(), _stream()), "ds2_fc_head_fwd")
        ctx.save_for_backward(g, b, w, xhat, stats)
        ctx.dims = (rows, H, Cn, T, B)
        ctx.eval_mode = not training
        ctx.sinks = [_sink(g), _sink(b), _sink(w)]
        return logits

    @staticmethod
    @_on_device
    def backward(ctx, dlogits):
        lib = get_lib()
        if ctx.eval_mode:
            raise _lib.Ds2Error("FcHead.backward: forward ran with training=False; the BatchNorm backward implements "
                                "the batch-statistics formula only")
        g, b, w, xhat, stats = ctx.saved_tensors
        rows, H, Cn, T, B = ctx.dims
        dlogits = _req(dlogits, "dlogits")
        dev = dlogits.device
        dx = torch.empty(T, B, H, device=dev)
        (dg, rdg), (db, rdb), (dw, rdw) = (_out(sk, like) for sk, like in zip(ctx.sinks, (g, b, w)))
        ws = workspace(lib.ds2_fc_head_workspace_bytes(rows, H, Cn), dev)
        check(lib.ds2_fc_head_bwd(rows, H, Cn, ptr(g), ptr(b), ptr(w), ptr(xhat), ptr(stats), ptr(dlogits), ptr(dx),
                                  ptr(dg), ptr(db), ptr(dw), ptr(ws), ws.numel(), _stream()), "ds2_fc_head_bwd")
        return dx, rdg, rdb, None, None, rdw, None, None, None, None


class CtcLoss(torch.autograd.Function):
    """sum over the batch of per-utterance CTC NLL (zero_infinity); logits (T,B,C) un-normalised."""

    @staticmethod
    @_on_device
    def forward(ctx, logits, targets, in_len, tgt_len, max_tgt_len, blank):
        lib = get_lib()
        logits = _req(logits, "logits")
        T, B, Cn = logits.shape
        dev = logits.device
        nll = torch.empty(B, device=dev)
        grad = torch.empty_like(logits)
        ws = workspace(lib.ds2_ctc_workspace_bytes(T, B, Cn, int(max_tgt_len)), dev)
        check(lib.ds2_ctc_loss_fwd_bwd(T, B, Cn, ptr(logits), ptr(targets), ptr(in_len), ptr(tgt_len),
                                       int(max_tgt_len), int(blank), ptr(nll), ptr(grad), ptr(ws), ws.numel(),
                                       _stream()), "ds2_ctc_loss_fwd_bwd")
        ctx.save_for_backward(grad)
        ctx.nll = nll
        return nll.sum()

    @staticmethod
    @_on_device
    def backward(ctx, dloss):
        (grad,) = ctx.saved_tensors
        return grad * dloss, None, None, None, None, None


def gemm(a, b, trans_a=False, trans_b=False, out=None, alpha=1.0, beta=0.0):
    """C = alpha * op(a) @ op(b) + beta * C through ds2_gemm (tests / roofline bench)."""
    lib = get_lib()
    a, b = _req(a, "a"), _req(b, "b")
    with torch.cuda.device(a.device):
        return _gemm(lib, a, b, trans_a, trans_b, out, alpha, beta)


def _gemm(lib, a, b, trans_a, trans_b, out, alpha, beta):
    M, K = (a.shape[1], a.shape[0]) if trans_a else a.shape
    N = b.shape[0] if trans_b else b.shape[1]
    if out is None:
        out = torch.empty(M, N, device=a.device)
    ws = workspace(max(256, lib.ds2_gemm_workspace_bytes(int(trans_a), int(trans_b), M, N, K)), a.device)
    check(lib.ds2_gemm(int(trans_a), int(trans_b), M, N, K, float(alpha), ptr(a), a.shape[1], ptr(b), b.shape[1],
                       float(beta), ptr(out), N, ptr(ws), ws.numel(), _stream()), "ds2_gemm")
    return out
