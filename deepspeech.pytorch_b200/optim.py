"""Flat fp32 parameter / gradient buffers + the fused clip-and-step kernels (SURVEY.md §8f N1).

The reference steps `torch.optim.AdamW` / SGD-Nesterov (model.py:273-297) after Lightning's
`clip_grad_norm_(400)` (configs/librispeech.yaml:12).  Here every parameter is a view into ONE
contiguous buffer (so the data-parallel exchange is a single all-reduce, dist.py) and the update is
two kernels over that buffer: a sum-of-squares reduction, then clip-scale + AdamW/SGD fused.
"""
import torch

from ._lib import check, current_stream, get_lib

_ALIGN = 64  # floats: 256-byte aligned views (TMA / float4 friendly)


class FlatParams:
    """`direct_grads=True` registers every gradient view as the sink of its parameter (ops.register_grad_sinks): the
    backward kernels then write the gradients straight into `self.grad` (no AccumulateGrad adds, no temporaries, no
    zero_grad needed — every parameter's gradient is overwritten by every backward)."""

    def __init__(self, model, direct_grads: bool = False):
        params = [p for p in model.parameters() if p.requires_grad]
        dev = params[0].device
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        self.n, self.params, self.offsets = n, params, offs
        self.data = torch.zeros(n, device=dev)
        self.grad = torch.zeros(n, device=dev)
        for p, o in zip(params, offs):
            self.data[o:o + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.data[o:o + p.numel()].view(p.shape)
            p.grad = self.grad[o:o + p.numel()].view(p.shape)
        self.direct_grads = bool(direct_grads)
        if self.direct_grads:
            from . import ops
            ops.register_grad_sinks((p, p.grad) for p in params)

    def zero_grad(self):
        if not self.direct_grads:          # with sinks every gradient is overwritten by the next backward
            self.grad.zero_()


class FusedOptimizer:
    """AdamW (AdamConfig) or SGD-Nesterov (SGDConfig) on a FlatParams, with global-norm clipping and the
    1/world gradient scale of DDP's mean folded in."""

    def __init__(self, flat: FlatParams, optim_cfg, max_norm: float = 400.0):
        from .configs import is_kind
        self.flat, self.cfg, self.max_norm = flat, optim_cfg, float(max_norm)
        self.adam = is_kind(optim_cfg, "AdamConfig")
        if not self.adam and not is_kind(optim_cfg, "SGDConfig"):
            raise ValueError("Optimizer has not been specified correctly.")
        self.lr = float(optim_cfg.learning_rate)
        self.step_count = 0
        dev = flat.data.device
        self.m = torch.zeros_like(flat.data)
        self.v = torch.zeros_like(flat.data) if self.adam else None
        self.norm = torch.zeros(1, device=dev)
        self.ws = torch.zeros(64, device=dev)

    def step(self, grad_scale: float = 1.0):
        with torch.cuda.device(self.flat.data.device):     # launches bind to the current device
            from . import ops
            ops.join_deferred()                            # weight-gradient GEMMs queued on the side stream
            self._step(grad_scale)

    def _step(self, grad_scale):
        lib = get_lib()
        f = self.flat
        st = current_stream()
        self.step_count += 1
        if self.adam:
            b1, b2 = self.cfg.betas
            check(lib.ds2_adamw_step(f.n, f.data.data_ptr(), f.grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                     self.lr, float(b1), float(b2), float(self.cfg.eps), float(self.cfg.weight_decay),
                                     self.step_count, float(grad_scale), self.max_norm, self.norm.data_ptr(),
                                     self.ws.data_ptr(), st), "ds2_adamw_step")
        else:
            check(lib.ds2_sgd_nesterov_step(f.n, f.data.data_ptr(), f.grad.data_ptr(), self.m.data_ptr(), self.lr,
                                            float(self.cfg.momentum), float(self.cfg.weight_decay),
                                            int(self.step_count == 1), float(grad_scale), self.max_norm,
                                            self.norm.data_ptr(), self.ws.data_ptr(), st), "ds2_sgd_nesterov_step")

    def anneal(self):
        """ExponentialLR(gamma=learning_anneal) once per epoch (model.py:293-296)"""
        self.lr *= float(self.cfg.learning_anneal)

    def torch_optimizer(self, params=None):
        """the torch.optim.AdamW / SGD(nesterov=True) that `configure_optimizers` builds (model.py:273-291) over
        `params` (default: the flat parameters, i.e. `model.parameters()` order), at the current learning rate and
        without state"""
        params = self.flat.params if params is None else list(params)
        c = self.cfg
        if self.adam:
            opt = torch.optim.AdamW(params, lr=float(c.learning_rate), betas=tuple(c.betas), eps=float(c.eps),
                                    weight_decay=float(c.weight_decay))
        else:
            opt = torch.optim.SGD(params, lr=float(c.learning_rate), momentum=float(c.momentum), nesterov=True,
                                  weight_decay=float(c.weight_decay))
        for g in opt.param_groups:
            g["initial_lr"] = float(c.learning_rate)    # what ExponentialLR adds to the group
            g["lr"] = self.lr
        return opt

    def state_dict(self):
        """the state in torch.optim.AdamW / SGD's layout: per parameter index (model.parameters() order) `step` and
        `exp_avg` / `exp_avg_sq` (AdamW) or `momentum_buffer` (SGD), and torch's `param_groups` with the current
        `lr`.  The state tensors are views of the flat `m` / `v` buffers, not copies; a parameter has no state before
        the first step, as in torch."""
        groups = self.torch_optimizer().state_dict()["param_groups"]
        state = {}
        if self.step_count > 0:
            for i, (p, o) in enumerate(zip(self.flat.params, self.flat.offsets)):
                n = p.numel()
                s = {"step": torch.tensor(float(self.step_count))}
                if self.adam:
                    s["exp_avg"] = self.m[o:o + n].view(p.shape)
                    s["exp_avg_sq"] = self.v[o:o + n].view(p.shape)
                else:
                    s["momentum_buffer"] = self.m[o:o + n].view(p.shape)
                state[i] = s
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """the inverse of `state_dict` (also accepts what torch.optim.AdamW / SGD saved over the same parameters):
        copies the moments into the flat buffers and restores the step count and the learning rate"""
        params = self.flat.params
        if len(sd["param_groups"]) != 1 or len(sd["param_groups"][0]["params"]) != len(params):
            raise ValueError(f"optimizer state for {[len(g['params']) for g in sd['param_groups']]} parameters, "
                             f"this optimizer has one group of {len(params)}")
        keys = ("exp_avg", "exp_avg_sq") if self.adam else ("momentum_buffer",)
        bufs = (self.m, self.v) if self.adam else (self.m,)
        state = sd["state"]
        steps = set()
        for b in bufs:
            b.zero_()
        for i, (p, o) in enumerate(zip(params, self.flat.offsets)):
            s = state.get(i)
            if s is None:
                continue
            for k, b in zip(keys, bufs):
                t = s[k]
                if t.numel() != p.numel():
                    raise ValueError(f"optimizer state {i}.{k}: {tuple(t.shape)} for a parameter of {tuple(p.shape)}")
                b[o:o + p.numel()].copy_(t.reshape(-1))
            if "step" in s:
                steps.add(int(float(s["step"])))
        if len(steps) > 1:
            raise ValueError(f"optimizer state: parameters at different step counts {sorted(steps)}")
        # torch's SGD keeps no step count: a momentum buffer means at least one step has been taken
        self.step_count = steps.pop() if steps else (1 if state else 0)
        self.lr = float(sd["param_groups"][0]["lr"])
