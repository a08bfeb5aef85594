"""DeepSpeech shell: the reference's drop-in seam (deepspeech_pytorch/model.py:138-310) over the
CUDA C-ABI.

Same constructor, attributes, `forward(x, lengths, hs) -> (out, output_lengths, new_hs)` contract,
Lightning hooks (`training_step`, `validation_step`, `configure_optimizers`) and — because the
parameters live in the same torch container classes at the same attribute paths — the same
`state_dict` keys, shapes and RNG-identical default initialisation as the reference, so reference
checkpoints load unchanged.  None of the container modules' own `forward`s is ever called: every
block runs through `ops.py` -> libds2_b200.so; without the library / a CUDA tensor it raises.
"""
import math
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops
from .configs import cfg_type, is_kind
from .decoder import GreedyDecoder
from .metrics import CharErrorRate, WordErrorRate

try:  # Lightning is optional: with it installed the shell is a LightningModule like the reference
    import pytorch_lightning as pl
    _Base = pl.LightningModule
except Exception:  # pragma: no cover - lightning is not in this image
    pl = None
    _Base = nn.Module

BN_MOMENTUM, BN_EPS = 0.1, 1e-5


def _rnn_code(rnn_cls):
    return {nn.LSTM: _lib.RNN_LSTM, nn.GRU: _lib.RNN_GRU, nn.RNN: _lib.RNN_TANH}[rnn_cls]


class _Holder(nn.Module):
    """parameter container; `.module` / `.seq_module` attribute names give the reference's keys"""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container of the CUDA shell: not callable")


class _MaskConvParams(_Holder):      # keys conv.seq_module.{0,1,3,4}.*  (model.py:157-164)
    def __init__(self):
        super().__init__()
        self.seq_module = nn.Sequential(
            nn.Conv2d(1, 32, kernel_size=(41, 11), stride=(2, 2), padding=(20, 5)), nn.BatchNorm2d(32),
            nn.Hardtanh(0, 20, inplace=True),
            nn.Conv2d(32, 32, kernel_size=(21, 11), stride=(2, 1), padding=(10, 5)), nn.BatchNorm2d(32),
            nn.Hardtanh(0, 20, inplace=True))


class _SequenceWiseParams(_Holder):  # keys *.module.*  (model.py:18-33)
    def __init__(self, module):
        super().__init__()
        self.module = module


class _BatchRNNParams(_Holder):      # keys rnns.i.{batch_norm.module,rnn}.*  (model.py:80-102)
    def __init__(self, input_size, hidden_size, rnn_cls, bidirectional, batch_norm):
        super().__init__()
        self.input_size, self.hidden_size, self.bidirectional = input_size, hidden_size, bidirectional
        self.batch_norm = _SequenceWiseParams(nn.BatchNorm1d(input_size)) if batch_norm else None
        self.rnn = rnn_cls(input_size=input_size, hidden_size=hidden_size, bidirectional=bidirectional, bias=True)
        self.rnn_code = _rnn_code(rnn_cls)

    def weights(self):
        names = ["weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"]
        out = [getattr(self.rnn, n) for n in names]
        if self.bidirectional:
            out += [getattr(self.rnn, n + "_reverse") for n in names]
        return out


class _LookaheadParams(_Holder):     # key lookahead.0.conv.weight  (model.py:105-123)
    def __init__(self, n_features, context):
        super().__init__()
        assert context > 0
        self.context, self.n_features = context, n_features
        self.conv = nn.Conv1d(n_features, n_features, kernel_size=context, stride=1, groups=n_features, padding=0,
                              bias=False)


class DeepSpeech(_Base):
    def __init__(self, labels: List, model_cfg, precision: int, optim_cfg, spect_cfg):
        super().__init__()
        if hasattr(self, "save_hyperparameters") and pl is not None:
            self.save_hyperparameters()
        self.model_cfg, self.precision, self.optim_cfg, self.spect_cfg = model_cfg, precision, optim_cfg, spect_cfg
        # model.py:152 — flavour is chosen by the *type* of the config
        self.bidirectional = not is_kind(model_cfg, "UniDirectionalConfig")
        self.labels = labels
        num_classes = len(labels)
        rnn_cls = model_cfg.rnn_type.value if hasattr(model_cfg.rnn_type, "value") else model_cfg.rnn_type

        self.conv = _MaskConvParams()
        freq = int(math.floor((spect_cfg.sample_rate * spect_cfg.window_size) / 2) + 1)
        if freq != 161:
            raise _lib.Ds2Error(f"the front-end kernels are built for 161 frequency bins, got {freq}")
        rnn_input_size = 32 * 41
        H = model_cfg.hidden_size
        self.rnns = nn.Sequential(
            _BatchRNNParams(rnn_input_size, H, rnn_cls, self.bidirectional, batch_norm=False),
            *(_BatchRNNParams(H, H, rnn_cls, self.bidirectional, batch_norm=True)
              for _ in range(model_cfg.hidden_layers - 1)))
        self.lookahead = nn.Sequential(_LookaheadParams(H, context=model_cfg.lookahead_context),
                                       nn.Hardtanh(0, 20, inplace=True)) if not self.bidirectional else None
        self.fc = nn.Sequential(_SequenceWiseParams(nn.Sequential(nn.BatchNorm1d(H),
                                                                   nn.Linear(H, num_classes, bias=False))))
        self.blank = self.labels.index('_')
        self.evaluation_decoder = GreedyDecoder(self.labels)  # Decoder used for validation (model.py:204)
        self.wer = WordErrorRate(decoder=self.evaluation_decoder, target_decoder=self.evaluation_decoder)
        self.cer = CharErrorRate(decoder=self.evaluation_decoder, target_decoder=self.evaluation_decoder)
        self.criterion = self._ctc_criterion

    # ------------------------------------------------------------------ lengths (model.py:299-310)
    def get_seq_lens(self, input_length):
        lens = np.ascontiguousarray(torch.as_tensor(input_length).cpu().numpy().astype(np.int32))
        out = np.empty_like(lens)
        _lib.check(_lib.get_lib().ds2_seq_lens_host(lens.ctypes.data, lens.size, out.ctypes.data), "ds2_seq_lens_host")
        return torch.from_numpy(out).int()

    # ------------------------------------------------------------------ forward (model.py:214-239)
    def forward(self, x, lengths, hs: Optional[list] = None):
        """model.py:214-239.  `precision == 16` (the reference wraps this call in autocast, model.py:255 /
        inference.py:94, and Lightning does so for training) selects the library's precision-16 mode for the duration
        of the call; the autograd nodes remember it for their backward.  Any other value leaves the process-wide
        switch (`set_precision`) alone."""
        if not x.is_cuda:
            raise _lib.Ds2Error("DeepSpeech (CUDA shell): input must be a CUDA tensor; there is no CPU path")
        if self.precision == 16:
            lib = _lib.get_lib()
            saved = lib.ds2_get_precision()
            if saved != _lib.PREC_F16:
                lib.ds2_set_precision(_lib.PREC_F16)
                try:
                    return self._forward(x, lengths, hs)
                finally:
                    lib.ds2_set_precision(saved)
        return self._forward(x, lengths, hs)

    def _forward(self, x, lengths, hs: Optional[list] = None):
        lengths = torch.as_tensor(lengths).cpu().int()
        output_lengths = self.get_seq_lens(lengths)
        ol = output_lengths.tolist()
        if any(l <= 0 for l in ol):
            raise RuntimeError("Length of all samples has to be greater than 0, but found an element in "
                               "'lengths' that is <= 0")                       # pack_padded_sequence's check
        if any(ol[i] < ol[i + 1] for i in range(len(ol) - 1)):
            raise RuntimeError("`lengths` array must be sorted in decreasing order when `enforce_sorted` is True.")
        dev = x.device
        len_dev = output_lengths.to(dev, non_blocking=True)
        training = self.training
        sm = self.conv.seq_module
        y = ops.ConvFrontend.apply(x.float(), len_dev, sm[0].weight, sm[0].bias, sm[1].weight, sm[1].bias,
                                   sm[1].running_mean, sm[1].running_var, sm[3].weight, sm[3].bias, sm[4].weight,
                                   sm[4].bias, sm[4].running_mean, sm[4].running_var, training, BN_MOMENTUM, BN_EPS)
        if training:
            sm[1].num_batches_tracked += 1
            sm[4].num_batches_tracked += 1
            hook = getattr(self, "front_end_grad_hook", None)
            if hook is not None and y.requires_grad:
                # fires when autograd reaches the front-end, i.e. when every other gradient is final
                # (dist.OverlappedGradAllReduce starts the exchange of those gradients here)
                y.register_hook(lambda g, _h=hook: _h())
        t_out = min(int(max(ol)), y.shape[0])
        y = y[:t_out]                                                           # pad_packed_sequence truncation
        if hs is None:
            hs = [None] * len(self.rnns)
        new_hs = []
        # dist.OverlappedGradAllReduce (gradient sinks on): the gradient of a block's INPUT exists only once the block's
        # backward has run, i.e. once its parameter gradients are final in the flat buffer -> exchange them right away
        bhook = getattr(self, "block_grad_hook", None) if training else None

        def _mark(t, name):
            if bhook is not None and t.requires_grad:
                t.register_hook(lambda g, _n=name: bhook(_n))
        for i, layer in enumerate(self.rnns):
            _mark(y, f"rnn{i}")
            h0 = c0 = None
            if hs[i] is not None:
                if layer.rnn_code == _lib.RNN_LSTM:
                    h0, c0 = hs[i]
                else:
                    h0 = hs[i]
            bn = layer.batch_norm.module if layer.batch_norm is not None else None
            y, hn, cn = ops.RnnLayer.apply(y, len_dev, layer.rnn_code, self.bidirectional, training, BN_MOMENTUM,
                                           BN_EPS, bn.weight if bn else None, bn.bias if bn else None,
                                           bn.running_mean if bn else None, bn.running_var if bn else None, h0, c0,
                                           *layer.weights())
            if bn is not None and training:
                bn.num_batches_tracked += 1
            new_hs.append((hn, cn) if layer.rnn_code == _lib.RNN_LSTM else hn)
        _mark(y, "head")
        if not self.bidirectional:
            y = ops.Lookahead.apply(y, self.lookahead[0].conv.weight)
        fbn, flin = self.fc[0].module[0], self.fc[0].module[1]
        logits = ops.FcHead.apply(y, fbn.weight, fbn.bias, fbn.running_mean, fbn.running_var, flin.weight, training,
                                  BN_MOMENTUM, BN_EPS, not training)            # eval: softmax (model.py:72-77)
        if training:
            fbn.num_batches_tracked += 1
        return logits.transpose(0, 1), output_lengths, new_hs

    # ------------------------------------------------------------------ loss (model.py:203,241-249)
    def _ctc_criterion(self, logits_tbc, targets, input_sizes, target_sizes):
        """CTCLoss(blank, reduction='sum', zero_infinity=True) applied to *logits* (T,B,C): the
        log-softmax of model.py:246 is fused into the kernel."""
        dev = logits_tbc.device
        target_sizes = torch.as_tensor(target_sizes).int()
        max_l = int(target_sizes.max()) if target_sizes.numel() else 0
        return ops.CtcLoss.apply(logits_tbc.contiguous(), targets.to(dev, non_blocking=True).long(),
                                 torch.as_tensor(input_sizes).int().to(dev, non_blocking=True),
                                 target_sizes.to(dev, non_blocking=True), max_l, self.blank)

    def training_step(self, batch, batch_idx):
        inputs, targets, input_percentages, target_sizes = batch
        input_sizes = input_percentages.mul_(int(inputs.size(3))).int()          # in place, like model.py:243
        out, output_sizes, _ = self(inputs, input_sizes)
        return self.criterion(out.transpose(0, 1), targets, output_sizes, target_sizes)

    def validation_step(self, batch, batch_idx):
        inputs, targets, input_percentages, target_sizes = batch
        input_sizes = input_percentages.mul_(int(inputs.size(3))).int()
        out, output_sizes, _ = self(inputs.to(next(self.parameters()).device), input_sizes)
        decoded_output, _ = self.evaluation_decoder.decode(out, output_sizes)
        self.wer(preds=out, preds_sizes=output_sizes, targets=targets, target_sizes=target_sizes)   # model.py:258-269
        self.cer(preds=out, preds_sizes=output_sizes, targets=targets, target_sizes=target_sizes)
        if pl is not None:
            self.log('wer', self.wer.compute(), prog_bar=True, on_epoch=True)
            self.log('cer', self.cer.compute(), prog_bar=True, on_epoch=True)
        return decoded_output

    # ------------------------------------------------------------------ optim (model.py:273-297)
    def configure_optimizers(self):
        if is_kind(self.optim_cfg, "SGDConfig"):
            optimizer = torch.optim.SGD(params=self.parameters(), lr=self.optim_cfg.learning_rate,
                                        momentum=self.optim_cfg.momentum, nesterov=True,
                                        weight_decay=self.optim_cfg.weight_decay)
        elif is_kind(self.optim_cfg, "AdamConfig"):
            optimizer = torch.optim.AdamW(params=self.parameters(), lr=self.optim_cfg.learning_rate,
                                          betas=self.optim_cfg.betas, eps=self.optim_cfg.eps,
                                          weight_decay=self.optim_cfg.weight_decay)
        else:
            raise ValueError("Optimizer has not been specified correctly.")
        scheduler = torch.optim.lr_scheduler.ExponentialLR(optimizer=optimizer, gamma=self.optim_cfg.learning_anneal)
        return [optimizer], [scheduler]
