"""Training, the reference's train.py / training.py:13-47 (`train`) with what Lightning's `Trainer.fit` does for it,
and loader/data_loader.py:282-360 (`DSRandomSampler`, `DSElasticDistributedSampler`).

One step is the device path of `bench.py`: `training_step` -> `backward` with the gradients written straight into one
flat buffer -> the overlapped all-reduce of that buffer (more than one process) -> the fused clip + AdamW / SGD-Nesterov
step.  The loop does not wait for the GPU: the loss is summed on the device and read every `log_every_n_steps` steps
and at the epoch end, and the input pipeline is at most one batch ahead (`SpectrogramBatcher`).  Validation counts
stay on the device as in `run_evaluation`.  Without Lightning and Hydra, the process count comes from torchrun's
environment (`dist.init_from_env`)."""
import dataclasses
import itertools
import json
import math
import os
import random
import time
import warnings

import numpy as np
import torch
from torch.utils.data import Sampler
from torch.utils.data.distributed import DistributedSampler

from . import _lib, dist as D, ops
from .checkpoint import FileCheckpointHandler
from .configs import ModelCheckpointConf, TrainerConf
from .evaluation import AudioDataLoader, SpectrogramDataset, run_evaluation
from .model import DeepSpeech
from .optim import FlatParams, FusedOptimizer

__all__ = ["train", "seed_everything", "DSRandomSampler", "DSElasticDistributedSampler", "FileCheckpointHandler"]


# ---------------------------------------------------------------------------------------------- samplers
def _bins(n, batch_size):
    ids = list(range(n))
    return [ids[i:i + batch_size] for i in range(0, len(ids), batch_size)]


def _epoch_order(n_bins, epoch):
    g = torch.Generator()
    g.manual_seed(epoch)
    return torch.randperm(n_bins, generator=g).tolist()


class DSRandomSampler(Sampler):
    """data_loader.py:282-315, a batch sampler: consecutive dataset indices in bins of `batch_size` (the last one
    shorter), the bins in a permutation drawn from a torch.Generator seeded with the epoch, each bin shuffled in place
    with `np.random.shuffle` as it is yielded (so the shuffles accumulate over epochs)."""

    def __init__(self, dataset, batch_size=1):
        super().__init__()
        self.dataset, self.batch_size = dataset, batch_size
        self.start_index = 0
        self.epoch = 0
        self.bins = _bins(len(dataset), batch_size)

    def __iter__(self):
        for x in _epoch_order(len(self.bins) - self.start_index, self.epoch):
            batch_ids = self.bins[x + self.start_index]
            np.random.shuffle(batch_ids)
            yield batch_ids

    def __len__(self):
        return len(self.bins) - self.start_index

    def set_epoch(self, epoch):
        self.epoch = epoch


class DSElasticDistributedSampler(DistributedSampler):
    """data_loader.py:318-360: DSRandomSampler's bins and epoch permutation, padded with its own head to a multiple of
    the process count, then dealt `rank::num_replicas` (`dist.shard_bins`); `num_replicas` and `rank` default to the
    initialised process group's."""

    def __init__(self, dataset, num_replicas=None, rank=None, batch_size=1):
        super().__init__(dataset=dataset, num_replicas=num_replicas, rank=rank)
        self.start_index = 0
        self.batch_size = batch_size
        self.bins = _bins(len(dataset), batch_size)
        self.num_samples = int(math.ceil(float(len(self.bins) - self.start_index) / self.num_replicas))
        self.total_size = self.num_samples * self.num_replicas

    def __iter__(self):
        indices = [x + self.start_index for x in _epoch_order(len(self.bins) - self.start_index, self.epoch)]
        indices += indices[:(self.total_size - len(indices))]
        assert len(indices) == self.total_size
        indices = [indices[i] for i in D.shard_bins(self.total_size, self.rank, self.num_replicas)]
        assert len(indices) == self.num_samples
        for x in indices:
            batch_ids = self.bins[x]
            np.random.shuffle(batch_ids)
            yield batch_ids

    def __len__(self):
        return self.num_samples


# ---------------------------------------------------------------------------------------------- set-up
def seed_everything(seed):
    """pytorch_lightning.seed_everything: python `random`, numpy and torch (CPU and every CUDA device)"""
    seed = int(seed)
    os.environ["PL_GLOBAL_SEED"] = str(seed)
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    return seed


# Trainer fields train() acts on, and fields it has no use for (placement comes from torchrun, there is no logger,
# progress bar, model summary, sanity check or cudnn)
_TRAINER_HONOURED = {"max_epochs", "min_epochs", "precision", "gradient_clip_val", "check_val_every_n_epoch",
                     "limit_train_batches", "limit_val_batches", "log_every_n_steps", "enable_checkpointing",
                     "default_root_dir", "resume_from_checkpoint"}
_TRAINER_NOT_READ = {"_target_", "accelerator", "devices", "strategy", "num_nodes", "logger", "enable_progress_bar",
                     "enable_model_summary", "num_sanity_val_steps", "benchmark"}
_CHECKPOINT_REFUSED = ("filepath", "every_n_train_steps", "train_time_interval", "save_on_train_epoch_end")
_WHY = {"accumulate_grad_batches": "the backward writes every gradient in place (gradient sinks), nothing accumulates",
        "val_check_interval": "validation runs at epoch ends only",
        "sync_batchnorm": "BatchNorm statistics are per process; rank 0's are broadcast before validation",
        "every_n_train_steps": "checkpoints are written at epoch ends only",
        "train_time_interval": "checkpoints are written at epoch ends only"}


def _refuse(where, name, value):
    why = _WHY.get(name, "not implemented")
    raise _lib.Ds2Error(f"train: {where}.{name} = {value!r} is not supported ({why})")


def check_config(cfg):
    """raise Ds2Error naming the first setting `train` cannot honour"""
    tdef = TrainerConf()
    for f in dataclasses.fields(TrainerConf):
        if f.name in _TRAINER_HONOURED or f.name in _TRAINER_NOT_READ:
            continue
        v = getattr(cfg.trainer, f.name, getattr(tdef, f.name))
        if v != getattr(tdef, f.name) and not (f.name == "gradient_clip_algorithm" and v == "norm"):
            _refuse("trainer", f.name, v)
    t = cfg.trainer
    if t.precision not in (16, 32):
        _refuse("trainer", "precision", t.precision)
    if not (isinstance(t.max_epochs, int) and t.max_epochs >= 0):
        _refuse("trainer", "max_epochs", t.max_epochs)
    if not (isinstance(t.check_val_every_n_epoch, int) and t.check_val_every_n_epoch >= 1):
        _refuse("trainer", "check_val_every_n_epoch", t.check_val_every_n_epoch)
    if not (isinstance(t.log_every_n_steps, int) and t.log_every_n_steps >= 1):
        _refuse("trainer", "log_every_n_steps", t.log_every_n_steps)
    if float(t.gradient_clip_val or 0) < 0:
        _refuse("trainer", "gradient_clip_val", t.gradient_clip_val)
    for name in ("limit_train_batches", "limit_val_batches"):
        v = getattr(t, name)
        if isinstance(v, bool) or not isinstance(v, (int, float)) or v < 0 or (isinstance(v, float) and v > 1):
            _refuse("trainer", name, v)
    cdef = ModelCheckpointConf()
    for name in _CHECKPOINT_REFUSED:
        v = getattr(cfg.checkpoint, name, None)
        if v != getattr(cdef, name):
            _refuse("checkpoint", name, v)
    aug = cfg.data.augmentation
    if aug.noise_dir:
        raise _lib.Ds2Error("train: noise injection (data.augmentation.noise_dir) is not implemented on the GPU input "
                            "pipeline")
    if aug.speed_volume_perturb:
        raise _lib.Ds2Error("train: speed / volume perturbation (data.augmentation.speed_volume_perturb) is not "
                            "implemented on the GPU input pipeline")


def n_batches(limit, total, name):
    """Lightning's reading of limit_*_batches: an int is a count, a float a fraction (rounded down) of `total`"""
    if isinstance(limit, int) or limit == 0.0:
        return min(total, int(limit))
    n = int(total * limit)
    if n == 0 and total > 0:
        raise _lib.Ds2Error(f"train: trainer.{name} = {limit} of {total} batches is 0 batches; use 0 to skip them")
    return n


def scheduler_state(opt, n_anneals):
    """torch's ExponentialLR(gamma=learning_anneal).state_dict() after `n_anneals` epochs, at `opt.lr`"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sched = torch.optim.lr_scheduler.ExponentialLR(opt.torch_optimizer([torch.zeros(1)]),
                                                       gamma=float(opt.cfg.learning_anneal))
    sched.last_epoch, sched._step_count, sched._last_lr = n_anneals, n_anneals + 1, [opt.lr]
    return sched.state_dict()


# ---------------------------------------------------------------------------------------------- train
def _checkpoint(model, opt, handler, epoch, step, weights_only):
    ck = {"epoch": epoch, "global_step": step,
          "state_dict": model.state_dict(),
          "hyper_parameters": {"labels": model.labels, "model_cfg": model.model_cfg, "precision": model.precision,
                               "optim_cfg": model.optim_cfg, "spect_cfg": model.spect_cfg}}
    if not weights_only:
        ck["optimizer_states"] = [opt.state_dict()]
        ck["lr_schedulers"] = [scheduler_state(opt, epoch + 1)]
        ck["callbacks"] = {"FileCheckpointHandler": handler.state_dict()}
    return ck


def restore(path, model, opt, handler=None):
    """load a checkpoint `train` wrote into the run's model, FusedOptimizer and handler -> (first epoch to run,
    global step)"""
    ck = torch.load(str(path), map_location=opt.flat.data.device, weights_only=False)
    if "optimizer_states" not in ck:
        raise _lib.Ds2Error(f"train: {path} holds the weights only (checkpoint.save_weights_only); it cannot "
                            "resume a run")
    model.load_state_dict(ck["state_dict"], strict=True)
    opt.load_state_dict(ck["optimizer_states"][0])
    if handler is not None and "FileCheckpointHandler" in ck.get("callbacks", {}):
        handler.load_state_dict(ck["callbacks"]["FileCheckpointHandler"])
    return int(ck["epoch"]) + 1, int(ck["global_step"])


def train(cfg):
    """training.py:13-47 (cfg: DeepSpeechConfig) -> one record per epoch run: {'epoch', 'global_step', 'loss' (mean
    training loss of the epoch), 'wer', 'cer' (None in epochs without validation), 'checkpoint' (path written, or
    None), 'logged_loss' ([(global_step, loss)] every log_every_n_steps steps), 'train_s' and 'val_s' (host seconds of the
    epoch's steps and of its validation, each ending in a wait for the GPU)}; prints one line per epoch.

    Both the training and the validation set are `SpectrogramDataset(normalize=True, aug_cfg=data.augmentation)`:
    the reference augments the validation set too (data_module.py:56-64), and so does this.  Every process validates
    the whole validation set with rank 0's BatchNorm statistics; only rank 0 writes checkpoints.  A resumed run
    (`trainer.resume_from_checkpoint`, or the newest checkpoint with `load_auto_checkpoint`) restores the parameters,
    BatchNorm statistics, optimizer moments and step, learning rate, epoch and best-k bookkeeping, and continues at the
    next epoch."""
    check_config(cfg)
    t, ccfg = cfg.trainer, cfg.checkpoint
    rank, world, local = D.init_from_env()
    if not torch.cuda.is_available():
        raise _lib.Ds2Error("train: needs a CUDA device; there is no CPU path")
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    seed_everything(cfg.seed)
    with open(cfg.data.labels_path) as f:
        labels = json.load(f)

    handler = FileCheckpointHandler(ccfg, t.default_root_dir) if t.enable_checkpointing else None
    resume = t.resume_from_checkpoint
    if handler is not None and cfg.load_auto_checkpoint:
        resume = handler.find_latest_checkpoint() or resume

    def dataset(path):
        return SpectrogramDataset(audio_conf=cfg.data.spect, input_path=path, labels=labels, normalize=True,
                                  aug_cfg=cfg.data.augmentation)
    train_set, val_set = dataset(cfg.data.train_path), dataset(cfg.data.val_path)
    if world > 1:
        sampler = DSElasticDistributedSampler(train_set, num_replicas=world, rank=rank,
                                              batch_size=cfg.data.batch_size)
    else:
        sampler = DSRandomSampler(train_set, batch_size=cfg.data.batch_size)
    # file readers that live for the whole run: a new set each epoch costs a start-up per epoch
    keep = cfg.data.num_workers > 0
    train_loader = AudioDataLoader(train_set, num_workers=cfg.data.num_workers, batch_sampler=sampler,
                                   persistent_workers=keep)
    val_loader = AudioDataLoader(val_set, num_workers=cfg.data.num_workers, batch_size=cfg.data.batch_size,
                                 persistent_workers=keep)
    n_train = n_batches(t.limit_train_batches, len(train_loader), "limit_train_batches")
    n_val = n_batches(t.limit_val_batches, len(val_loader), "limit_val_batches")

    model = DeepSpeech(labels=labels, model_cfg=cfg.model, optim_cfg=cfg.optim, precision=t.precision,
                       spect_cfg=cfg.data.spect).to(dev).train()
    flat = FlatParams(model, direct_grads=True)
    opt = FusedOptimizer(flat, cfg.optim, max_norm=float(t.gradient_clip_val or 0))
    exchange = D.OverlappedGradAllReduce(flat, model)

    start_epoch, step = restore(resume, model, opt, handler) if resume else (0, 0)

    # as bench.py: the step on a high-priority stream, the recurrent weight-gradient GEMMs deferred to a side stream
    caller_stream = torch.cuda.current_stream(dev)
    main = torch.cuda.Stream(device=dev, priority=-1)
    main.wait_stream(caller_stream)
    records = []
    own_side = ops.side_stream() is None
    try:
        with torch.cuda.stream(main):
            if own_side:
                ops.enable_deferred_weight_grads(dev)
            for epoch in range(start_epoch, t.max_epochs):
                t0 = time.perf_counter()
                sampler.set_epoch(epoch)
                model.train()
                loss_sum = torch.zeros((), device=dev)
                logged = []
                n = 0
                for batch in itertools.islice(train_loader, n_train):
                    loss = model.training_step(batch, n)
                    loss.backward()
                    exchange.finish()
                    opt.step(grad_scale=1.0 / world)
                    loss_sum += loss.detach()
                    n += 1
                    step += 1
                    if step % t.log_every_n_steps == 0:
                        logged.append((step, float(loss.detach())))
                if world > 1:
                    torch.distributed.all_reduce(loss_sum)
                mean_loss = float(loss_sum) / max(1, n * world)     # waits for the epoch's last step
                train_s = time.perf_counter() - t0
                opt.anneal()

                wer = cer = None
                validate = n_val > 0 and (epoch + 1) % t.check_val_every_n_epoch == 0
                if validate:
                    D.broadcast_buffers(model)
                    wer, cer = run_evaluation(itertools.islice(val_loader, n_val), model, model.evaluation_decoder,
                                              dev, model.evaluation_decoder, t.precision)
                    model.train()
                val_s = time.perf_counter() - t0 - train_s
                path = None
                if handler is not None and (validate or n_val == 0):
                    if not validate:
                        D.broadcast_buffers(model)
                    if rank == 0:
                        metrics = {} if wer is None else {"wer": wer, "cer": cer}

                        def save(p):
                            os.makedirs(os.path.dirname(p), exist_ok=True)
                            torch.save(_checkpoint(model, opt, handler, epoch, step, handler.save_weights_only), p)
                        path = handler.on_epoch_end(epoch, step, metrics, save)
                print(f"Epoch {epoch}  step {step}  loss {mean_loss:.4f}" +
                      ("" if wer is None else f"  WER {wer:.3f}  CER {cer:.3f}"), flush=True)
                records.append({"epoch": epoch, "global_step": step, "loss": mean_loss, "wer": wer, "cer": cer,
                                "checkpoint": path, "logged_loss": logged, "train_s": train_s, "val_s": val_s})
    finally:
        if own_side:
            ops.enable_deferred_weight_grads(enable=False)
        caller_stream.wait_stream(main)
    return records
