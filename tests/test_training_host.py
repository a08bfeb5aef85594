"""CPU: the training configs, samplers, checkpoint bookkeeping, optimizer state and refused settings of `train`.

The configs' defaults and the samplers' bin orders are compared with tests/golden/training/reference_training.json,
written by tools/make_training_golden.py from the reference's own configs/lightning_config.py, configs/train_config.py
and loader/data_loader.py."""
import dataclasses
import json
import os
import time

import numpy as np
import pytest
import torch

import deepspeech_pytorch_b200 as ds
from conftest import GOLDEN_DIR
from deepspeech_pytorch_b200.optim import FlatParams, FusedOptimizer
from deepspeech_pytorch_b200.training import check_config, n_batches, scheduler_state

GOLDEN = json.load(open(os.path.join(GOLDEN_DIR, "training", "reference_training.json")))


def _defaults(obj):
    out = {}
    for f in dataclasses.fields(obj):
        v = getattr(obj, f.name)
        out[f.name] = list(v) if isinstance(v, tuple) else v
    return out


def test_config_fields_and_defaults_are_the_references():
    assert _defaults(ds.TrainerConf()) == GOLDEN["TrainerConf"]
    assert _defaults(ds.ModelCheckpointConf()) == GOLDEN["ModelCheckpointConf"]
    cfg = ds.DeepSpeechConfig()
    for k, v in GOLDEN["DeepSpeechConfig"].items():
        assert getattr(cfg, k) == v
    assert type(cfg.model) is ds.BiDirectionalConfig and type(cfg.optim) is ds.AdamConfig
    assert type(cfg.checkpoint) is ds.ModelCheckpointConf and type(cfg.data) is ds.DataConfig
    assert type(cfg.augmentation) is ds.AugmentationConfig
    assert ds.DeepSpeechConfig().trainer is not cfg.trainer          # no shared mutable defaults


@pytest.mark.parametrize("case", range(len(GOLDEN["samplers"])))
def test_samplers_give_the_references_bin_orders(case):
    g = GOLDEN["samplers"][case]
    data = list(range(g["n"]))
    np.random.seed(GOLDEN["np_seed"])
    if g["world"] == 1:
        samplers = [ds.DSRandomSampler(data, batch_size=g["batch_size"])]
    else:
        samplers = [ds.DSElasticDistributedSampler(data, num_replicas=g["world"], rank=r, batch_size=g["batch_size"])
                    for r in range(g["world"])]
    for epoch, want in zip(g["epochs"], g["orders"]):
        got = []
        for s in samplers:
            s.set_epoch(epoch)
            got.append([list(map(int, b)) for b in s])
            assert len(s) == len(got[-1])
        assert got == want, (g["n"], g["batch_size"], g["world"], epoch)


def test_elastic_sampler_deals_the_bins_as_shard_bins():
    from deepspeech_pytorch_b200.dist import shard_bins
    s = ds.DSElasticDistributedSampler(list(range(9)), num_replicas=2, rank=1, batch_size=2)   # 5 bins, 1 padded
    assert len(s) == 3 and s.total_size == 6
    assert shard_bins(6, 1, 2) == [1, 3, 5]


# ---------------------------------------------------------------------------------------------- checkpoints
class _Writer:
    def __init__(self):
        self.saved = []

    def __call__(self, path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(path)
        self.saved.append(os.path.basename(path))


def _handler(tmp_path, **kw):
    return ds.FileCheckpointHandler(ds.ModelCheckpointConf(dirpath=str(tmp_path / "ck"), **kw))


def _files(tmp_path):
    d = tmp_path / "ck"
    return sorted(os.listdir(d)) if d.is_dir() else []


@pytest.mark.parametrize("mode", ["min", "max"])
def test_top_k_keeps_the_best(tmp_path, mode):
    h, w = _handler(tmp_path, monitor="wer", mode=mode, save_top_k=2), _Writer()
    wers = [50.0, 40.0, 45.0, 60.0, 30.0]
    for e, x in enumerate(wers):
        h.on_epoch_end(e, 10 * (e + 1), {"wer": x, "cer": x / 2}, w)
    order = sorted(range(len(wers)), key=lambda i: wers[i], reverse=(mode == "max"))
    keep = sorted(f"epoch={e}-step={10 * (e + 1)}.ckpt" for e in order[:2])
    assert _files(tmp_path) == keep
    best = order[0]
    assert os.path.basename(h.best_model_path) == f"epoch={best}-step={10 * (best + 1)}.ckpt"
    assert h.best_model_score == wers[best]
    # a value no better than the k-th is not written
    n = len(w.saved)
    h.on_epoch_end(9, 100, {"wer": h.kth_value, "cer": 0.0}, w)
    assert len(w.saved) == n


def test_no_monitor_keeps_the_newest_or_all(tmp_path):
    h, w = _handler(tmp_path), _Writer()
    for e in range(3):
        h.on_epoch_end(e, e + 1, {}, w)
    assert _files(tmp_path) == ["epoch=2-step=3.ckpt"]
    h2 = ds.FileCheckpointHandler(ds.ModelCheckpointConf(dirpath=str(tmp_path / "all"), save_top_k=-1))
    for e in range(3):
        h2.on_epoch_end(e, e + 1, {}, w)
    assert sorted(os.listdir(tmp_path / "all")) == [f"epoch={e}-step={e + 1}.ckpt" for e in range(3)]
    with pytest.raises(ds.Ds2Error, match="save_top_k"):
        ds.FileCheckpointHandler(ds.ModelCheckpointConf(save_top_k=3))


def test_save_last_every_n_epochs_and_top_k_zero(tmp_path):
    h, w = _handler(tmp_path, save_last=True, save_top_k=0, every_n_epochs=2), _Writer()
    for e in range(5):
        h.on_epoch_end(e, e + 1, {"wer": 1.0, "cer": 1.0}, w)
    assert _files(tmp_path) == ["last.ckpt"] and w.saved == ["last.ckpt"] * 2     # epochs 1 and 3


def test_filename_templates(tmp_path):
    m = {"epoch": 3, "step": 120, "wer": 12.3456, "cer": 4.5}
    h = _handler(tmp_path, filename="{epoch:02d}-{wer:.2f}")
    assert os.path.basename(h.format_checkpoint_name(m)) == "epoch=03-wer=12.35.ckpt"
    h = _handler(tmp_path, filename="ds2-{epoch}-{step}-{cer:.1f}", auto_insert_metric_name=False)
    assert os.path.basename(h.format_checkpoint_name(m)) == "ds2-3-120-4.5.ckpt"
    h = _handler(tmp_path, filename="{missing}")
    assert os.path.basename(h.format_checkpoint_name(m)) == "missing=0.ckpt"
    h, w = _handler(tmp_path, filename="fixed", save_top_k=-1), _Writer()
    for e in range(3):
        h.on_epoch_end(e, e, {}, w)
    assert _files(tmp_path) == ["fixed-v1.ckpt", "fixed-v2.ckpt", "fixed.ckpt"]


def test_default_dirpath_and_find_latest(tmp_path):
    (tmp_path / "lightning_logs" / "version_3").mkdir(parents=True)
    h = ds.FileCheckpointHandler(ds.ModelCheckpointConf(), default_root_dir=str(tmp_path))
    assert h.find_latest_checkpoint() is None
    assert h.resolve_dirpath() == str(tmp_path / "lightning_logs" / "version_4" / "checkpoints")
    w = _Writer()
    h2 = _handler(tmp_path, save_top_k=-1)
    for e in range(3):
        h2.on_epoch_end(e, e, {}, w)
        time.sleep(0.02)
    assert os.path.basename(h2.find_latest_checkpoint()) == "epoch=2-step=2.ckpt"
    with open(tmp_path / "ck" / "epoch=1-step=1.ckpt", "a") as f:   # a write moves ctime
        f.write("x")
    assert os.path.basename(h2.find_latest_checkpoint()) == "epoch=1-step=1.ckpt"


def test_handler_state_round_trips(tmp_path):
    h, w = _handler(tmp_path, monitor="cer", save_top_k=2), _Writer()
    for e, x in enumerate([3.0, 2.0, 4.0]):
        h.on_epoch_end(e, e, {"wer": 0.0, "cer": x}, w)
    h2 = _handler(tmp_path, monitor="cer", save_top_k=2)
    h2.load_state_dict(h.state_dict())
    assert h2.state_dict() == h.state_dict()
    h2.on_epoch_end(3, 3, {"wer": 0.0, "cer": 1.0}, w)
    assert _files(tmp_path) == ["epoch=1-step=1.ckpt", "epoch=3-step=3.ckpt"]


# ---------------------------------------------------------------------------------------------- optimizer state
class _Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(5, 3)
        self.b = torch.nn.Conv1d(3, 3, 2)


@pytest.mark.parametrize("adam", [True, False])
def test_fused_optimizer_state_round_trips(adam):
    torch.manual_seed(0)
    model = _Tiny()
    cfg = ds.AdamConfig(learning_rate=1e-3) if adam else ds.SGDConfig(learning_rate=1e-3)
    opt = FusedOptimizer(FlatParams(model), cfg)
    assert opt.state_dict()["state"] == {}
    for p, o in zip(opt.flat.params, opt.flat.offsets):     # the padding between parameters stays 0
        opt.m[o:o + p.numel()].normal_()
        if adam:
            opt.v[o:o + p.numel()].uniform_()
    opt.step_count, opt.lr = 7, 1e-3 * 0.99 ** 2
    sd = opt.state_dict()
    names = ["exp_avg", "exp_avg_sq"] if adam else ["momentum_buffer"]
    params = list(model.parameters())
    assert sorted(sd["state"]) == list(range(len(params)))
    for i, p in enumerate(params):
        for k in names:
            t = sd["state"][i][k]
            assert t.shape == p.shape
            assert t.untyped_storage().data_ptr() == (opt.m if k != "exp_avg_sq" else opt.v).untyped_storage().data_ptr()
        assert float(sd["state"][i]["step"]) == 7
    assert sd["param_groups"][0]["params"] == list(range(len(params)))
    assert sd["param_groups"][0]["lr"] == opt.lr and sd["param_groups"][0]["initial_lr"] == 1e-3
    # torch's own optimizer accepts it, and gives back the same state
    ref = torch.optim.AdamW(model.parameters()) if adam else torch.optim.SGD(model.parameters(), lr=1, momentum=0.9)
    ref.load_state_dict(sd)
    opt2 = FusedOptimizer(FlatParams(_Tiny()), cfg)
    opt2.load_state_dict(ref.state_dict())
    assert torch.equal(opt2.m, opt.m) and opt2.step_count == 7 and opt2.lr == opt.lr
    if adam:
        assert torch.equal(opt2.v, opt.v)
    with pytest.raises(ValueError):
        FusedOptimizer(FlatParams(torch.nn.Linear(2, 2)), cfg).load_state_dict(sd)


def test_scheduler_state_is_torchs_exponential_lr():
    opt = FusedOptimizer(FlatParams(_Tiny()), ds.AdamConfig(learning_rate=2e-3, learning_anneal=0.9))
    for _ in range(3):
        opt.anneal()
    tor = torch.optim.AdamW(_Tiny().parameters(), lr=2e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(tor, gamma=0.9)
    for _ in range(3):
        tor.step()
        sched.step()
    got = scheduler_state(opt, 3)
    want = sched.state_dict()
    assert got.keys() == want.keys()
    assert got["last_epoch"] == want["last_epoch"] == 3 and got["base_lrs"] == want["base_lrs"]
    assert got["_last_lr"][0] == pytest.approx(want["_last_lr"][0], rel=1e-15)


# ---------------------------------------------------------------------------------------------- refused settings
REFUSED = [("trainer", "accumulate_grad_batches", 2), ("trainer", "val_check_interval", 0.5),
           ("trainer", "fast_dev_run", True), ("trainer", "overfit_batches", 0.1), ("trainer", "sync_batchnorm", True),
           ("trainer", "precision", "bf16"), ("trainer", "max_time", "00:01:00:00"), ("trainer", "gpus", 2),
           ("trainer", "limit_train_batches", 1.5), ("trainer", "deterministic", True),
           ("trainer", "reload_dataloaders_every_n_epochs", 1), ("trainer", "max_epochs", -1),
           ("checkpoint", "every_n_train_steps", 100), ("checkpoint", "train_time_interval", "1h"),
           ("checkpoint", "save_on_train_epoch_end", True), ("checkpoint", "filepath", "x.ckpt")]


@pytest.mark.parametrize("where,name,value", REFUSED)
def test_unsupported_fields_raise_naming_the_field(where, name, value):
    cfg = ds.DeepSpeechConfig()
    setattr(getattr(cfg, where), name, value)
    with pytest.raises(ds.Ds2Error, match=f"{where}.{name}"):
        ds.train(cfg)


@pytest.mark.parametrize("name", ["noise_dir", "speed_volume_perturb"])
def test_augmentations_without_a_gpu_path_raise_before_anything_runs(name):
    cfg = ds.DeepSpeechConfig()
    setattr(cfg.data.augmentation, name, "/noise" if name == "noise_dir" else True)
    with pytest.raises(ds.Ds2Error, match=f"data.augmentation.{name}"):
        ds.train(cfg)


def test_fields_that_are_not_read_are_accepted():
    cfg = ds.DeepSpeechConfig()
    cfg.trainer.accelerator, cfg.trainer.devices, cfg.trainer.strategy = "auto", 1, "ddp"
    cfg.trainer.logger, cfg.trainer.enable_progress_bar, cfg.trainer.num_sanity_val_steps = False, False, 0
    cfg.trainer.precision, cfg.trainer.gradient_clip_val, cfg.trainer.limit_val_batches = 16, 400, 3
    cfg.checkpoint.monitor, cfg.checkpoint.verbose, cfg.checkpoint.save_top_k = "wer", True, 1
    check_config(cfg)


def test_limit_batches_reads_as_lightning():
    assert n_batches(1.0, 10, "x") == 10 and n_batches(0.25, 10, "x") == 2
    assert n_batches(3, 10, "x") == 3 and n_batches(30, 10, "x") == 10 and n_batches(0, 10, "x") == 0
    assert n_batches(1, 10, "x") == 1
    with pytest.raises(ds.Ds2Error, match="limit_train_batches"):
        n_batches(0.05, 10, "limit_train_batches")
