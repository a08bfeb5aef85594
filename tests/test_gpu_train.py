"""-m gpu: `train` end to end on a seeded toy WAV set, against a hand-written loop over the same parts, `evaluate`,
torch's optimizers and a straight run; the input pipeline's staging buffers under a host that runs ahead."""
import json
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

import deepspeech_pytorch_b200 as ds
from deepspeech_pytorch_b200.evaluation import SpectrogramDataset
from deepspeech_pytorch_b200.input_pipeline import SpectrogramBatcher
from deepspeech_pytorch_b200.optim import FlatParams, FusedOptimizer
from deepspeech_pytorch_b200.training import restore
from gpu_helpers import rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 16000
WORDS = ["ABE", "BAD", "CAB", "DEED", "ACE", "BEAD", "DAB", "ECE"]
BATCH = 4
# Two runs of the same steps differ only where the kernels reduce with float atomics (BatchNorm / bias gradient sums,
# the clip norm), a few ulps per step.  Over the toy runs' 8 steps the whole parameter vector stays within this relative
# L2 distance (single near-zero tensors such as a BatchNorm bias can differ by more, relative to their own norm).
TOL = 1e-4


def params_rel_l2(got, want):
    keys = [k for k, v in want.items() if v.is_floating_point()]
    return rel_l2(torch.cat([got[k].reshape(-1) for k in keys]), torch.cat([want[k].reshape(-1) for k in keys]))


def _write_set(root, name, n, rng, lo, hi):
    samples = []
    lens = rng.choice(np.arange(int(lo * SR), int(hi * SR), 160), n, replace=False)   # distinct frame counts
    for k, m in enumerate(lens):
        t = np.arange(m) / SR
        y = 0.3 * np.sin(2 * np.pi * (180 + 35 * k) * t) + 0.05 * rng.standard_normal(m)
        wavfile.write(str(root / f"{name}{k}.wav"), SR, np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16))
        (root / f"{name}{k}.txt").write_text(' '.join(rng.choice(WORDS, int(rng.integers(1, 4))).tolist()))
        samples.append({"wav_path": f"{name}{k}.wav", "transcript_path": f"{name}{k}.txt"})
    man = root / f"{name}.json"
    man.write_text(json.dumps({"root_path": str(root), "samples": samples}))
    return str(man)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    """13 training utterances (bins of 4, 4, 4, 1) and 6 validation utterances, 0.4 - 1.2 s, and the labels"""
    root = tmp_path_factory.mktemp("train")
    rng = np.random.default_rng(11)
    labels = root / "labels.json"
    labels.write_text(json.dumps(list(ds.LABELS)))
    return {"train": _write_set(root, "tr", 13, rng, 0.4, 1.2), "val": _write_set(root, "va", 6, rng, 0.4, 1.2),
            "labels": str(labels)}


def _cfg(data, out, rnn="gru", optim=None, epochs=2, precision=32, **ck):
    cfg = ds.DeepSpeechConfig(optim=optim or ds.SGDConfig(learning_rate=3e-4, learning_anneal=0.9),
                              model=ds.BiDirectionalConfig(rnn_type=getattr(ds.RNNType, rnn), hidden_size=32,
                                                           hidden_layers=2), seed=7)
    cfg.data = ds.DataConfig(train_path=data["train"], val_path=data["val"], batch_size=BATCH, num_workers=0,
                             labels_path=data["labels"])
    cfg.trainer.max_epochs, cfg.trainer.precision, cfg.trainer.gradient_clip_val = epochs, precision, 400
    cfg.checkpoint.dirpath = str(out)
    for k, v in ck.items():
        setattr(cfg.checkpoint, k, v)
    return cfg


def _hand_loop(data, cfg):
    """the loop `train` runs, written out: DSRandomSampler's bins, the batcher, FlatParams / FusedOptimizer / anneal"""
    ds.seed_everything(cfg.seed)
    dev = torch.device("cuda")
    model = ds.DeepSpeech(list(ds.LABELS), cfg.model, cfg.trainer.precision, cfg.optim, cfg.data.spect).to(dev).train()
    flat = FlatParams(model, direct_grads=True)
    opt = FusedOptimizer(flat, cfg.optim, max_norm=cfg.trainer.gradient_clip_val)
    dataset = SpectrogramDataset(cfg.data.spect, cfg.data.train_path, list(ds.LABELS), normalize=True,
                                 aug_cfg=cfg.data.augmentation)
    sampler = ds.DSRandomSampler(dataset, batch_size=BATCH)
    batcher = SpectrogramBatcher(cfg.data.spect, normalize=True, augmentation_conf=cfg.data.augmentation)
    losses = []
    for epoch in range(cfg.trainer.max_epochs):
        sampler.set_epoch(epoch)
        model.train()
        ep = []
        for i, ids in enumerate(sampler):
            items = [dataset[j] for j in ids]
            loss = model.training_step(batcher([w for w, _ in items], [t for _, t in items]), i)
            loss.backward()
            opt.step()
            ep.append(float(loss.detach()))
        losses.append(sum(ep) / len(ep))
        opt.anneal()
    return losses, model, opt


def _ckpt(path):
    return torch.load(path, map_location="cuda", weights_only=False)


@pytest.fixture(scope="module")
def sgd_run(data, tmp_path_factory):
    out = tmp_path_factory.mktemp("sgd")
    cfg = _cfg(data, out, save_top_k=-1)
    return cfg, ds.train(cfg), out


def test_train_equals_the_hand_loop(data, sgd_run):
    cfg, recs, _ = sgd_run
    assert [r["epoch"] for r in recs] == [0, 1] and [r["global_step"] for r in recs] == [4, 8]
    losses, model, _ = _hand_loop(data, cfg)
    for r, want in zip(recs, losses):
        assert abs(r["loss"] - want) <= TOL * abs(want), (r["loss"], want)
    assert params_rel_l2(_ckpt(recs[-1]["checkpoint"])["state_dict"], model.state_dict()) <= TOL


def test_validation_equals_evaluate(data, sgd_run):
    _, recs, _ = sgd_run
    for r in recs:
        cfg = ds.EvalConfig(test_path=data["val"], batch_size=BATCH, num_workers=0)
        cfg.model.model_path = r["checkpoint"]
        assert ds.evaluate(cfg) == (r["wer"], r["cer"])


@pytest.mark.parametrize("adam", [False, True])
def test_checkpoint_loads_into_load_model_and_torch(data, sgd_run, tmp_path, adam):
    if adam:
        cfg = _cfg(data, tmp_path, optim=ds.AdamConfig(learning_rate=1e-3, learning_anneal=0.9), epochs=1)
        path = ds.train(cfg)[-1]["checkpoint"]
    else:
        cfg, recs, _ = sgd_run
        path = recs[-1]["checkpoint"]
    ck = _ckpt(path)
    assert sorted(ck) == ["callbacks", "epoch", "global_step", "hyper_parameters", "lr_schedulers",
                          "optimizer_states", "state_dict"]
    model = ds.load_model(torch.device("cuda"), path).train()      # strict
    tmodel = ds.load_model(torch.device("cuda"), path).train()
    topt = tmodel.configure_optimizers()[0][0]
    assert type(topt) is (torch.optim.AdamW if adam else torch.optim.SGD)
    topt.load_state_dict(ck["optimizer_states"][0])
    sched = torch.optim.lr_scheduler.ExponentialLR(topt, gamma=cfg.optim.learning_anneal)
    sched.load_state_dict(ck["lr_schedulers"][0])
    flat = FlatParams(model)
    fopt = FusedOptimizer(flat, cfg.optim, max_norm=0.0)
    fopt.load_state_dict(ck["optimizer_states"][0])
    assert sched.get_last_lr()[0] == fopt.lr == topt.param_groups[0]["lr"]
    # one step from the checkpoint on the same gradients: torch's optimizer against the fused kernel
    g = torch.Generator(device="cuda").manual_seed(3)
    for p, tp in zip(model.parameters(), tmodel.parameters()):
        p.grad.copy_(torch.randn(p.shape, device="cuda", generator=g) * 1e-2)
        tp.grad = p.grad.clone()
    topt.step()
    fopt.step()
    # fp32: an AdamW update is ~lr per element, so on a parameter of ~3e-3 (a BatchNorm bias) its last-bit
    # differences weigh ~1e-6 of the tensor
    for (k, p), tp in zip(model.named_parameters(), tmodel.parameters()):
        assert rel_l2(p, tp) <= 1e-5, k
    sched.step()
    fopt.anneal()
    assert sched.get_last_lr()[0] == pytest.approx(fopt.lr, rel=1e-15)


def test_resume_continues_the_run(data, sgd_run, tmp_path):
    cfg, straight, out = sgd_run
    first = ds.train(_cfg(data, tmp_path, epochs=1, save_top_k=-1))
    # what a resumed run restores right after loading is the saved state, bit for bit
    ck = _ckpt(first[-1]["checkpoint"])
    c2 = _cfg(data, tmp_path, epochs=2, save_top_k=-1)
    model = ds.DeepSpeech(list(ds.LABELS), c2.model, 32, c2.optim, c2.data.spect).cuda().train()
    opt = FusedOptimizer(FlatParams(model, direct_grads=True), c2.optim, max_norm=400)
    assert restore(first[-1]["checkpoint"], model, opt) == (1, 4)
    for k, v in model.state_dict().items():
        assert torch.equal(v, ck["state_dict"][k]), k
    saved = ck["optimizer_states"][0]
    for i, s in opt.state_dict()["state"].items():
        assert torch.equal(s["momentum_buffer"], saved["state"][i]["momentum_buffer"])
        assert float(s["step"]) == float(saved["state"][i]["step"]) == 4
    assert opt.lr == saved["param_groups"][0]["lr"]
    # then the run goes on from the next epoch
    c2.load_auto_checkpoint = True
    resumed = ds.train(c2)
    assert [(r["epoch"], r["global_step"]) for r in resumed] == [(1, 8)]
    assert sorted(os.listdir(tmp_path)) == sorted(os.listdir(out))
    got, want = _ckpt(resumed[-1]["checkpoint"])["state_dict"], _ckpt(straight[-1]["checkpoint"])["state_dict"]
    assert params_rel_l2(got, want) <= TOL
    assert resumed[-1]["loss"] == pytest.approx(straight[-1]["loss"], rel=TOL)


@pytest.mark.parametrize("rnn", ["lstm", "gru"])
def test_precision_16_with_spec_augment_learns(data, tmp_path, rnn):
    cfg = _cfg(data, tmp_path, rnn=rnn, optim=ds.AdamConfig(learning_rate=2e-3), epochs=6, precision=16)
    cfg.data.augmentation.spec_augment = True
    cfg.checkpoint.monitor, cfg.checkpoint.save_last = "wer", True
    recs = ds.train(cfg)
    losses = [r["loss"] for r in recs]
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < 0.7 * losses[0], losses
    assert "last.ckpt" in os.listdir(tmp_path)
    assert ds.load_model(torch.device("cuda"), str(tmp_path / "last.ckpt")).precision == 16


def test_batcher_waits_before_rewriting_its_staging_buffers():
    """a copy queued behind other work must read the batch it was issued for, not the next one"""
    rng = np.random.default_rng(5)
    lens = [16000, 12000, 9000]
    batches = [[rng.standard_normal(n).astype(np.float32) for n in lens] for _ in range(2)]
    tr = [[1, 2, 3]] * len(lens)
    alone = []
    for waves in batches:
        b = SpectrogramBatcher(ds.SpectConfig())
        alone.append(b(waves, tr)[0])
        torch.cuda.synchronize()
    b = SpectrogramBatcher(ds.SpectConfig())
    b(batches[0], tr)                       # allocates the staging buffers
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)          # ~0.1 s of device work ahead of the copies
    outs = [b(waves, tr)[0] for waves in batches]
    torch.cuda.synchronize()
    for got, want in zip(outs, alone):
        assert torch.equal(got, want)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_worker(rank, port, data, out, q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        os.environ.update(RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                          MASTER_PORT=str(port))
        import deepspeech_pytorch_b200.training as T
        seen = []

        class Recording(T.FusedOptimizer):          # keeps the run's optimizer, and so its flat parameters
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                seen.append(self)
        T.FusedOptimizer = Recording
        recs = T.train(_cfg(data, out, epochs=1))
        q.put((rank, recs[-1]["checkpoint"], recs[-1]["global_step"], seen[0].flat.data.cpu().numpy()))
        torch.distributed.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "error", traceback.format_exc(), None))
        raise


def test_two_ranks_stay_identical_and_only_rank_0_writes(data, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one GPU per rank")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    outs = [tmp_path / "r0", tmp_path / "r1"]
    procs = [ctx.Process(target=_rank_worker, args=(r, port, data, str(outs[r]), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        item = q.get(timeout=600)
        assert item[1] != "error", item[2]
        res[item[0]] = item
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert res[1][1] is None and not outs[1].exists()          # rank 1 wrote nothing
    assert res[0][2] == res[1][2] == 2                         # 4 bins dealt over 2 ranks
    assert os.listdir(outs[0]) == ["epoch=0-step=2.ckpt"]
    assert np.array_equal(res[0][3], res[1][3])
