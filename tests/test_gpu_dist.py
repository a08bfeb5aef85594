"""-m gpu: row a12 — the data-parallel step reproduces DDP's semantics numerically (SURVEY.md §4 T3).

Reference semantics (configs/librispeech.yaml:14 `strategy: ddp`, training.py:42-47): every rank computes the
SUM-reduced CTC loss of its own minibatch, DDP averages the gradients over ranks, BatchNorm running statistics are
not synchronised and rank 0's are what gets checkpointed.  Two real ranks run the CUDA path on their own shard —
both processes on cuda:0 over gloo (which moves CUDA tensors) when the box has one GPU, over NCCL on cuda:0 / cuda:1
when it has two — through `OverlappedGradAllReduce` and the fused optimizer's 1/world scale; the flat gradient must
equal the oracle's mean of per-shard gradients and the parameters after one fused AdamW step must equal torch AdamW
applied to that mean."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

from conftest import ROOT

pytestmark = pytest.mark.gpu

CFG = dict(rnn_type="lstm", H=32, layers=2, B=3, T=90)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _shard(rank):
    sys.path.insert(0, ROOT)
    from oracle import ds2_oracle as O
    return O.synth_batch(CFG["B"], CFG["T"], seed=40 + rank, lmin=4, lmax=10)


def _params():
    from oracle import ds2_oracle as O
    ocfg = O.OracleConfig(rnn_type=CFG["rnn_type"], hidden_size=CFG["H"], hidden_layers=CFG["layers"],
                          bidirectional=True)
    return ocfg, O.init_params(ocfg, seed=9)


def _worker(rank, world, port, backend, direct, q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank if backend == "nccl" else 0),
                          MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        import deepspeech_pytorch_b200 as ds
        from deepspeech_pytorch_b200 import dist as D
        from deepspeech_pytorch_b200.optim import FlatParams, FusedOptimizer
        from gpu_helpers import make_model
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        D.init_from_env(backend)
        ds.set_precision("fp32")
        _, P = _params()
        model = make_model(CFG["rnn_type"], True, CFG["H"], CFG["layers"], params=P, device=dev).train()
        flat = FlatParams(model, direct_grads=direct)   # True: per-block exchange from the backward hooks
        opt = FusedOptimizer(flat, model.optim_cfg, max_norm=400.0)
        ex = D.OverlappedGradAllReduce(flat, model)
        x, targets, pct, tsz = _shard(rank)
        loss = model.training_step((x.to(dev), targets, pct.clone(), tsz), 0)
        loss.backward()
        ex.finish()
        torch.cuda.synchronize()
        # numpy: pickled by value (torch tensors travel as shared-memory handles that die with this process)
        grads = {k: (p.grad.detach() / world).cpu().numpy() for k, p in model.named_parameters()}
        opt.step(grad_scale=1.0 / world)
        D.broadcast_buffers(model, src=0)
        torch.cuda.synchronize()
        sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
        q.put((rank, float(loss), grads, sd))
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, "error", traceback.format_exc(), repr(e)))
        raise


@pytest.mark.parametrize("backend,direct", [("gloo", False), ("gloo", True), ("nccl", True)])
def test_two_rank_step_equals_oracle_mean_gradient(backend, direct):
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one GPU per rank (bench.py --gpus 2/4/8 covers it on the 8-GPU box)")
    from oracle import ds2_oracle as O
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, direct, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = {}
    for _ in range(world):
        item = q.get(timeout=600)
        assert item[1] != "error", item[2]
        results[item[0]] = item
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    # oracle: per-shard train steps on the CPU, mean of the gradients (DDP), rank 0's BN buffers
    ocfg, P = _params()
    refs = []
    for r in range(world):
        x, targets, pct, tsz = _shard(r)
        refs.append(O.train_step(x, targets, pct.clone(), tsz, P, ocfg))
    for r in range(world):
        assert abs(results[r][1] - refs[r]["loss"]) <= 1e-4 * max(1.0, abs(refs[r]["loss"]))
    mean = {k: sum(ref["grads"][k] for ref in refs) / world for k in refs[0]["grads"]}
    for r in range(world):
        for k, g in results[r][2].items():
            g = torch.from_numpy(g)
            d = float(mean[k].abs().max()) or 1.0
            assert float((g - mean[k]).abs().max()) / d < 2e-3, (r, k)
    # parameters after the fused clip + AdamW step == torch.optim.AdamW on the averaged gradient
    leaves = {k: torch.nn.Parameter(v.clone()) for k, v in P.items() if k in mean}
    for k, p in leaves.items():
        p.grad = mean[k].clone()
    torch.nn.utils.clip_grad_norm_(list(leaves.values()), 400.0)
    torch.optim.AdamW(list(leaves.values()), lr=1.5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5).step()
    for r in range(world):
        sd = {k: torch.from_numpy(v) for k, v in results[r][3].items()}
        for k, p in leaves.items():
            # AdamW's first step moves every weight by ~lr regardless of the gradient scale: compare the UPDATE
            # (where the gradient is far above eps = 1e-8, so that g / (|g| + eps) is insensitive to its last bits)
            upd, ref_upd = sd[k] - P[k], p.detach() - P[k]
            keep = mean[k].abs() > 1e-5
            assert float(((upd - ref_upd).abs() * keep).max()) < 0.02 * 1.5e-4 + 1e-7, (r, k)
        for k, v in refs[0]["new_buffers"].items():        # every rank now holds rank 0's running statistics
            d = float(v.abs().max()) or 1.0
            assert float((sd[k] - v).abs().max()) / d < 1e-3, (r, k)
    assert not torch.allclose(refs[0]["new_buffers"]["fc.0.module.0.running_mean"],
                              refs[1]["new_buffers"]["fc.0.module.0.running_mean"])   # the shards really differ
