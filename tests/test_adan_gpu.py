"""GPU: the fused Adan update (csrc/adan.cu, make-it-3d_b200/optimizer.py; SURVEY.md 8f-1) against vectors recorded from the
REFERENCE's optimizer.py + clip_grad_norm_ (tests/golden/adan.npz), at the real model size against the CPU oracle, and -- on a
2-GPU box -- the reduce-scatter -> sharded update -> all-gather form against the single-process update of the summed gradients."""
import importlib
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _close(a, ref, rtol=3e-6):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert np.max(np.abs(a - ref)) <= rtol * max(1e-30, np.abs(ref).max()), float(np.max(np.abs(a - ref)) / np.abs(ref).max())


def test_adan_matches_reference_optimizer_vectors():
    om = importlib.import_module("make-it-3d_b200.optimizer")
    z = load_golden("adan.npz")
    params = [torch.nn.Parameter(torch.from_numpy(z[f"p0_{i}"].copy()).cuda()) for i in range(4)]
    lr = float(z["lr"])
    opt = om.Adan([{"params": params[:1], "lr": lr * 10}, {"params": params[1:], "lr": lr}], eps=1e-8, weight_decay=2e-5, max_grad_norm=5.0,
                  foreach=False, clip_grad_norm=10.0)
    for step in range(4):
        for i, p in enumerate(params):
            p.grad = torch.from_numpy(z[f"g{step}_{i}"].copy()).cuda()
        opt.step()
        torch.cuda.synchronize()
        for i, p in enumerate(params):
            _close(p.detach().cpu().numpy(), z[f"p{step + 1}_{i}"])
            for k in ("exp_avg", "exp_avg_sq", "exp_avg_diff", "neg_pre_grad"):
                _close(opt.state[p][k].cpu().numpy().reshape(z[f"{k}{step + 1}_{i}"].shape), z[f"{k}{step + 1}_{i}"])
        # like the reference, .grad is left clipped (both factors applied): neg_pre_grad == -grad
        assert torch.equal(params[1].grad.view(-1), -opt.state[params[1]]["neg_pre_grad"])


def test_adan_full_model_size_vs_oracle():
    """12 196 240-element hash table + the 6 MLP tensors, three steps, vs oracle/adan_ref.py on the host"""
    from oracle.adan_ref import AdanRef
    om = importlib.import_module("make-it-3d_b200.optimizer")
    g = torch.Generator().manual_seed(1)
    shapes = [(12196240,), (64, 32), (64,), (64, 64), (64,), (4, 64), (4,)]
    host = [torch.randn(s, generator=g) * 0.05 for s in shapes]
    params = [torch.nn.Parameter(h.clone().cuda()) for h in host]
    opt = om.Adan([{"params": params[:1], "lr": 5e-2}, {"params": params[1:], "lr": 5e-3}], eps=1e-8, weight_decay=2e-5, max_grad_norm=5.0,
                  clip_grad_norm=10.0)
    ref = AdanRef([{"params": host[:1], "lr": 5e-2}, {"params": host[1:], "lr": 5e-3}], eps=1e-8, weight_decay=2e-5, max_grad_norm=5.0, clip_grad_norm=10.0)
    for step, sc in enumerate((1e-4, 2e-3, 1e-2)):
        grads = [torch.randn(s, generator=g) * sc for s in shapes]
        for p, gr in zip(params, grads):
            p.grad = gr.clone().cuda()
        opt.step()
        ref.step([grads[:1], grads[1:]])
    torch.cuda.synchronize()
    for p, h in zip(params, host):
        _close(p.detach().cpu().numpy(), h.numpy(), rtol=1e-5)


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, result):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    par = importlib.import_module("make-it-3d_b200.parallel")
    om = importlib.import_module("make-it-3d_b200.optimizer")
    par.init_distributed(backend="nccl")
    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(2)
    shapes = [(4 * 1024 * 1024,), (64, 64), (64,)]
    init = [torch.randn(s, generator=g) * 0.05 for s in shapes]
    params = [torch.nn.Parameter(t.clone().to(dev)) for t in init]
    opt = om.Adan([{"params": params[:1], "lr": 5e-2}, {"params": params[1:], "lr": 5e-3}], weight_decay=2e-5, max_grad_norm=5.0, clip_grad_norm=10.0)
    per_rank = [[[torch.randn(s, generator=g) * sc for s in shapes] for _ in range(world)] for sc in (1e-3, 2e-2)]
    for st in range(2):
        for p, gr in zip(params, per_rank[st][rank]):
            p.grad = gr.clone().to(dev)
        opt.step()
    torch.cuda.synchronize()
    out = dict(params=[p.detach().cpu() for p in params])
    if rank == 0:
        single = [torch.nn.Parameter(t.clone().to(dev)) for t in init]
        opt1 = om.Adan([{"params": single[:1], "lr": 5e-2}, {"params": single[1:], "lr": 5e-3}], weight_decay=2e-5, max_grad_norm=5.0,
                       clip_grad_norm=10.0)
        opt1._world = lambda: (1, 0)                       # single-process statement: summed gradients, no collectives
        for st in range(2):
            for i, p in enumerate(single):
                p.grad = sum(per_rank[st][r][i] for r in range(world)).to(dev)
            opt1.step()
        torch.cuda.synchronize()
        out["single"] = [p.detach().cpu() for p in single]
    result[rank] = out
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_sharded_adan_equals_single_process_update():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mgr = mp.Manager()
    result = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), result), nprocs=2, join=True)
    r0, r1 = result[0], result[1]
    for a, b, s in zip(r0["params"], r1["params"], r0["single"]):
        assert torch.equal(a, b)                                   # replicas stay bit-identical
        _close(a.numpy(), s.numpy(), rtol=2e-6)
