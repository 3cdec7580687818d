"""2 GPUs (skipped on a 1-GPU machine): the ray-parallel render step over NCCL ==
single-process sequential accumulation of the same G = 2 views (SURVEY.md 8e: "define G-GPU step == single-GPU accumulation of
the same G poses' gradients ... and test exactly that equivalence").

Each rank marches every 2nd pixel of BOTH views (balanced sample counts whatever the poses), fragments go to the view's owner by
all-to-all, per-view loss means use the all-gathered total sample counts, gradients are summed by GradientAllReduce.  Expected:
  * the owner's image / depth / weights_sum are BIT-identical to the unsharded render of that view (same samples, same kernels),
  * per-view regulariser means and the summed parameter gradients agree to summation-order accuracy,
  * the two ranks march (nearly) the same number of samples although one view is heavier than the other."""
import argparse
import importlib
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

HW = 64


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _setup(device):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conftest import load_golden
    from helpers import fr, make_table, sphere_bitfield
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    g = load_golden("render_albedo.npz")
    o = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1, lambda_smooth=1, max_depth=10.0)
    net = nt.NeRFNetwork(o)
    table = make_table(net.encoder.params.numel(), int(g["table_seed"]), float(g["table_scale"]))
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(table))
        for l, (w, b) in enumerate((("w1", "b1"), ("w2", "b2"), ("w3", "b3"))):
            net.sigma_net.net[l].weight.copy_(torch.from_numpy(g[w]))
            net.sigma_net.net[l].bias.copy_(torch.from_numpy(g[b]))
    net = net.to(device).train()
    net.density_bitfield = torch.from_numpy(sphere_bitfield(0.3)).to(device)
    poses = torch.from_numpy(np.stack([fr.orbit_pose(1.0, 90.0, 180.0), fr.orbit_pose(1.5, 75.0, 40.0)]))     # close (heavy) and far (light) view
    intr = torch.tensor([[HW / (2 * math.tan(math.radians(f) / 2))] * 2 + [HW / 2, HW / 2] for f in (20.0, 18.0)])
    rng = np.random.default_rng(5)
    A = torch.from_numpy(rng.standard_normal((2, HW * HW, 3)).astype(np.float32)).to(device)
    B = torch.from_numpy(rng.standard_normal((2, HW * HW)).astype(np.float32)).to(device)
    bg = torch.from_numpy(rng.random((2, 3), dtype=np.float32)).to(device)
    light = torch.nn.functional.normalize(torch.from_numpy(rng.standard_normal((2, 3)).astype(np.float32)), dim=1).to(device)
    return net, poses, intr, A, B, bg, light


def _loss(out, A, B):
    return (out["image"][0] * A).sum() + (out["weights_sum"][0] * B).sum() + 30.0 * out["loss_orient"] + 50.0 * out["loss_smooth"]


def _worker(rank, world, port, result):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    par = importlib.import_module("make-it-3d_b200.parallel")
    par.init_distributed(backend="nccl")
    device = torch.device("cuda", rank)
    net, poses, intr, A, B, bg, light = _setup(device)
    rp = par.RayParallel()
    reducer = par.GradientAllReduce(net.encoder.params, list(net.sigma_net.parameters()), op="sum")
    kw = dict(perturb=True, shading="lambertian", ambient_ratio=0.1, force_all_rays=True, max_steps=512, step_seed=par.shared_seed(3, 11))
    out = net.render(None, None, cam_poses=poses, cam_intrinsics=intr, cam_hw=(HW, HW), bg_color=bg, light_d=light, ray_parallel=rp, **kw)
    _loss(out, A[rank], B[rank]).backward()
    reducer()
    torch.cuda.synchronize()
    ws = list(net._workspaces.values())[0]
    res = dict(image=out["image"][0].detach().cpu(), depth=out["depth"][0, :, 0].detach().cpu(), ws=out["weights_sum"][0].detach().cpu(), lo=float(out["loss_orient"]),
               ls=float(out["loss_smooth"]), marched=int(ws.counter[0]), g_table=net.encoder.params.grad.detach().cpu(),
               g_mlp=[p.grad.detach().cpu() for p in net.sigma_net.parameters()])
    if rank == 0:
        # the single-process statement of the same step: both views rendered whole, gradients accumulated
        net.zero_grad()
        seq = []
        for v in range(world):
            o = net.render(None, None, cam_poses=poses[v:v + 1], cam_intrinsics=intr[v], cam_hw=(HW, HW), bg_color=bg[v], light_d=light[v], **kw)
            _loss(o, A[v], B[v]).backward()
            seq.append(dict(image=o["image"][0].detach().cpu(), depth=o["depth"][0, :, 0].detach().cpu(), ws=o["weights_sum"][0].detach().cpu(), lo=float(o["loss_orient"]),
                            ls=float(o["loss_smooth"]), marched=int(list(net._workspaces.values())[0].counter[0])))
        torch.cuda.synchronize()
        res["seq"] = seq
        res["seq_g_table"] = net.encoder.params.grad.detach().cpu()
        res["seq_g_mlp"] = [p.grad.detach().cpu() for p in net.sigma_net.parameters()]
    # replicas refresh the occupancy grid themselves with a seed every rank shares: no broadcast, identical bitfields (parallel.py)
    net.update_extra_state(decay=0.95, seed=par.shared_seed(3, 16))
    torch.cuda.synchronize()
    res["bitfield"] = net.density_bitfield.cpu()
    res["grid"] = net.density_grid.cpu()
    result[rank] = res
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_two_rank_ray_parallel_step_equals_sequential_accumulation():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mgr = mp.Manager()
    result = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), result), nprocs=2, join=True)
    r0, r1 = result[0], result[1]
    seq = r0["seq"]
    for v, r in ((0, r0), (1, r1)):
        assert torch.equal(r["image"], seq[v]["image"]) and torch.equal(r["ws"], seq[v]["ws"]) and torch.equal(r["depth"], seq[v]["depth"])
        assert abs(r["lo"] / seq[v]["lo"] - 1) < 2e-5 and abs(r["ls"] / seq[v]["ls"] - 1) < 2e-5
    # every rank holds the same, summed gradients == sequential accumulation
    assert torch.equal(r0["g_table"], r1["g_table"])
    gs = r0["seq_g_table"]
    assert float((r0["g_table"] - gs).abs().max()) <= 5e-5 * float(gs.abs().max())
    assert int((r0["g_table"] != 0).sum()) == int((gs != 0).sum())
    for a, b in zip(r0["g_mlp"], r0["seq_g_mlp"]):        # per-CTA weight-gradient sums over ~1.5 M evaluations in a different tile order
        assert float((a - b).abs().max()) <= 2e-4 * float(b.abs().max())
    # balance: the views differ in samples (close view ~1.18x the far one), the ranks do not
    assert seq[0]["marched"] > 1.1 * seq[1]["marched"]
    assert r0["marched"] + r1["marched"] == seq[0]["marched"] + seq[1]["marched"]
    assert abs(r0["marched"] - r1["marched"]) < 0.03 * (r0["marched"] + r1["marched"])
    assert torch.equal(r0["bitfield"], r1["bitfield"]) and torch.equal(r0["grid"], r1["grid"])
    print(f"samples: views {seq[0]['marched']} / {seq[1]['marched']}  ->  ranks {r0['marched']} / {r1['marched']}")
