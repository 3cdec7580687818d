"""GPU: ray generation in the kernel (row R0), the single-entry fused render (mi3d_render_forward / mi3d_render_backward,
SURVEY.md 8b) against the unfused B1 / B2 entry points, and multi-view batches against sequential single-view renders."""
import argparse
import importlib
import math

import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import fr, make_table, max_abs, sphere_bitfield

pytestmark = pytest.mark.gpu


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _net(g, **optkw):
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    o = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1, lambda_smooth=1, max_depth=10.0)
    for k, v in optkw.items():
        setattr(o, k, v)
    net = nt.NeRFNetwork(o)
    table = make_table(net.encoder.params.numel(), int(g["table_seed"]), float(g["table_scale"]))
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(table))
        for l, (w, b) in enumerate((("w1", "b1"), ("w2", "b2"), ("w3", "b3"))):
            net.sigma_net.net[l].weight.copy_(torch.from_numpy(g[w]))
            net.sigma_net.net[l].bias.copy_(torch.from_numpy(g[b]))
    net = net.cuda().train()
    net.density_bitfield = _cu(sphere_bitfield(0.3))
    return net


def test_get_rays_kernel_matches_reference_vectors():
    """mi3d_get_rays vs the vectors recorded from the REFERENCE's get_rays (nerf/utils.py:51-116; tests/golden/make_golden.py):
    rays_o bit for bit; depth_scale within 2 ulp (torch's vectorised pow / reciprocal); rays_d within 2 ulp of a unit vector
    (torch's CPU matmul may contract the 3-term dot product into FMAs, this kernel rounds every operation)."""
    U = importlib.import_module("make-it-3d_b200.nerf.utils")
    g = load_golden("small_ops.npz")
    r = U.get_rays(_cu(g["pose"])[None], (40.0, 42.0, 8.0, 7.5), 15, 16, -1)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(r["rays_o"][0].cpu().numpy(), g["rays_o"])
    sc = r["depth_scale"][0].cpu().numpy()
    d = r["rays_d"][0].cpu().numpy()
    ulp_s = np.abs(sc - g["depth_scale"]) / np.spacing(g["depth_scale"])
    # components near zero: measure in ulps of the vector's length (unit vectors: 1 ulp(1.0) = 1.19e-7)
    ulp = np.abs(d - g["rays_d"]) / np.maximum(np.spacing(np.abs(g["rays_d"]).astype(np.float32)), np.float32(2.0 ** -24))
    print(f"depth_scale: max {ulp_s.max():.1f} ulp, {np.mean(sc == g['depth_scale']) * 100:.1f} % bit-identical; "
          f"rays_d: max {ulp.max():.1f} ulp, {np.mean(d == g['rays_d']) * 100:.1f} % bit-identical, max abs {np.abs(d - g['rays_d']).max():.2e}")
    assert ulp_s.max() <= 2.0 and ulp.max() <= 2.0           # the bound: at most 2 ulp per value
    assert r["inds"].shape == (1, 240) and max_abs(np.linalg.norm(d, axis=1), 1.0) < 1e-6
    with pytest.raises(NotImplementedError):
        U.get_rays(_cu(g["pose"])[None], (40.0, 42.0, 8.0, 7.5), 15, 16, 64)


def _loss(out, A, B):
    return (out["image"] * A).sum() + (out["weights_sum"] * B).sum() + 30.0 * out["loss_orient"].sum() + 50.0 * out["loss_smooth"].sum()


def _grads(net):
    return [net.encoder.params.grad.clone()] + [p.grad.clone() for p in net.sigma_net.parameters()]


@pytest.mark.parametrize("shading", ["albedo", "lambertian"])
def test_fused_entry_points_match_unfused(shading):
    """mi3d_render_forward / mi3d_render_backward with in-kernel ray generation == march / field / composite through the separate
    B1 / B2 entry points on rays from mi3d_get_rays: same kernels, so images are bit-identical; gradients differ by RED order."""
    U = importlib.import_module("make-it-3d_b200.nerf.utils")
    ops = importlib.import_module("make-it-3d_b200.nerf.field_ops")
    g = load_golden("render_albedo.npz")
    net = _net(g)
    HW = 48
    pose = torch.from_numpy(fr.orbit_pose(1.2, 75.0, 200.0))[None]
    focal = HW / (2 * math.tan(math.radians(20.0) / 2))
    intr = (focal, focal, HW / 2, HW / 2)
    rng = np.random.default_rng(9)
    noises, A, B = _cu(rng.random(HW * HW, dtype=np.float32)), _cu(rng.standard_normal((1, HW * HW, 3)).astype(np.float32)), _cu(rng.standard_normal((1, HW * HW)).astype(np.float32))
    light = _cu(np.array([0.2, 0.6, 0.77], np.float32))
    kw = dict(bg_color=_cu(np.array([0.3, 0.1, 0.6], np.float32)), perturb=True, light_d=light, shading=shading, ambient_ratio=0.1,
              force_all_rays=True, max_steps=512, noises=noises, step_seed=1234)
    out = net.render(None, None, cam_poses=pose, cam_intrinsics=intr, cam_hw=(HW, HW), **kw)
    _loss(out, A, B).backward()
    fused = dict(image=out["image"].clone(), depth=out["depth"].clone(), ws=out["weights_sum"].clone(), lo=out["loss_orient"].clone(),
                 ls=out["loss_smooth"].clone(), grads=_grads(net), total=int(list(net._workspaces.values())[0].counter[0]))
    net.zero_grad()
    rays = U.get_rays(pose.cuda(), intr, HW, HW, -1)
    ops.PROFILE = []                                           # routes render_train through the unfused three-call path
    try:
        out2 = net.render(rays["rays_o"], rays["rays_d"], depth_scale=rays["depth_scale"], **kw)
        _loss(out2, A, B).backward()
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    assert {p[0] for p in prof} == {"k_field_fwd", "k_field_bwd"}
    assert fused["total"] == int(list(net._workspaces.values())[0].counter[0]) and fused["total"] > 20000
    assert torch.equal(fused["image"], out2["image"]) and torch.equal(fused["ws"], out2["weights_sum"]) and torch.equal(fused["depth"], out2["depth"])
    assert torch.equal(fused["lo"], out2["loss_orient"]) and torch.equal(fused["ls"], out2["loss_smooth"])
    for a, b in zip(fused["grads"], _grads(net)):
        assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())


def test_multi_view_batch_equals_sequential_views():
    """One march / field / composite over a batch of G views (mi3d_view_segs: per-view sample segments, per-view zero rows and
    loss denominators, per-view background and light) == G single-view renders with accumulated gradients.  This is the
    single-GPU half of the ray-parallel equivalence (tests/test_ray_parallel_gpu.py covers the ranks)."""
    g = load_golden("render_albedo.npz")
    net = _net(g)
    HW, G = 32, 3
    poses = torch.from_numpy(np.stack([fr.orbit_pose(1.1, 80.0, 170.0), fr.orbit_pose(1.4, 100.0, 40.0), fr.orbit_pose(1.25, 72.0, 300.0)]))
    fov = [20.0, 16.0, 24.0]
    intr = torch.tensor([[HW / (2 * math.tan(math.radians(f) / 2))] * 2 + [HW / 2, HW / 2] for f in fov])
    rng = np.random.default_rng(13)
    A, B = _cu(rng.standard_normal((G, HW * HW, 3)).astype(np.float32)), _cu(rng.standard_normal((G, HW * HW)).astype(np.float32))
    bg = _cu(rng.random((G, 3), dtype=np.float32))
    light = torch.nn.functional.normalize(_cu(rng.standard_normal((G, 3)).astype(np.float32)), dim=1)
    kw = dict(perturb=True, shading="lambertian", ambient_ratio=0.1, force_all_rays=True, max_steps=512, step_seed=77)
    out = net.render(None, None, cam_poses=poses, cam_intrinsics=intr, cam_hw=(HW, HW), bg_color=bg, light_d=light, **kw)
    assert out["image"].shape == (G, HW * HW, 3) and out["loss_orient"].shape == (G,) and out["loss_smooth"].shape == (G,)
    _loss(out, A, B).backward()
    batch = dict(image=out["image"].clone(), ws=out["weights_sum"].clone(), depth=out["depth"].clone(), lo=out["loss_orient"].clone(),
                 ls=out["loss_smooth"].clone(), grads=_grads(net))
    ws = list(net._workspaces.values())[0]
    segs = ws.segs()
    counts = [segs.bounds[v + 1] - segs.bounds[v] for v in range(G)]
    assert segs.n_views == G and all(c > 3000 for c in counts) and segs.bounds[G] == int(ws.counter[0])
    assert [segs.mpad[v] for v in range(G)] == [c + 128 - c % 128 for c in counts]
    assert segs.bounds[2 * G] == sum(segs.mpad[v] for v in range(G))         # every view's zero rows are evaluated here
    net.zero_grad()
    seq_counts = []
    for v in range(G):
        o = net.render(None, None, cam_poses=poses[v:v + 1], cam_intrinsics=intr[v], cam_hw=(HW, HW), bg_color=bg[v], light_d=light[v], **kw)
        seq_counts.append(int(list(net._workspaces.values())[0].counter[0]))
        assert torch.equal(o["image"][0], batch["image"][v]) and torch.equal(o["weights_sum"][0], batch["ws"][v])
        assert torch.equal(o["depth"][0], batch["depth"][v])
        assert abs(float(o["loss_orient"]) / float(batch["lo"][v]) - 1) < 2e-5 and abs(float(o["loss_smooth"]) / float(batch["ls"][v]) - 1) < 2e-5
        _loss(dict(o, image=o["image"][0], weights_sum=o["weights_sum"][0]), A[v], B[v]).backward()
    assert seq_counts == counts
    for a, b in zip(batch["grads"], _grads(net)):
        assert float((a - b).abs().max()) <= 5e-5 * float(b.abs().max())


@pytest.mark.parametrize("shading", ["albedo", "lambertian"])
def test_eval_renderer_device_loop_equals_host_loop(shading):
    """mi3d_render_eval (the alive-ray loop of renderer.py:526-551 with all loop state on the device, no per-iteration host sync)
    == the reference-shaped host loop over march_rays / field / composite_rays: every ray sees the same samples, so image, depth,
    weights_sum and the normal image are bit-identical (the alive list is compacted in a different order, nothing else differs)."""
    U = importlib.import_module("make-it-3d_b200.nerf.utils")
    g = load_golden("render_albedo.npz")
    net = _net(g).eval()
    HW = 96
    pose = torch.from_numpy(fr.orbit_pose(1.2, 75.0, 200.0))[None].cuda()
    focal = HW / (2 * math.tan(math.radians(25.0) / 2))
    rays = U.get_rays(pose, (focal, focal, HW / 2, HW / 2), HW, HW, -1)
    light = _cu(np.array([0.2, 0.6, 0.77], np.float32))
    kw = dict(depth_scale=rays["depth_scale"], bg_color=_cu(np.array([0.3, 0.1, 0.6], np.float32)), perturb=False, light_d=light, shading=shading,
              ambient_ratio=0.1, max_steps=1024, T_thresh=1e-4)
    with torch.no_grad():
        dev = net.render(rays["rays_o"], rays["rays_d"], eval_loop="device", **kw)
        host = net.render(rays["rays_o"], rays["rays_d"], eval_loop="host", **kw)
    torch.cuda.synchronize()
    assert float(dev["weights_sum"].max()) > 0.9 and float(dev["weights_sum"].min()) == 0.0          # object and background both in view
    rep = {k: (float((dev[k].float() - host[k].float()).abs().max()), float((dev[k] != host[k]).float().mean())) for k in ("image", "depth", "weights_sum", "normal", "mask")}
    print("max |diff|, fraction differing:", rep)
    for k in ("image", "depth", "weights_sum", "normal", "mask"):
        assert torch.equal(dev[k], host[k]), (k, rep)
