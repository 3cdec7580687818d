"""Per-phase CUDA-event timing of the render path at the BASELINE workload (128x128, sphere r=0.2, camera radius 1.25).
Usage (GPU box): python tools/prof_render.py [--hw 128] [--evals 13] [--iters 10]"""
import argparse
import importlib
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402      (oracle-free input builders: orbit_pose, sphere_bitfield_numpy)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hw", type=int, default=128)
    ap.add_argument("--radius", type=float, default=0.2)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--shading", default="albedo")
    args = ap.parse_args()
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    opt = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1,
                             lambda_smooth=1, max_depth=10.0)
    torch.manual_seed(0)
    net = nt.NeRFNetwork(opt).cuda().train()
    with torch.no_grad():
        table = ((np.random.default_rng(3).random(net.encoder.params.numel(), dtype=np.float32) * 2 - 1) * 0.5).astype(np.float32)
        net.encoder.params.copy_(torch.from_numpy(table))
    net.density_bitfield = torch.from_numpy(bench.sphere_bitfield_numpy(args.radius)).cuda()
    # camera radius 1.25, theta 80, phi 170, fovy 20 (the camera of the parity tests' fixtures), rays from the product's own k_get_rays
    utils = importlib.import_module("make-it-3d_b200.nerf.utils")
    pose = torch.from_numpy(bench.orbit_pose(1.25, 80.0, 170.0))[None].cuda()
    focal = args.hw / (2 * math.tan(math.radians(20.0) / 2))
    rays = utils.get_rays(pose, (focal, focal, args.hw / 2, args.hw / 2), args.hw, args.hw, -1)
    ro, rd, sc = rays["rays_o"], rays["rays_d"], rays["depth_scale"]
    bg = torch.rand(3, device="cuda")
    light = torch.tensor([0.0, 0.6, 0.8], device="cuda")
    gimg = torch.randn(1, args.hw * args.hw, 3, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for lam_smooth in (1, 0):
        net.opt.lambda_smooth = lam_smooth
        tf, tb1, tb2 = [], [], []
        for it in range(args.iters + 3):
            flush.zero_()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            net.zero_grad(set_to_none=True)
            e[0].record()
            out = net.render(ro, rd, depth_scale=sc, bg_color=bg, perturb=True, light_d=light, ambient_ratio=0.1 if args.shading != "albedo" else 1.0,
                             shading=args.shading, force_all_rays=True, max_steps=512)
            e[1].record()
            (out["image"] * gimg).sum().backward(retain_graph=True)          # SDS-style backward: image gradient only
            e[2].record()
            loss = 0.01 * out["loss_orient"] + (out["loss_smooth"] if lam_smooth else 0) + (out["weights_sum"] ** 2).mean()
            loss.backward()                                                    # second backward: regularisers
            e[3].record()
            torch.cuda.synchronize()
            if it >= 3:
                tf.append(e[0].elapsed_time(e[1])); tb1.append(e[1].elapsed_time(e[2])); tb2.append(e[2].elapsed_time(e[3]))
        ws = list(net._workspaces.values())[0]
        M = int(ws.counter[0])
        k = 13 if lam_smooth else 7
        med = lambda v: float(np.median(v))
        print(f"hw={args.hw} M={M} k={k} shading={args.shading}: fwd {med(tf):.3f} ms | bwd(image only) {med(tb1):.3f} ms | bwd(regularisers) {med(tb2):.3f} ms"
              f" | fwd evals/s {M * k / med(tf) / 1e6:.1f} G/s-equivalent(M/ms)")


if __name__ == "__main__":
    main()
