"""What the render path computes at the benchmark scene, for comparing two builds of libmi3d.so (MI3D_LIB_PATH selects one):
the inputs of tools/prof_render.py (128x128, sphere r=0.2, camera radius 1.25), lambertian, lambda_smooth = 1, fixed `noises` and
`smooth_noise`; one forward, the image-only backward, the regularisers' backward, one update_extra_state(seed=...).
    python tools/field_outputs.py --out a.npz              (GPU) writes image, depth, weights_sum, the two losses, the six MLP
                                                           gradients and the table gradient after each backward, density grid / bitfield
    python tools/field_outputs.py --compare a.npz b.npz    per array: bit-identical or max |a - b| / max |a|
Forward outputs and the density grid are deterministic; the gradients are fp32 atomics whose order varies from run to run, so judge
a gradient difference between two builds against the difference between two runs of one build."""
import argparse
import importlib
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dump(path, hw):
    import torch

    import bench  # oracle-free input builders: orbit_pose, sphere_bitfield_numpy
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    utils = importlib.import_module("make-it-3d_b200.nerf.utils")
    field_ops = importlib.import_module("make-it-3d_b200.nerf.field_ops")
    opt = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1, lambda_smooth=1, max_depth=10.0)
    torch.manual_seed(0)
    net = nt.NeRFNetwork(opt).cuda().train()
    rng = np.random.default_rng(3)
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(((rng.random(net.encoder.params.numel(), dtype=np.float32) * 2 - 1) * 0.5).astype(np.float32)))
    net.density_bitfield = torch.from_numpy(bench.sphere_bitfield_numpy(0.2)).cuda()
    pose = torch.from_numpy(bench.orbit_pose(1.25, 80.0, 170.0))[None].cuda()
    focal = hw / (2 * math.tan(math.radians(20.0) / 2))
    rays = utils.get_rays(pose, (focal, focal, hw / 2, hw / 2), hw, hw, -1)
    cu = lambda a: torch.from_numpy(a).cuda()
    kw = dict(depth_scale=rays["depth_scale"], bg_color=cu(np.array([0.1, 0.2, 0.3], np.float32)), perturb=True,
              light_d=cu(np.array([0.0, 0.6, 0.8], np.float32)), ambient_ratio=0.1, shading="lambertian", force_all_rays=True, max_steps=512,
              noises=cu(rng.random(hw * hw, dtype=np.float32)))
    with torch.no_grad():       # the march depends on `noises` only: learn the sample count, then draw one perturbation per padded row
        net.render(rays["rays_o"], rays["rays_d"], **kw)
    M = int(list(net._workspaces.values())[0].counter[0])
    kw["smooth_noise"] = cu(rng.standard_normal((M + 128, 3)).astype(np.float32))
    gimg = cu(rng.standard_normal((1, hw * hw, 3)).astype(np.float32))
    out = net.render(rays["rays_o"], rays["rays_d"], **kw)
    res = {"M": np.int64(M)}
    for k in ("image", "depth", "weights_sum", "loss_orient", "loss_smooth"):
        res[k] = out[k].detach().cpu().numpy()
    params = [("table", net.encoder.params)] + [(f"{n}{l + 1}", getattr(net.sigma_net.net[l], a)) for l in range(3) for n, a in (("w", "weight"), ("b", "bias"))]
    (out["image"] * gimg).sum().backward(retain_graph=True)                # SDS-style backward: image gradient only
    for n, p in params:
        res[f"g_image_{n}"] = p.grad.cpu().numpy()
    (0.01 * out["loss_orient"] + out["loss_smooth"] + (out["weights_sum"] ** 2).mean()).backward()   # regularisers; gradients accumulate
    for n, p in params:
        res[f"g_both_{n}"] = p.grad.cpu().numpy()
    net.update_extra_state(seed=7)
    res["density_grid"] = net.density_grid.cpu().numpy()
    res["density_bitfield"] = net.density_bitfield.cpu().numpy()
    res["mean_density"] = net.mean_density.cpu().numpy()
    np.savez(path, **res)
    print(f"{path}: M = {M}, backward scratch {field_ops.bwd_scratch(torch.device('cuda', 0)).numel() / 1e9:.3f} GB, "
          f"max_memory_allocated {torch.cuda.max_memory_allocated() / 1e9:.3f} GB on {torch.cuda.get_device_name(0)}")


def compare(pa, pb):
    a, b = np.load(pa), np.load(pb)
    print(f"# {pa} vs {pb}")
    for k in a.files:
        x, y = a[k], b[k]
        if x.tobytes() == y.tobytes():
            print(f"{k:24s} bit-identical")
        else:
            x64, y64 = x.astype(np.float64), y.astype(np.float64)
            print(f"{k:24s} max |a - b| / max |a| = {np.abs(x64 - y64).max() / max(np.abs(x64).max(), 1e-30):.3e}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--hw", type=int, default=128)
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        compare(*args.compare)
    else:
        dump(args.out, args.hw)
