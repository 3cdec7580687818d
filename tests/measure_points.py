"""Times the refine stage's point renderer and z-buffer on the GPU (python tests/measure_points.py [--out FILE]).

Shapes of one refine iteration (nerf/utils.py:846-868): a dense surface cloud (the union of 33 depth-map clouds of a sphere, about
1.3 M points), 19 channels (3 colour + 16 features) rendered at 800^2, 400^2 and 200^2 with the refine radius (2 px at 800^2) and
8 points per pixel, the 800^2 coverage mask (3 channels of ones, no gradient), and the colour backward.  Plus z_buffer on 1 M points
at 800^2 (load_views' preprocessing, once per view).
Reported: ms per leg (CUDA events over the timed calls), per-kernel time (torch.profiler, a separate pass) against the bytes each kernel
must move at least (computed from the shapes below), and the card name and power limit read in the same run.  There is no pytorch3d
arm: the package is not installed, so no speed-up against it is measured.  Lives under tests/ because it imports the oracle's scene
helpers."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import points_ref as pr  # noqa: E402


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_ms(fn, reps=5):
    """CUDA kernel time per call by kernel name (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = next((k for k in ("k_points_bin_count", "k_points_tile_scan", "k_points_bin_emit", "k_points_raster", "k_points_feat_grad",
                                     "k_zbuffer_min", "k_zbuffer_mask") if k in e.name), "other")
            out[name] = out.get(name, 0.0) + e.device_time / 1e3 / reps
    return out


def tile_pairs(v, K, w2c, S, radius):
    """(point, 16x16 tile) pairs the binning emits: the footprint of csrc/points.cu axis_range, evaluated with torch"""
    px, py, pz = pr.project_ndc(v, K, w2c, S, S)
    ok = (pz >= 0) & torch.isfinite(px) & torch.isfinite(py)
    n = torch.ones_like(px)
    for p in (px, py):
        a = torch.floor((S * (1 - p - radius) - 1) * 0.5) - 1
        b = torch.ceil((S * (1 - p + radius) - 1) * 0.5) + 1
        ok &= (b >= 0) & (a <= S - 1)
        lo, hi = a.clamp(0, S - 1).long() // 16, b.clamp(0, S - 1).long() // 16
        n = n * (hi - lo + 1)
    return int(n[ok].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_points.py needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    card = q.strip().splitlines()[0] if q.strip() else "unknown"
    ru = importlib.import_module("make-it-3d_b200.nerf.refine_utils")

    H, ppp, C = 800, 8, 19
    radius = 2.0 / H * 2.0
    v = torch.from_numpy(pr.surface_cloud(33, 207, seed=0)).cuda()
    P = v.shape[0]
    feats = torch.rand(P, C, device="cuda", requires_grad=True)
    ones = torch.ones(P, 3, device="cuda")
    w2c = torch.linalg.inv(torch.from_numpy(pr.lookat_c2w(1.2, 60.0, 20.0)).float()).cuda()
    Ks = {s: torch.from_numpy(pr.intrinsics(s)).float().cuda() for s in (800, 400, 200)}
    grads = {s: torch.rand(1, C, s, s, device="cuda") for s in (800, 400, 200)}

    def fwd(s, f=feats):
        return ru.render_point(v, f, s, s, Ks[s], w2c, (s, s), radius, ppp)

    def fwd_bwd(s):
        fwd(s).backward(grads[s])

    def iteration():
        imgs = [fwd(s) for s in (800, 400, 200)]
        fwd(800, ones)
        torch.autograd.backward(imgs, [grads[s] for s in (800, 400, 200)])

    vz = pr.surface_cloud(33, 185, seed=1)[:1_000_000].astype(np.float64)
    w2c_np = np.linalg.inv(pr.lookat_c2w(1.2, 60.0, 20.0))
    K_np = pr.intrinsics(H)
    zb = lambda: ru.z_buffer(vz, w2c_np, H, H, K_np)

    legs = [("render_800_c19_fwd", lambda: fwd(800)), ("render_400_c19_fwd", lambda: fwd(400)), ("render_200_c19_fwd", lambda: fwd(200)),
            ("mask_800_c3_fwd", lambda: fwd(800, ones)), ("render_800_c19_fwd_bwd", lambda: fwd_bwd(800)),
            ("render_400_c19_fwd_bwd", lambda: fwd_bwd(400)), ("render_200_c19_fwd_bwd", lambda: fwd_bwd(200)),
            ("refine_iteration_renders", iteration), ("z_buffer_1M_800_numpy_io", zb)]
    rows = []
    for name, fn in legs:
        with torch.no_grad() if name.endswith("_fwd") else torch.enable_grad():
            ms = timed(fn, args.warmup, args.iters)
            km = kernel_ms(fn)
        rows.append(dict(leg=name, ms_per_call=round(ms, 3), kernel_ms={k: round(t, 4) for k, t in km.items()}))

    # bytes each kernel must move at least, one 800^2 C=19 forward + backward: every input read once, every output written once
    S, K = 800, ppp
    pairs = tile_pairs(v.cpu(), Ks[800].cpu(), w2c.cpu(), S, radius)
    px_slots = S * S * K
    need = {"k_points_bin_count": P * 12 + P * 16 + pairs * 4,            # points in, projected points out, one counter RED per pair
            "k_points_bin_emit": P * 16 + pairs * 4,                       # projected points in, list entries out
            "k_points_raster": pairs * (4 + 16) + px_slots * 8 + S * S * C * 4 + P * C * 4,   # list + gathered points, idx / w, image, feats
            "k_points_feat_grad": P * 12 + px_slots * 8 + S * S * C * 4 + P * C * 4}          # points, idx / w, grad image in; dfeat out
    kt = next(r for r in rows if r["leg"] == "render_800_c19_fwd_bwd")["kernel_ms"]
    roof = {k: dict(mbytes=round(b / 1e6, 1), ms=kt.get(k), gb_per_s=round(b / (kt[k] * 1e-3) / 1e9, 1) if kt.get(k) else None)
            for k, b in need.items()}
    nz = len(vz)
    zt = next(r for r in rows if r["leg"] == "z_buffer_1M_800_numpy_io")["kernel_ms"]
    for k, b in (("k_zbuffer_min", nz * 24 + nz * 8), ("k_zbuffer_mask", nz * 24 + nz * 8 + nz)):
        roof[k] = dict(mbytes=round(b / 1e6, 1), ms=zt.get(k), gb_per_s=round(b / (zt[k] * 1e-3) / 1e9, 1) if zt.get(k) else None)
    out = dict(card=card, points=P, zbuffer_points=nz, point_tile_pairs_800=pairs, radius_ndc=radius, ppp=ppp, channels=C,
               warmup=args.warmup, iters=args.iters, legs=rows, kernel_bytes_800_c19=roof,
               note="no pytorch3d arm: the package is not installed, so no speed-up against it is measured")
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
