"""Time the refine stage's point-cloud construction (nerf/refine_utils.load_views) at the refine stage's size: a seeded synthetic
33-view 800^2 mvimg folder built on the fly (oracle/views_ref.make_mvimg).  Reports the native wall time (ending in a device
synchronise), per-kernel CUDA times from torch.profiler, the CPU oracle's time on the same inputs with the host core count, the
point counts, and whether native and oracle agree.  Prints the card name and power limit read in the same run.
    python tests/measure_load_views.py [--views 33] [--size 800] [--out load_views.json]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import views_ref as vr      # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=33)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_load_views needs a GPU"
    ru = importlib.import_module("make-it-3d_b200.nerf.refine_utils")
    S = a.size
    with tempfile.TemporaryDirectory() as tmp:
        gt, rgb_f, depth_f, mask_f, poses, K = vr.make_mvimg(os.path.join(tmp, "mvimg"), a.views, S, seed=0)
        outdir = os.path.join(tmp, "refine")
        os.makedirs(outdir)
        args = (gt, rgb_f, depth_f, mask_f, poses, S, S, K, 2, 8, outdir, "cuda")
        ru.load_views(*args)                                                 # warm-up: module load, allocator
        walls = []
        for _ in range(a.reps):
            np.random.seed(0)                                                # the npoint subsample draws from numpy's global RNG
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = ru.load_views(*args)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ru.load_views(*args)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                t = getattr(e, "device_time_total", None)
                t = e.cuda_time_total if t is None else t
                kern[e.key[:90]] = {"ms": round(t / 1e3, 4), "calls": e.count}
        # the oracle decodes the same files' arrays with cv2 and runs on the host
        import cv2
        dec = lambda fs, fl: [cv2.imread(f, fl) for f in fs]
        depths, masks = dec(depth_f, cv2.IMREAD_UNCHANGED), dec(mask_f, cv2.IMREAD_UNCHANGED)
        rgbs = [im[..., ::-1] for im in dec(rgb_f, cv2.IMREAD_UNCHANGED)]
        np.random.seed(0)
        t0 = time.perf_counter()
        ref = vr.load_views_ref(gt, depths, masks, rgbs, poses, S, S, K, 2, 8)
        t_ref = time.perf_counter() - t0
    same_counts = all(x.shape == y.shape for x, y in zip(out, ref))
    agree = same_counts and all(float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-30)) <= tol if x.size else True
                                for x, y, tol in zip(out, ref, (1e-12, 1e-6, 1e-12, 1e-6)))
    res = {"card": card(), "views": a.views, "size": S, "native_wall_ms": [round(w * 1e3, 2) for w in walls],
           "native_wall_ms_min": round(min(walls) * 1e3, 2), "kernel_ms_total": round(sum(v["ms"] for v in kern.values()), 3),
           "kernels": dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms"])),
           "oracle_host_s": round(t_ref, 2), "host_cores": os.cpu_count(), "torch_threads": torch.get_num_threads(),
           "points_cano": int(out[0].shape[0]), "points_novel": int(out[2].shape[0]),
           "oracle_points": [int(ref[0].shape[0]), int(ref[2].shape[0])], "native_matches_oracle": bool(agree)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
