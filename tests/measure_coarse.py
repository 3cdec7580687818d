"""Time one coarse iteration (nerf/coarse.py CoarseStep.step) against the reference iteration restated on the same drop-ins
(tests/test_coarse_gpu.py::eager_train_step, two render backwards on SDS iterations), alternated in one process, for front, SDS
(t = 500) and denoise (t = 300) iterations at 128 x 128.  The field is bench.py's (sphere occupancy, "trained-like" table); the
guidance holds seeded full-size SD-2.0 weights and CLIP seeded ViT-B/16 weights.  Each time is a host clock around `reps` iterations
ending in a device synchronise.  Prints the card name and power limit read in the same run.
    python tests/measure_coarse.py [--reps 10] [--rounds 3] [--out coarse.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_coarse_gpu as tc  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_coarse.py needs a GPU"
    dev = "cuda"
    g = torch.Generator().manual_seed(0)
    sc = tc.build_scene(full_size_sd=True)
    opt = tc.make_opt()
    cs = tc.make_step(sc, opt)
    model_b = tc.make_model(opt)
    adan_b = tc.make_adan(model_b)
    bg = torch.tensor([0.3, 0.6, 0.2], device=dev)
    light = torch.tensor([0.0, 0.6, 0.8], device=dev)
    noise, eps = torch.randn(1, 4, 64, 64, generator=g).to(dev), torch.randn(1, 4, 64, 64, generator=g).to(dev)
    cases = {"front": (tc.view(0.0, front=True), None), "sds": (tc.view(40.0), 500), "denoise": (tc.view(-50.0), 300)}
    native = lambda c: (lambda: cs.step(c[0], 2000, shading="albedo", bg_color=bg, t=c[1], noise=noise, eps_posterior=eps, light_d=light))
    eager = lambda c: (lambda: tc.eager_train_step(model_b, adan_b, opt, sc, c[0], 2000, "albedo", bg, light, t=c[1], noise=noise,
                                                   eps_posterior=eps))
    for c in cases.values():                      # warm-up: engine planning, graph capture, allocator
        for _ in range(2):
            native(c)()
            eager(c)()
    res = {k: {"native_ms": [], "eager_ms": []} for k in cases}
    for _ in range(a.rounds):
        for k, c in cases.items():
            res[k]["native_ms"].append(timed(native(c), a.reps))
            res[k]["eager_ms"].append(timed(eager(c), a.reps))
    out = {"card": card(), "hw": tc.HW, "reps": a.reps, "rounds": a.rounds}
    for k, v in res.items():
        out[k] = {"native_ms": statistics.median(v["native_ms"]), "eager_ms": statistics.median(v["eager_ms"]),
                  "native_all": v["native_ms"], "eager_all": v["eager_ms"]}
    # the loss kernel on its own (front view: all four launches, then the backward)
    d = cases["front"][0]
    out_r = cs.model.render(d["rays_o"], d["rays_d"], depth_scale=d["depth_scale"], bg_color=bg, perturb=True, force_all_rays=True,
                            light_d=light, **{k: v for k, v in vars(opt).items() if k in ("max_steps", "dt_gamma")})
    img, dep, ws = (out_r[k].detach().requires_grad_() for k in ("image", "depth", "weights_sum"))

    def losses():
        terms, pred512, _ = tc.co.coarse_losses(img, dep, ws, tc.HW, tc.HW, cs.ref, bg, cs.prior, cs.mask, True)
        terms.sum().backward()
    out["loss_kernels_fwd_bwd_ms"] = timed(losses, 50)
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
