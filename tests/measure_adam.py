"""Time `optimizer.Adam` (csrc/adam.cu) at the coarse stage's shapes, and a coarse iteration with it.

1. The optimiser step alone on a real `NeRFNetwork(opt).get_params(1e-3)` (12 196 240 table floats plus the MLP, about 1 % non-zero
   table gradients): the fused path (mi3d_sumsq + one mi3d_adam_step per tensor) against `torch.nn.utils.clip_grad_norm_(params, 10)`
   + torch.optim.Adam's foreach step.  Bytes/s use the step's nominal traffic of 36 B per element: the norm pass reads g (4 B), the
   update reads and writes p g m v (32 B).
2. A front and an SDS (t = 500) coarse iteration at 128 x 128 (`CoarseStep.step`, seeded full-size SD-2.0 and CLIP as in
   tests/measure_coarse.py) with Adam against Adan.

Times come from CUDA events around windows of at least `--window` seconds each, after a warm-up; the two arms alternate window by
window for `--rounds` rounds and the median per-step time is reported.  A step of part 1 is short enough that its wall time is the
host's launch time, so part 1 also reports the GPU time of its kernels and copies (torch.profiler, 20 steps, median of `--rounds`).
The card name and power limit are read in the same run.
    python tests/measure_adam.py [--rounds 5] [--window 1.0] [--out adam.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_coarse_gpu as tc  # noqa: E402
import test_adam_gpu as ta  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def window_ms(fn, seconds):
    """mean ms per call over a window of at least `seconds`, by CUDA events (the batch size grows until a window is long enough)"""
    n = 1
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= seconds * 1e3:
            return ms / n
        n = max(n * 2, int(n * seconds * 1e3 / max(ms, 1e-3) * 1.1) + 1)


def device_ms(fn, n):
    """GPU time per call: the summed durations of the kernels and copies torch.profiler records over n calls (the wall time of a
    step this small is the host's launch time)"""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return us * 1e-3 / n


def alternate(arms, rounds, seconds):
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(window_ms(fn, seconds))
    return {k: dict(median_ms=statistics.median(v), all_ms=v) for k, v in times.items()}


def optimiser_step(a):
    pa, mine, pb, ref = ta.make_arms(ta.CLIP)
    gs = ta.grads(pa, 0, 1.0)
    ta.set_grads(pa, gs)
    ta.set_grads(pb, gs)
    n = sum(p.numel() for p in pa)
    arms = {"fused": mine.step, "torch_clip_foreach_adam": lambda: ta.torch_step(pb, ref, ta.CLIP)}
    for fn in arms.values():                       # warm-up: state, scratch, foreach kernels
        for _ in range(5):
            fn()
    res = alternate(arms, a.rounds, a.window)
    nbytes = 36 * n
    for k, r in res.items():
        r["device_ms"] = statistics.median(device_ms(arms[k], 20) for _ in range(a.rounds))
        r["GB_per_s_wall"] = nbytes / (r["median_ms"] * 1e-3) / 1e9
        r["GB_per_s_device"] = nbytes / (r["device_ms"] * 1e-3) / 1e9
    return dict(elements=n, nominal_bytes=nbytes, **res)


def coarse_iterations(a):
    dev = "cuda"
    g = torch.Generator().manual_seed(0)
    sc = tc.build_scene(full_size_sd=True)
    opt = tc.make_opt()
    steps = {}
    for name, make in (("adam", ta.make_adam), ("adan", tc.make_adan)):
        model = tc.make_model(opt)
        steps[name] = tc.co.CoarseStep(model, sc["guidance"], sc["clip"], make(model), opt, sc["ref"], sc["prior"], sc["depth_mask"],
                                       sc["text_z"], sc["tokens"])
    bg = torch.tensor([0.3, 0.6, 0.2], device=dev)
    light = torch.tensor([0.0, 0.6, 0.8], device=dev)
    noise, eps = torch.randn(1, 4, 64, 64, generator=g).to(dev), torch.randn(1, 4, 64, 64, generator=g).to(dev)
    out = {}
    for case, (data, t) in {"front": (tc.view(0.0, front=True), None), "sds": (tc.view(40.0), 500)}.items():
        arms = {k: (lambda cs=cs: cs.step(data, 2000, shading="albedo", bg_color=bg, t=t, noise=noise, eps_posterior=eps, light_d=light))
                for k, cs in steps.items()}
        for fn in arms.values():
            for _ in range(3):
                fn()
        out[case] = alternate(arms, a.rounds, a.window)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_adam.py needs a GPU"
    res = dict(card=card(), optimiser_step=optimiser_step(a), coarse_iteration_128=coarse_iterations(a))
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
