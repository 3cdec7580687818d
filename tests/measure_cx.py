"""Times the refine stage's contextual loss on the GPU (python tests/measure_cx.py [--out FILE] [--iters K]).

Settings: N = 1, 800 x 800 (the refine size), relu5_4, seeded weights, graph replay on, warm-up, then timed calls.  Legs:
  fwd_bwd        ContextualLoss(x, y) + backward into x          (nerf/utils.py:455-457, 882)
  fwd_only       the same under torch.no_grad()
  oracle_default the A/B arm: oracle/cx_ref.py in eager fp32 PyTorch, forward + backward, cuDNN defaults (TF32 convs, how the
                 reference runs the package)
  oracle_fp32    the same with TF32 off
Reported: ms per call (CUDA events), the tile-GEMM share of the engine's time (torch.profiler, kernels named k_tc_gemm_vgg, one
separate profiled call), achieved TFLOP/s from the algorithmic count (777 600 * H * W FLOP per image pass: 2 images forward, 1 image
input-gradient), and the card's name and power limit read in the same run.  Lives under tests/ because it imports the oracle."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cx_ref  # noqa: E402

FLOP_PER_PIXEL = 777_600      # VGG19 conv1_1 .. conv5_4, 2 * MACs per input pixel


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--size", type=int, default=800)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_cx.py needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cl = importlib.import_module("make-it-3d_b200.nerf.contextual_loss")
    H = W = args.size
    params = cx_ref.seeded_params(0, "cuda")
    m = cl.ContextualLoss(device="cuda", state_dict=params)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(1, 3, H, W, device="cuda", generator=g)
    y = 0.3 * x + 0.7 * torch.rand(1, 3, H, W, device="cuda", generator=g)
    xg = x.clone().requires_grad_(True)

    def fwd_bwd():
        xg.grad = None
        m(xg, y).backward()

    def fwd_only():
        with torch.no_grad():
            m(x, y)

    def oracle():
        xr = x.clone().requires_grad_(True)
        cx_ref.contextual_loss(xr, y, params).backward()

    res = {"card": card, "H": H, "W": W, "iters": args.iters}
    res["fwd_bwd_ms"] = timed(fwd_bwd, 5, args.iters)
    res["fwd_only_ms"] = timed(fwd_only, 5, args.iters)
    res["graph_replays"] = m.engine(1, H, W).graph_replays()
    # tile-GEMM share of one forward + backward
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fwd_bwd()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA":
            kern[e.key] = kern.get(e.key, 0.0) + e.self_device_time_total / 1e3
    total = sum(kern.values())
    tc = sum(v for k, v in kern.items() if "k_tc_gemm_vgg" in k)
    res["kernel_ms_profiled"] = total
    res["tile_gemm_ms"] = tc
    res["tile_gemm_share"] = tc / total if total else None
    res["top_kernels_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:8])
    flop_call = FLOP_PER_PIXEL * H * W * 3        # x and y forward, x input gradient
    res["tflop_per_call"] = flop_call / 1e12
    res["achieved_tflops_fwd_bwd"] = flop_call / (res["fwd_bwd_ms"] * 1e-3) / 1e12
    res["achieved_tflops_tile_gemm"] = flop_call / (tc * 1e-3) / 1e12 if tc else None
    res["achieved_tflops_fwd_only"] = FLOP_PER_PIXEL * H * W * 2 / (res["fwd_only_ms"] * 1e-3) / 1e12
    for name, tf32 in (("oracle_default", True), ("oracle_fp32", False)):
        torch.backends.cudnn.allow_tf32 = tf32
        res[name + "_ms"] = timed(oracle, 2, max(5, args.iters // 3))
    torch.backends.cudnn.allow_tf32 = True
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
