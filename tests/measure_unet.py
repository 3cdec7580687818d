"""Times the refine stage's gated U-Net on the GPU (python tests/measure_unet.py [--out FILE] [--iters K] [--size S]).

Settings: N = 1, inputs at S^2 / (S/2)^2 / (S/4)^2 (800 by default, the refine size), graph replay on, warm-up, then timed calls.  Legs:
  train_fwd_bwd   train-mode forward + backward (input and weight gradients)        (nerf/utils.py:863, 893)
  fwd_only        train-mode forward under torch.no_grad()
  eval_fwd        eval-mode forward under torch.no_grad()                           (nerf/utils.py:937)
  oracle_default  the A/B arm: oracle/unet_ref.py in eager PyTorch, forward + backward, cuDNN defaults (TF32 convs, how the reference
                  runs the module)
  oracle_fp32     the same with TF32 off
Reported: ms per call (CUDA events), the algorithmic conv FLOP of one forward and the FLOP the direct-conv kernels execute (output
channels padded to 16, input channels to 8, pixels to 32 x 32 tiles), a per-kernel breakdown from one separate profiled call
(torch.profiler), and the card's name and power limit read in the same run.  Lives under tests/ because it imports the oracle."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import unet_ref  # noqa: E402

# (cin, cout, k, level) of every conv of one forward; a gated block's conv_f and conv_m run as one conv with 2c outputs
CONVS = [(19, 32, 3, 0), (16, 26, 3, 1), (32, 90, 3, 2), (64, 32, 3, 1), (64, 64, 3, 1), (32, 16, 3, 0), (32, 32, 3, 0), (16, 3, 1, 0)]


def flops(H, W):
    alg = exe = 0
    for cin, cout, k, lvl in CONVS:
        h, w = H >> lvl, W >> lvl
        alg += 2 * cin * cout * k * k * h * w
        if k == 3:
            exe += 2 * (-(-cin // 8) * 8) * (-(-cout // 16) * 16) * 9 * (-(-h // 32) * 32) * (-(-w // 32) * 32)
        else:
            exe += 2 * cin * cout * h * w
    return alg, exe


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
    assert torch.cuda.is_available(), "measure_unet.py needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    H = W = args.size
    torch.manual_seed(0)
    net = um.UNet(num_input_channels=3 + 16).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    xs = [torch.rand(1, 19, H >> i, W >> i, device="cuda", generator=g).requires_grad_(True) for i in range(3)]
    w = torch.randn(1, 3, H, W, device="cuda", generator=g)

    def train_fwd_bwd():
        for t in xs + list(net.parameters()):
            t.grad = None
        (net(xs) * w).sum().backward()

    def fwd_only():
        with torch.no_grad():
            net(xs)

    def eval_fwd():
        net.eval()
        with torch.no_grad():
            net(xs)
        net.train()

    p = {k: (v.detach().clone().requires_grad_(True) if k in unet_ref.param_names() else v.detach().clone()) for k, v in net.state_dict().items()}

    def oracle():
        xr = [x.detach().requires_grad_(True) for x in xs]
        (unet_ref.unet(xr, p) * w).sum().backward()

    res = {"card": card, "H": H, "W": W, "iters": args.iters}
    res["train_fwd_bwd_ms"] = timed(train_fwd_bwd, 5, args.iters)
    res["fwd_only_ms"] = timed(fwd_only, 5, args.iters)
    res["eval_fwd_ms"] = timed(eval_fwd, 5, args.iters)
    res["graph_replays"] = net.engines[(1, H, W, xs[0].device)].graph_replays()
    alg, exe = flops(H, W)
    res["fwd_gflop_algorithmic"] = alg / 1e9
    res["fwd_gflop_executed"] = exe / 1e9
    res["train_gflop_algorithmic"] = 3 * alg / 1e9       # forward, input gradient, weight gradient
    res["achieved_tflops_train"] = 3 * alg / (res["train_fwd_bwd_ms"] * 1e-3) / 1e12
    res["achieved_tflops_fwd"] = alg / (res["fwd_only_ms"] * 1e-3) / 1e12
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train_fwd_bwd()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA":
            kern[e.key] = kern.get(e.key, 0.0) + e.self_device_time_total / 1e3
    res["kernel_ms_profiled"] = sum(kern.values())
    res["kernels_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:12])
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
