"""Time the DPT-Hybrid depth model (nerf/dpt.py) at the one shape the reference runs it ([1, 3, 384, 384]), seeded weights.  A/B arms
on the same card: the fp32 oracle (oracle/dpt_ref.py) in eager PyTorch, and transformers' DPTForDepthEstimation at the DPT-Hybrid
configuration in fp32 and with TF32 matmuls / convs.  FLOPs are counted from shapes (torch.utils.flop_counter over the oracle).
Prints one JSON line (card name and power limit read in the same run).

  python tests/measure_dpt.py [--calls 30] [--warmup 5]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpt_ref  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else torch.cuda.get_device_name()


def time_calls(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def flops(p, x):
    """(conv + linear GFLOP, attention-product GFLOP) of one forward, counted from shapes"""
    from torch.utils.flop_counter import FlopCounterMode
    with FlopCounterMode(display=False) as fc, torch.no_grad():
        dpt_ref.forward(p, x)
    total = fc.get_total_flops()
    attn = 2 * 2 * 12 * 577 * 577 * 64 * 12                    # Q K^T and P V, 12 heads x 12 blocks
    return (total - attn) / 1e9, attn / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dpt = importlib.import_module("make-it-3d_b200.nerf.dpt")
    sd = dpt_ref.default_init(seed=3)
    model = dpt.DPTDepthModel(state_dict=sd)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 3, 384, 384, generator=g).clamp(-1, 1).cuda()
    line = {"card": card(), "shape": [1, 3, 384, 384]}
    line["engine_ms"] = time_calls(lambda: model.forward(x), args.calls, args.warmup)
    p = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        line["oracle_fp32_ms"] = time_calls(lambda: dpt_ref.forward(p, x), args.calls, args.warmup)
    gf, ga = flops(p, x)
    line["gflop_conv_linear"], line["gflop_attention"] = round(gf, 2), round(ga, 2)
    line["engine_tflops"] = round((gf + ga) / line["engine_ms"], 2)
    try:
        import transformers
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_dpt_oracle_cpu import _hf_config
        hf = transformers.DPTForDepthEstimation(_hf_config()).eval().cuda()
        with torch.no_grad():
            line["transformers_fp32_ms"] = time_calls(lambda: hf(pixel_values=x), args.calls, args.warmup)
            torch.backends.cudnn.allow_tf32 = True
            torch.backends.cuda.matmul.allow_tf32 = True
            line["transformers_tf32_ms"] = time_calls(lambda: hf(pixel_values=x), args.calls, args.warmup)
    except ImportError:
        line["transformers_fp32_ms"] = line["transformers_tf32_ms"] = None
    print(json.dumps(line))


if __name__ == "__main__":
    main()
