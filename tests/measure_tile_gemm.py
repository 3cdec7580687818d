"""Where the tile kernel's time goes in one G = 1 SDS step, launch by launch, against the operand bytes it pulls from L2.

Builds bench.py's models (bench.build_models, seed 0) and runs the SD lists of one SDS step (VAE encode, U-Net x2 + CFG + SDS,
encode backward) with the engine's per-launch event bracket on (mi3d_sd_profile: plain launches, an event pair around every tile
launch).  --rounds rounds of enough steps to fill --window seconds each; a launch's time is its mean over the steps of a round,
then the median over the rounds.  Per launch it reports M N K, block_n, splits, conv, ms, the achieved TFLOP/s, the L2 -> SM
operand bytes computed from the tile plan and the implied bytes/s, then a summary per shape class.

Operand bytes (computed from the tile plan, not measured): every (tile, k-block) loads one A box (128 rows x 128 B) and its B tile
(block_n rows x 128 B) from L2; split-K work items partition a tile's k-blocks.  bytes/s = those bytes over the launch's time.

As a yardstick only, the largest shapes of each class are also timed through torch: torch.matmul on fp16 [M,K] x [K,N] (cuBLAS)
and torch.nn.functional.conv2d in channels_last fp16 (cuDNN), plain launches, >= --window s windows, medians of --rounds.
Prints the card name and power limit read in the same run, the tables, then one JSON line.

  python tests/measure_tile_gemm.py [--rounds 5] [--window 1.0] [--torch-shapes 3]
"""
import argparse
import collections
import ctypes as C
import importlib
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

A_BOX = 128 * 128                       # BLOCK_M rows x BLOCK_K fp16
VAE_M = {512 * 512: 512, 256 * 256: 256, 128 * 128: 128, 64 * 64: 64}          # G = 1: VAE pixels per image -> width
UNET_M = {2 * 64 * 64: 0, 2 * 32 * 32: 1, 2 * 16 * 16: 2, 2 * 8 * 8: 3}        # U-Net batch 2 (CFG): pixels -> level


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else torch.cuda.get_device_name()


def shape_class(M, N, K, splits, conv):
    if splits > 1:
        return "split-K"
    if conv == 1:
        if M in VAE_M:
            return f"VAE conv {VAE_M[M]}"
        if M in UNET_M:
            return f"U-Net conv level {UNET_M[M]}"
        return "other conv"
    if K % 9 == 0:
        return "stride-2 im2col GEMM"
    return "U-Net / VAE linear"


def operand_bytes(M, N, K, bn, batch):
    """L2 -> SM bytes of one launch from its tile plan (see the module docstring)"""
    return (M + 127) // 128 * (N // bn) * batch * (K // 64) * (A_BOX + bn * 128)


def conv_geometry(M, K):
    """(images, H = W, Cin) of an implicit 3x3 conv launch of the G = 1 step"""
    if M in VAE_M:
        return 1, VAE_M[M], K // 9
    return 2, int(math.isqrt(M // 2)), K // 9


def window_ms(fn, seconds, rounds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    n = max(3, math.ceil(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
    out = []
    for _ in range(rounds):
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / n)
    return statistics.median(out)


def torch_ms(M, N, K, conv, seconds, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    if conv == 1:
        imgs, hw, cin = conv_geometry(M, K)
        x = torch.randn(imgs, cin, hw, hw, device="cuda", generator=g).half().to(memory_format=torch.channels_last)
        w = (torch.randn(N, cin, 3, 3, device="cuda", generator=g) * 0.05).half().to(memory_format=torch.channels_last)
        return window_ms(lambda: torch.nn.functional.conv2d(x, w, padding=1), seconds, rounds)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    b = (torch.randn(K, N, device="cuda", generator=g) * 0.05).half()
    return window_ms(lambda: torch.matmul(a, b), seconds, rounds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--torch-shapes", type=int, default=3, help="torch yardstick: this many largest distinct shapes per class")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_tile_gemm.py needs a GPU")
    L = importlib.import_module("make-it-3d_b200._lib")
    name = card()
    print(f"card: {name}", flush=True)
    device = torch.device("cuda", 0)
    _, guidance = bench.build_models(device, seed=0)
    gen = torch.Generator().manual_seed(0)
    rgb = torch.rand(1, 3, bench.HW, bench.HW, generator=gen).to(device).requires_grad_()
    ctx = torch.randn(2, 77, 1024, generator=gen).to(device)
    noise = torch.randn(1, 4, 64, 64, generator=gen).to(device)
    eps = torch.randn(1, 4, 64, 64, generator=gen).to(device)
    guidance._t.fill_(450)

    def sds_step():
        rgb.grad = None
        lat = guidance.encode_imgs(rgb, eps)
        _, grad = guidance.unet_sds(lat, noise, guidance._t, ctx, 10.0)
        lat.backward(gradient=grad)

    step_ms = window_ms(sds_step, 0.3, 1)                 # graph replay: the pipeline's own per-step time
    steps = max(3, math.ceil(args.window * 1e3 / step_ms))
    per_round = []
    with tempfile.TemporaryDirectory(prefix="mi3d_tile_") as tmp:
        for r in range(args.rounds):
            L.check(L.lib().mi3d_sd_profile(guidance.engine.h, C.c_int(1), None, None), "sd_profile")
            for _ in range(steps):
                sds_step()
            torch.cuda.synchronize()
            ms, n = C.c_float(0), C.c_int(0)
            path = os.path.join(tmp, f"round{r}.txt")
            L.check(L.lib().mi3d_sd_profile_dump(guidance.engine.h, C.c_int(0), C.byref(ms), C.byref(n), path.encode()), "sd_profile_dump")
            rows = [ln.split() for ln in open(path).read().splitlines() if ln.strip()]
            per = len(rows) // steps
            acc = []
            for i in range(per):
                f = rows[i]
                acc.append(((int(f[0]), int(f[1]), int(f[2]), int(f[3]), int(f[4]), int(f[5]), int(f[6])),
                            sum(float(rows[s * per + i][8]) for s in range(steps)) / steps))
            per_round.append(acc)
    launches = []
    for i, (key, _) in enumerate(per_round[0]):
        M, N, K, bn, splits, conv, batch = key
        if conv == 2:
            continue                                          # the fused attention, not the tile kernel
        ms = statistics.median(rr[i][1] for rr in per_round)
        flop = 2.0 * M * N * K * batch
        by = operand_bytes(M, N, K, bn, batch)
        launches.append(dict(M=M, N=N, K=K, block_n=bn, splits=splits, conv=conv, batch=batch, ms=round(ms, 4),
                             tflops=round(flop / ms / 1e9, 1), operand_gb=round(by / 1e9, 4), operand_tbs=round(by / ms / 1e9, 2),
                             cls=shape_class(M, N, K, splits, conv), flop=flop, bytes=by))
    print(f"\n{'M':>7} {'N':>5} {'K':>6} {'bn':>4} {'spl':>3} {'conv':>4} {'ms':>8} {'TFLOP/s':>8} {'opnd GB':>8} {'TB/s':>6}  class")
    for x in launches:
        print(f"{x['M']:>7} {x['N']:>5} {x['K']:>6} {x['block_n']:>4} {x['splits']:>3} {x['conv']:>4} {x['ms']:>8.4f} {x['tflops']:>8.1f} "
              f"{x['operand_gb']:>8.4f} {x['operand_tbs']:>6.2f}  {x['cls']}")
    classes = collections.OrderedDict()
    for x in sorted(launches, key=lambda x: x["cls"]):
        c = classes.setdefault(x["cls"], dict(launches=0, ms=0.0, flop=0.0, bytes=0.0))
        c["launches"] += 1; c["ms"] += x["ms"]; c["flop"] += x["flop"]; c["bytes"] += x["bytes"]
    # torch yardstick on the largest distinct shapes of each class
    yard = []
    for cls in classes:
        shapes = collections.OrderedDict()
        for x in launches:
            if x["cls"] == cls and x["batch"] == 1:
                k = (x["M"], x["N"], x["K"], x["conv"])
                shapes.setdefault(k, []).append(x["ms"])
        for (M, N, K, conv), ts in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2])[:args.torch_shapes]:
            t_ms = torch_ms(M, N, K, conv, args.window, args.rounds)
            ours = statistics.median(ts)
            yard.append(dict(cls=cls, M=M, N=N, K=K, conv=conv, ours_ms=round(ours, 4), ours_tflops=round(2.0 * M * N * K / ours / 1e9, 1),
                             torch=("cudnn conv2d channels_last" if conv == 1 else "cublas matmul"), torch_ms=round(t_ms, 4),
                             torch_tflops=round(2.0 * M * N * K / t_ms / 1e9, 1)))
    print(f"\n{'class':<24} {'n':>3} {'ms':>8} {'TFLOP/s':>8} {'opnd GB':>8} {'TB/s':>6}")
    summary = {}
    for cls, c in classes.items():
        summary[cls] = dict(launches=c["launches"], ms=round(c["ms"], 3), tflops=round(c["flop"] / c["ms"] / 1e9, 1),
                            operand_gb=round(c["bytes"] / 1e9, 3), operand_tbs=round(c["bytes"] / c["ms"] / 1e9, 2))
        s = summary[cls]
        print(f"{cls:<24} {s['launches']:>3} {s['ms']:>8.3f} {s['tflops']:>8.1f} {s['operand_gb']:>8.3f} {s['operand_tbs']:>6.2f}")
    print(f"\n{'class':<24} {'M':>7} {'N':>5} {'K':>6} {'ours ms':>8} {'TFLOP/s':>8} {'torch ms':>8} {'TFLOP/s':>8}")
    for y in yard:
        print(f"{y['cls']:<24} {y['M']:>7} {y['N']:>5} {y['K']:>6} {y['ours_ms']:>8.4f} {y['ours_tflops']:>8.1f} {y['torch_ms']:>8.4f} {y['torch_tflops']:>8.1f}")
    tot_ms = sum(x["ms"] for x in launches)
    res = dict(metric="tile kernel launches of one G = 1 SDS step: time, TFLOP/s, computed L2 -> SM operand bytes", card=name,
               sds_step_ms_graph_replay=round(step_ms, 3), steps_per_round=steps, rounds=args.rounds,
               tile_launches=len(launches), tile_ms=round(tot_ms, 3),
               tile_tflops=round(sum(x["flop"] for x in launches) / tot_ms / 1e9, 1), classes=summary, torch_yardstick=yard,
               launches=[{k: v for k, v in x.items() if k not in ("flop", "bytes")} for x in launches])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
