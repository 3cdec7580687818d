"""Time the sampler (produce_latents on mi3d_sd_sample) at 512 x 512, 50 steps, guidance 7.5, in one run, for seeded full-size SD-2.0
and SD-1.5 topologies:

* produce_latents, one prompt (CUDA events around the call; graph replay on);
* unet_sds timed 50 times back to back in the same run: the sampler should cost 50 U-Net passes plus element-wise work, so
  (produce_latents - 50 x unet_sds) / 50 is the per-step overhead;
* the eager comparison arm: the reference's loop (nerf/sd.py:183-197) on the fp32 oracle U-Net under torch.autocast('cuda');
* decode_latents at 512.

Prints the card name and power limit, then one JSON line.

  python tests/measure_sample.py [--reps 3] [--steps 50]
"""
import argparse
import importlib
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import sd_sample_ref  # noqa: E402
from measure_sd15 import card  # noqa: E402
from oracle import sd_ref  # noqa: E402


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts), max(ts)


def eager_loop(unet, ctx, lat, steps):
    """nerf/sd.py:183-197 as the reference runs it: autocast fp16, one batch-2 U-Net call per step, DDIMScheduler.step on the output"""
    ts = sd_sample_ref.ddim_timesteps(steps)
    alphas = sd_ref.alphas_cumprod().cuda()
    with torch.no_grad(), torch.autocast("cuda"):
        for t in ts:
            out = unet(torch.cat([lat] * 2), torch.tensor([int(t)], device="cuda"), ctx)
            un, tx = out.chunk(2)
            lat = sd_sample_ref.ddim_step_ref(tx + 7.5 * (tx - un), int(t), lat, steps, alphas=alphas)
    return lat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    print(card(), flush=True)
    res = {"card": card(), "steps": args.steps, "size": 512}
    for name, ucfg, ocfg in (("sd2.0", sdm.sd20_unet_cfg(), sd_ref.sd20_unet_config()),
                             ("sd1.5", sdm.sd15_unet_cfg(), None)):
        g = sdm.StableDiffusion("cuda", unet_cfg=ucfg)                # seeded weights at the checkpoint's topology
        gen = torch.Generator().manual_seed(0)
        lat = torch.randn(1, 4, 64, 64, generator=gen).cuda()
        ctx = torch.randn(2, 77, ucfg["cross_dim"], generator=gen).cuda()
        noise = torch.randn(1, 4, 64, 64, generator=gen).cuda()
        t = torch.tensor([437], dtype=torch.long, device="cuda")
        for _ in range(2):                                           # plan, capture the graphs, cache the schedule
            out = g.produce_latents(ctx, num_inference_steps=args.steps, latents=lat)
            g.unet_sds(lat, noise, t, ctx, 7.5)
            g.decode_latents(out)
        torch.cuda.synchronize()
        r = {}
        r["produce_latents_ms"] = timed(lambda: g.produce_latents(ctx, num_inference_steps=args.steps, latents=lat), args.reps)

        def sds_n():
            for _ in range(args.steps):
                g.unet_sds(lat, noise, t, ctx, 7.5)
        r["unet_sds_x%d_ms" % args.steps] = timed(sds_n, args.reps)
        r["decode_latents_ms"] = timed(lambda: g.decode_latents(out), args.reps)
        r["overhead_per_step_ms"] = (r["produce_latents_ms"][0] - r["unet_sds_x%d_ms" % args.steps][0]) / args.steps
        if ocfg is not None:
            unet = sd_sample_ref.UNet(ocfg).eval()
            unet.load_state_dict({k.replace("/", "."): v.detach().cpu() for k, v in g.unet.items()})
            unet = unet.cuda().requires_grad_(False)
            eager_loop(unet, ctx, lat, 2)
            r["eager_autocast_ms"] = timed(lambda: eager_loop(unet, ctx, lat, args.steps), max(1, args.reps - 1))
            del unet
        print(name, json.dumps(r), flush=True)
        res[name] = r
        del g
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
