"""Time one refine iteration (nerf/refine.py RefineStep.step) against the reference loop body restated on the same drop-ins
(tests/test_refine_gpu.py::eager_iteration), alternated in one process, for front, SDS (t = 500) and denoise (t = 300) iterations, plus
the final render per view.  The cloud comes from a seeded synthetic 33-view 800^2 mvimg folder (oracle/views_ref.make_mvimg) through
load_views; every model holds seeded full-size weights (SD-2.0 guidance, CLIP ViT-B/16, VGG19 contextual loss, the gated U-Net).
Each time is a host clock around `reps` iterations ending in a device synchronise.  Prints the card name and power limit read in
the same run.
    python tests/measure_refine.py [--views 33] [--reps 5] [--out refine.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import views_ref as vr  # noqa: E402

import test_refine_gpu as tr  # noqa: E402


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
    ap.add_argument("--views", type=int, default=33)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_refine.py needs a GPU"
    S = tr.S
    ru, rf = tr.ru, tr.rf
    with tempfile.TemporaryDirectory() as tmp:
        folder = os.path.join(tmp, "mvimg")
        gt, rgb_f, depth_f, mask_f, poses, K = vr.make_mvimg(folder, a.views, S, seed=0)
        vc, cc, vn, cn = ru.load_views(gt, rgb_f, depth_f, mask_f, poses, S, S, K, 2, 8, folder, "cuda")
    dev = "cuda"
    gt_t = torch.tensor(gt, dtype=torch.float32).permute(2, 0, 1)[None].contiguous().to(dev)
    mask = (gt_t.amax(1, keepdim=True) > 0.05).float()
    guidance = tr.sd_mod.StableDiffusion(dev)                           # seeded full-size SD-2.0
    clip, cx = tr.clip_mod.CLIP(dev), tr.cx_mod.ContextualLoss(device=dev)
    gen = torch.Generator().manual_seed(0)
    text_z = torch.randn(2, 77, 1024, generator=gen).to(dev)
    tokens = torch.randint(1, 49000, (1, 77), generator=gen).to(dev)
    rs = rf.RefineStep(vc, cc, vn, cn, K, tr._unet(0), cx, clip, guidance, text_z, gt_t, mask, tokens, seed=0)
    e = tr.Eager(rs, tr._unet(0))
    w_front = tr._w2c(dict(poses=poses), None)
    w_side = tr._w2c(dict(poses=poses), 3)
    g = torch.Generator().manual_seed(1)
    noise, eps = torch.randn(1, 4, 64, 64, generator=g).to(dev), torch.randn(1, 4, 64, 64, generator=g).to(dev)
    cases = {"front": (w_front, True, {}), "sds": (w_side, False, dict(t=500, noise=noise, eps_posterior=eps)),
             "denoise": (w_side, False, dict(t=300, noise=noise, eps_posterior=eps))}
    native = lambda c: (lambda: rs.step(c[0], c[1], **c[2]))
    eager = lambda c: (lambda: tr.eager_iteration(e, c[0], c[1], guidance, text_z, clip, cx, gt_t, mask, tokens, **c[2]))
    for c in cases.values():                      # warm-up: engine planning, graph capture, allocator
        for _ in range(2):
            native(c)()
            eager(c)()
    res = {k: {"native_ms": [], "eager_ms": []} for k in cases}
    for _ in range(a.rounds):
        for k, c in cases.items():
            res[k]["native_ms"].append(timed(native(c), a.reps))
            res[k]["eager_ms"].append(timed(eager(c), a.reps))
    render_ms = timed(lambda: rs.render(w_side), 10)
    out = {"card": card(), "points": int(rs.points.shape[0]), "p_cano": rs.p_cano, "p_novel": rs.p_novel, "reps": a.reps,
           "rounds": a.rounds, "render_ms_per_view": render_ms}
    for k, v in res.items():
        out[k] = {"native_ms": statistics.median(v["native_ms"]), "eager_ms": statistics.median(v["eager_ms"]),
                  "native_all": v["native_ms"], "eager_all": v["eager_ms"]}
    # Adam and image-loss kernels on their own: bytes they must move over their time
    P = rs.points.shape[0]
    n_unet = sum(p.numel() for p in rs.unet_params)
    adam_bytes = 4 * (7 * (P * 19 + n_unet) + P * 3)         # read p, g, m, v; write p, m, v; read the colour origins
    out["adam_ms"] = timed(lambda: rs.opt.step(), 20)
    out["adam_GBps"] = adam_bytes / out["adam_ms"] / 1e6
    _, w0 = ru.render_point_weights(rs.all_v, rs.points.detach(), S, S, rs.K[0], w_side, [S, S], rf.RADIUS, rf.PPP)
    pred = torch.rand(1, 3, S, S, device=dev)
    img_bytes = 4 * (S * S * 8 + 3 * S * S * 2 + S * S * 3)  # weights, pred, gt, mask; coverage + dilation written
    out["image_losses_ms"] = timed(lambda: rf.image_losses(pred, w0, gt_t, mask, True), 50)
    out["image_losses_GBps"] = img_bytes / out["image_losses_ms"] / 1e6
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
