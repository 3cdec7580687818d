"""Time a G-view coarse iteration (CoarseStep.step_views: one multi-view render, one SDS step at U-Net batch 2G) against G single-view
iterations (CoarseStep.step, U-Net batch 2), alternated in one process, for G = 1, 2, 4, 8 as far as memory allows.  The scene is
tests/measure_coarse.py's: 128 x 128 renders of bench.py's field, seeded full-size SD-2.0 guidance, seeded CLIP ViT-B/16.  Every view
takes the SDS branch (t = 500).  Iteration times are a host clock around `reps` iterations ending in a device synchronise; the SD parts
(unet_sds, VAE encode, encode backward) are CUDA events around `reps` calls on the G-view engine.  Also reports each G-view engine's
workspace.  Every timed window runs for at least --window seconds; medians over --rounds alternated windows, with the extremes.
Then whole epochs of `train_one_epoch(views_per_step=G)` on a reference-shaped shuffled loader (index % 4 == 0 front views), for the
time per item and the peak memory a run holds.  Prints the card name and power limit read in the same run.
    python tests/measure_multiview.py [--views 1 2 4 8] [--window 1.5] [--rounds 5] [--epoch-items 100] [--out multiview.json]
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_coarse_gpu as tc  # noqa: E402
from measure_coarse import card, timed  # noqa: E402

L = tc.sd_mod.L


def event_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def sd_parts(gd, G, reps):
    """ms per call of unet_sds, encode and encode backward on the G-view engine (CUDA events around reps calls)"""
    eng, hw = gd.views_engine(G), gd.vae_cfg["image_hw"] // 8
    g = torch.Generator().manual_seed(G)
    rgb = torch.rand(G, 3, tc.HW, tc.HW, generator=g).cuda()
    eps, noise = torch.randn(G, 4, hw, hw, generator=g).cuda(), torch.randn(G, 4, hw, hw, generator=g).cuda()
    te = torch.randn(2 * G, 77, gd.unet_cfg["cross_dim"], generator=g).cuda()
    lat, grad_rgb = torch.empty(G, 4, hw, hw, device="cuda"), torch.empty_like(rgb)
    t = torch.tensor([500], dtype=torch.long, device="cuda")
    lib = L.lib()

    def encode():
        with eng.on_stream():
            L.check(lib.mi3d_sd_encode(eng.h, L.ptr(rgb), C.c_int(tc.HW), C.c_int(tc.HW), L.ptr(eps), L.ptr(lat), L.stream()), "sd_encode")

    def encode_bwd():
        with eng.on_stream():
            L.check(lib.mi3d_sd_encode_backward(eng.h, L.ptr(lat), L.ptr(eps), C.c_int(tc.HW), C.c_int(tc.HW), L.ptr(grad_rgb), L.stream()),
                    "sd_encode_backward")
    parts = dict(unet_sds=lambda: gd.unet_sds(lat, noise, t, te, 10.0), encode=encode, encode_backward=encode_bwd)
    for fn in parts.values():                     # warm-up: graph capture on the third call
        for _ in range(3):
            fn()
    return {k: event_ms(fn, reps) for k, fn in parts.items()}


def epoch(cs, trainer_kw, views_per_step, n_items, seed):
    """one train_one_epoch over a loader shaped like the reference's (n_items shuffled, index % 4 == 0 front, provider.py), from
    global_step 2000 (every novel view guided); returns (ms per view, peak allocated GiB)"""
    co = tc.co
    g = torch.Generator().manual_seed(seed)
    order = torch.randperm(n_items, generator=g).tolist()
    loader = [tc.view(0.0 if i % 4 == 0 else 360.0 * i / n_items, front=i % 4 == 0, large=i % 7 == 3) for i in order]
    trainer = argparse.Namespace(global_step=2000, epoch=1, log=lambda *a: None, stats={"loss": []}, scheduler_update_every_step=True,
                                 fp16=False, ema=None, world_size=1, _coarse_step=cs, **trainer_kw)
    trainer.model.update_extra_state = lambda *a, **k: None          # the same field for both arms: no density-grid refresh
    cs.guidance_views = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    co.train_one_epoch(trainer, loader, views_per_step=views_per_step)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n_items, torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--window", type=float, default=1.5, help="seconds per timed window (at least)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--epoch-items", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_multiview.py needs a GPU"
    sc = tc.build_scene(full_size_sd=True)
    gd = sc["guidance"]
    opt = tc.make_opt()
    cs = tc.make_step(sc, opt)
    views = [tc.view(40.0 + 37.0 * i) for i in range(max(a.views))]
    kw = dict(shading="albedo", t=500)
    batched = lambda G: (lambda: cs.step_views(views[:G], 2000, **kw))
    sequential = lambda G: (lambda: [cs.step(views[v], 2001 + v, **kw) for v in range(G)])
    res = dict(metric="coarse iteration over G novel views: step_views (U-Net batch 2G) vs G x step (U-Net batch 2), 128^2 renders, "
                      "seeded full-size SD-2.0, all views SDS (t = 500)", card=card(), window_s=a.window, rounds=a.rounds, views={})
    for G in a.views:
        # StableDiffusion keeps one multi-view engine: planning G replaces the previous one
        try:
            torch.cuda.reset_peak_memory_stats()
            for fn in (batched(G), sequential(G)):    # warm-up: engine planning, graph capture, allocator
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
        except (torch.cuda.OutOfMemoryError, L.Mi3dError) as e:
            res["views"][G] = dict(skipped=f"{type(e).__name__}: {str(e)[:200]}")
            torch.cuda.empty_cache()
            continue
        r = res["views"][G] = dict(workspace_gib=round(gd.views_engine(G).nbytes / 2 ** 30, 3))
        reps = max(2, math.ceil(a.window * 1e3 / timed(sequential(G), 1)))      # iterations per window of >= a.window seconds
        samples = dict(batched=[], sequential=[])
        for _ in range(a.rounds):                 # alternated: both arms see the same host / clock conditions
            samples["batched"].append(timed(batched(G), reps))
            samples["sequential"].append(timed(sequential(G), reps))
        for arm, s in samples.items():
            m = statistics.median(s)
            r[arm] = dict(ms_per_iteration=round(m, 3), ms_per_view=round(m / G, 3), min=round(min(s), 3), max=round(max(s), 3))
        r["reps_per_window"] = reps
        r["per_view_speedup"] = round(r["sequential"]["ms_per_view"] / r["batched"]["ms_per_view"], 4)
        # the range of the speedup over the windows' extremes: worst batched against best sequential and the reverse
        r["per_view_speedup_range"] = [round(min(samples["sequential"]) / max(samples["batched"]), 4),
                                       round(max(samples["sequential"]) / min(samples["batched"]), 4)]
        r["sd_ms_per_view"] = {k: round(v / G, 3) for k, v in sd_parts(gd, G, 4 * reps).items()}
        r["peak_allocated_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)
    # whole epochs on a reference-shaped loader: front views cut the groups to every size up to G, so this is the memory a run holds
    trainer_kw = dict(model=cs.model, guidance=gd, clip_model=sc["clip"], optimizer=cs.optimizer, opt=opt, ref_imgs=sc["ref"],
                      depth_prediction=sc["prior"], depth_mask=sc["depth_mask"], text_z=sc["text_z"], clip_text_tokens=sc["tokens"],
                      workspace="", img_path=os.path.join(os.path.dirname(os.path.abspath(a.out or "x")), "multiview_png"),
                      lr_scheduler=torch.optim.lr_scheduler.LambdaLR(cs.optimizer, lambda it: 1.0))
    res["epoch"] = {}
    gd._view_engine = None                    # the single-view epoch holds no multi-view engine
    torch.cuda.empty_cache()
    for G in (1,) + tuple(g for g in a.views if g > 1):
        ms, peak = epoch(cs, trainer_kw, G, a.epoch_items, seed=1)             # warm (engine planning) ...
        ms, peak = epoch(cs, trainer_kw, G, a.epoch_items, seed=2)             # ... then measured
        res["epoch"][G] = dict(ms_per_item=round(ms, 3), peak_allocated_gib=round(peak, 3))
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
