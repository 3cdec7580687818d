"""Several novel views per coarse iteration on one GPU: the SD engine planned for G views (U-Net at batch 2G, VAE encoder at batch G)
against G single-view calls and the fp32 oracle, no mixing across the images of a batch, the per-view SDS / denoise branch choice,
`CoarseStep.step_views` against G single-view `step` calls, and `train_one_epoch(..., views_per_step=G)` end to end.  Fixtures are
those of tests/test_sd_gpu.py (tiny SD) and tests/test_coarse_gpu.py (scene, field, CLIP)."""
import argparse
import importlib
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import sd_ref  # noqa: E402
from test_coarse_gpu import HW, build_scene, make_adan, make_model, make_opt, make_step, scene, view  # noqa: E402,F401
from test_coarse_gpu import _rel as _rel_l2  # noqa: E402
from test_sd_gpu import _rel, tiny  # noqa: E402,F401

pytestmark = pytest.mark.gpu

G = 3


def _inputs(seed, g=G):
    gen = torch.Generator().manual_seed(seed)
    rgb = torch.rand(g, 3, 64, 64, generator=gen)
    eps = torch.randn(g, 4, 32, 32, generator=gen)
    noise = torch.randn(g, 4, 32, 32, generator=gen)
    ctx = torch.randn(2 * g, 77, 128, generator=gen)            # [uncond x G, cond x G], every row distinct
    return rgb.cuda(), eps.cuda(), noise.cuda(), ctx.cuda()


def _one(ctx, v, g=G):
    return torch.stack([ctx[v], ctx[g + v]])


class ColourClip:
    """a CLIP stand-in whose losses depend on the image: features = per-channel means; text features = the first 3 token values"""

    def encode_image(self, x):
        return x.mean(dim=(2, 3))

    def encode_text(self, tok):
        return tok[:, :3].float()


def test_batched_sds_matches_single_views_and_the_oracle(tiny):
    sdm, g, unet, vae = tiny
    rgb, eps, noise, ctx = _inputs(31)
    large = [False, True, False]
    rb = rgb.clone().requires_grad_()
    loss, imgs = g.train_step(ctx, rb, islarge=large, guidance_scale=10, t=500, eps_posterior=eps, noise=noise)
    assert loss == 0 and imgs == [None] * G and g.last["sds"] == [True] * G
    batch = {k: g.last[k].clone() for k in ("latents", "noise_pred", "grad")}
    assert g.views_engine(G).views == G and g.views_engine(G) is not g.engine
    for v in range(G):
        rv = rgb[v:v + 1].clone().requires_grad_()
        g.train_step(_one(ctx, v), rv, islarge=large[v], guidance_scale=10, t=500, eps_posterior=eps[v:v + 1], noise=noise[v:v + 1])
        torch.cuda.synchronize()
        # CFG amplifies the U-Net's (text - uncond) by the guidance scale: noise_pred and grad are compared at that scale, as
        # test_sd_gpu compares them with the oracle; the U-Net's own output is held to 1e-2 below
        for k, (tol, cmin) in (("latents", (1e-2, 0.9999)), ("noise_pred", (3e-2, 0.999)), ("grad", (3e-2, 0.999))):
            e, c = _rel(batch[k][v], g.last[k][0])
            print(f"view {v} {k:10s} batch vs single rel_l2={e:.3e} cos={c:.6f}")
            assert e < tol and c > cmin, (v, k, e, c)
        e, c = _rel(rb.grad[v], rv.grad[0])
        print(f"view {v} d pred_rgb  batch vs single rel_l2={e:.3e} cos={c:.6f}")
        assert e < 3e-2 and c > 0.999
        # guidance scale 0: noise_pred is the U-Net's text-row output, row G + v of the batch-2G pass against row 1 of the batch-2 pass
        tt = torch.tensor([500], dtype=torch.long, device="cuda")
        raw_b, _ = g.unet_sds(batch["latents"], noise, tt, ctx, 0.0)
        raw_1, _ = g.unet_sds(batch["latents"][v:v + 1], noise[v:v + 1], tt, _one(ctx, v), 0.0)
        e, c = _rel(raw_b[v], raw_1[0])
        print(f"view {v} U-Net out   batch vs single rel_l2={e:.3e} cos={c:.6f}")
        assert e < 1e-2 and c > 0.9999, (v, "U-Net output", e, c)
        # each view against the fp32 oracle (the bounds of test_sd_gpu's oracle comparisons)
        rr = rgb[v:v + 1].cpu().clone().requires_grad_()
        ref = sd_ref.sds_train_step_ref_at(unet, vae, _one(ctx, v).cpu(), rr, 500, eps[v:v + 1].cpu(), noise[v:v + 1].cpu(), 256, guidance_scale=10.0)
        e, c = _rel(batch["latents"][v], ref["latents"][0])
        assert e < 1e-2 and c > 0.9999, (v, "oracle latents", e, c)
        e, c = _rel(batch["noise_pred"][v], ref["noise_pred"][0])
        assert e < 3e-2 and c > 0.999, (v, "oracle noise_pred", e, c)
        e, c = _rel(rb.grad[v], rr.grad[0])
        print(f"view {v} d pred_rgb  batch vs oracle rel_l2={e:.3e} cos={c:.6f}")
        assert e < 5e-2 and c > 0.998, (v, "oracle d pred_rgb", e, c)


def test_views_do_not_leak_into_each_other(tiny):
    """changing view 1's image leaves view 0's latents as they were and its SDS gradient within the engine's run-to-run spread (the
    U-Net's split-K partial sums may land in another order); attention or GroupNorm over the batch would move both"""
    sdm, g, unet, vae = tiny
    rgb, eps, noise, ctx = _inputs(32)

    def run(r):
        rr = r.clone().requires_grad_()
        g.train_step(ctx, rr, islarge=True, guidance_scale=10, t=600, eps_posterior=eps, noise=noise)
        torch.cuda.synchronize()
        return g.last["latents"].clone(), g.last["grad"][0].clone(), rr.grad[0].clone()
    base, again = run(rgb), run(rgb)
    spread = [float((a[:1] - b[:1]).abs().max()) for a, b in zip(base, again)]
    other = rgb.clone()
    other[1] = torch.rand(3, 64, 64, generator=torch.Generator().manual_seed(5)).cuda()
    changed = run(other)
    assert float((changed[0][0] - base[0][0]).abs().max()) <= 2 * spread[0]      # bit-identical when the encode is repeatable
    for k in (1, 2):
        d = float((changed[k] - base[k]).abs().max())
        assert d <= max(4 * spread[k], 1e-4 * float(base[k].abs().max())), (k, d, spread[k])
    assert float((changed[0][1] - base[0][1]).abs().max()) > 0.1 * float(base[0][1].abs().max())     # the changed view itself moves


def test_branch_mix_at_small_t(tiny):
    """t = 300: the non-large views take the denoise branch (decoded image, CLIP value, no gradient), the large view the SDS gradient;
    the returned loss is the sum of the per-view CLIP values"""
    sdm, g, unet, vae = tiny
    rgb, eps, noise, ctx = _inputs(33)
    large = [False, True, False]
    gen = torch.Generator().manual_seed(6)
    ref_rgb = torch.rand(G, 3, 256, 256, generator=gen).cuda()
    ref_text = torch.rand(G, 77, generator=gen).cuda()
    clip = ColourClip()
    rb = rgb.clone().requires_grad_()
    loss, imgs = g.train_step(ctx, rb, islarge=large, t=300, eps_posterior=eps, noise=noise, ref_rgb=ref_rgb, ref_text=ref_text,
                              clip_model=clip)
    assert g.last["sds"] == large and imgs[1] is None
    assert float(rb.grad[0].abs().max()) == 0.0 and float(rb.grad[2].abs().max()) == 0.0 and float(rb.grad[1].abs().max()) > 0
    want = 0.0
    for v in range(G):
        rv = rgb[v:v + 1].clone().requires_grad_()
        lv, iv = g.train_step(_one(ctx, v), rv, islarge=large[v], t=300, eps_posterior=eps[v:v + 1], noise=noise[v:v + 1],
                              ref_rgb=ref_rgb[v:v + 1], ref_text=ref_text[v:v + 1], clip_model=clip)
        if large[v]:
            e, c = _rel(rb.grad[v], rv.grad[0])
            assert e < 3e-2 and c > 0.999, (e, c)
            continue
        assert rv.grad is None and imgs[v].shape == (1, 3, 256, 256)
        e, c = _rel(imgs[v], iv)
        assert e < 1e-2 and c > 0.9999, (v, e, c)
        want += float(lv)
    assert abs(float(loss) - want) <= 1e-3 * abs(want), (float(loss), want)
    # defer: the surrogate of the SDS views joins the same loss; its gradient is the SDS gradient
    rd = rgb.clone().requires_grad_()
    ld, _ = g.train_step(ctx, rd, islarge=large, t=300, eps_posterior=eps, noise=noise, ref_rgb=ref_rgb, ref_text=ref_text, clip_model=clip,
                         defer=True)
    assert rd.grad is None
    ld.backward()
    assert float((rd.grad - rb.grad).abs().max()) <= 1e-4 * float(rb.grad.abs().max())


def _novel_views():
    return [view(40.0), view(-50.0), view(20.0, large=True)]


@pytest.mark.parametrize("global_step,t,batched", [(100, None, True), (1999, 500, True), (1999, 300, True), (398, 500, True),
                                                   (1999, 500, False), (1999, 300, False)])
def test_step_views_equals_single_view_steps(scene, global_step, t, batched):
    """one G-view iteration == the sum of the G single-view iterations (same draws), gradients compared before the optimizer step.
    Before diff_iters (no guidance) the render, loss kernel and CLIP terms are the single-view ones: gradients to 3e-3, the non-front
    bound of test_one_iteration_matches_the_reference_step.  With guidance the SDS gradient of the batch comes from a U-Net pass at
    batch 2G and an encode at batch G, whose split-K sums land in another order than at batch 2 / 1 (the latents differ by ~3e-4, the
    SDS gradient by ~7e-3; test_batched_sds_matches_single_views_and_the_oracle holds it to 3e-2): gradients to 2e-2, and the SDS
    gradient handed to the render is compared view by view (a view mixed up with another would fail there).  A group started at 398
    holds steps 399, 400, 401: view 0 gets no guidance, views 1 and 2 one batch of 2.  batched=False: guidance_views set to another size,
    so the group's guidance runs view by view on the single-view engine: gradients to 3e-3 again."""
    opt = make_opt()
    datas = _novel_views()
    gen = torch.Generator().manual_seed(8)
    bg = torch.rand(G, 3, generator=gen).cuda()
    light = torch.nn.functional.normalize(torch.randn(G, 3, generator=gen), dim=1).cuda()
    noises = torch.rand(G * HW * HW, generator=gen).cuda()
    noise, eps = torch.randn(G, 4, 32, 32, generator=gen).cuda(), torch.randn(G, 4, 32, 32, generator=gen).cuda()
    kw = dict(shading="lambertian", t=t, step_seed=11)
    cs = make_step(scene, opt)
    cs.optimizer.step = lambda *a, **k: None
    cs.guidance_views = None if batched else 2
    gd = scene["guidance"]
    gd.last = {}
    res = cs.step_views(datas, global_step, bg_color=bg, light_d=light, noises=noises, noise=noise, eps_posterior=eps, **kw)
    grads_a = {n: p.grad.clone() for n, p in cs.model.named_parameters()}
    guided = [v for v in range(G) if global_step + 1 + v >= opt.diff_iters]
    sds_views = [v for v in guided if t is not None and (datas[v]["is_large"] or t > 400)]
    if batched and len(guided) > 1:
        assert gd.last["sds"] == [v in sds_views for v in guided]        # one batch over the guided views only
        grad_rgb_a = {v: gd.last["grad_rgb"][i] for i, v in enumerate(guided)}
    else:
        assert "sds" not in gd.last                                     # no batched call
    grad_rgb_b = {}
    cs_b = make_step(scene, opt, make_model(opt))
    cs_b.optimizer.step = lambda *a, **k: None
    grads_b, loss_b, guid_b = {}, 0.0, 0.0
    for v in range(G):
        r = cs_b.step(datas[v], global_step + 1 + v, bg_color=bg[v], light_d=light[v], noises=noises[v * HW * HW:(v + 1) * HW * HW],
                      noise=noise[v:v + 1], eps_posterior=eps[v:v + 1], **kw)
        if v in sds_views:
            grad_rgb_b[v] = gd.last["grad_rgb"][0].clone()
        loss_b += r["loss"].item()
        guid_b += r["guidance"].item()
        for n, p in cs_b.model.named_parameters():
            grads_b[n] = grads_b[n] + p.grad if n in grads_b else p.grad.clone()
    torch.cuda.synchronize()
    print(f"t={t}: loss {res['loss'].item():.6f} vs {loss_b:.6f}, guidance {res['guidance'].item():.6f} vs {guid_b:.6f}")
    assert abs(res["loss"].item() - loss_b) <= 1e-4 * abs(loss_b)
    assert set(res) == {"loss", "opacity", "entropy", "orient", "smooth", "clip", "guidance"}
    tol_grad = 3e-3 if (t is None or not batched) else 2e-2
    if batched and len(guided) > 1:
        for v in sds_views:
            e, c = _rel(grad_rgb_a[v], grad_rgb_b[v])
            print(f"view {v} SDS d pred_rgb batch vs single rel_l2={e:.3e} cos={c:.6f}")
            assert e < 3e-2 and c > 0.999, (v, e, c)
    if t == 300:
        assert guid_b != 0.0 and cs.last_views[0]["denoised"] is not None and cs.last_views[2]["denoised"] is None
    for n, gb in grads_b.items():
        if n == "encoder.params":
            continue
        print(f"{n}: rel_l2 {_rel_l2(grads_a[n], gb):.3e}")
        assert _rel_l2(grads_a[n], gb) <= tol_grad, (n, _rel_l2(grads_a[n], gb))
    table_a, table_b = grads_a["encoder.params"], grads_b["encoder.params"]
    sample = torch.randint(0, table_b.numel(), (1 << 18,), generator=torch.Generator().manual_seed(0)).cuda()
    assert float(table_b[sample].abs().max()) > 0
    print(f"encoder.params (sample): rel_l2 {_rel_l2(table_a[sample], table_b[sample]):.3e}")
    assert _rel_l2(table_a[sample], table_b[sample]) <= tol_grad, _rel_l2(table_a[sample], table_b[sample])


def test_step_views_never_synchronises(scene):
    opt = make_opt()
    cs = make_step(scene, opt)
    datas = _novel_views()
    for t in (500, 300, None):                               # warm-up: engine planning and workspaces may synchronise
        cs.step_views(datas, 2000, t=t)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for t in (500, 300, None):
            res = cs.step_views(datas, 2000, t=t)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert np.isfinite(res["loss"].item())


def test_train_one_epoch_groups_novel_views(scene, tmp_path):
    opt = make_opt(diff_iters=4, albedo_iters=2, update_extra_interval=3)
    model = make_model(opt)
    adan = make_adan(model)
    sched = torch.optim.lr_scheduler.LambdaLR(adan, lambda it: 1.0)
    logs, refreshes, calls = [], [], []
    orig = model.update_extra_state
    model.update_extra_state = lambda *a, **k: (refreshes.append(1), orig(*a, **k))[1]
    trainer = argparse.Namespace(model=model, guidance=scene["guidance"], clip_model=scene["clip"], optimizer=adan, opt=opt,
                                 ref_imgs=scene["ref"], depth_prediction=scene["prior"], depth_mask=scene["depth_mask"],
                                 text_z=scene["text_z"], clip_text_tokens=scene["tokens"], global_step=0, epoch=1, workspace=str(tmp_path),
                                 img_path=str(tmp_path / "images"), log=logs.append, stats={"loss": []}, lr_scheduler=sched,
                                 scheduler_update_every_step=True, fp16=False, ema=None, world_size=1)
    co = importlib.import_module("make-it-3d_b200.nerf.coarse")
    cs = co._coarse_step(trainer)
    step, step_views = cs.step, cs.step_views
    cs.step = lambda d, gs, **k: (calls.append(("step", bool(d["is_front"]), gs)), step(d, gs, **k))[1]
    cs.step_views = lambda ds, gs, **k: (calls.append(("views", len(ds), gs)), step_views(ds, gs, **k))[1]
    # items 0, 4, 8 are front views; 5 is large
    loader = [view(0.0 if i % 4 == 0 else 45.0 * i, front=i % 4 == 0, large=i == 5) for i in range(11)]
    co.train_one_epoch(trainer, loader, views_per_step=3)
    assert calls == [("step", True, 1), ("views", 3, 1), ("step", True, 5), ("views", 3, 5), ("step", True, 9), ("views", 2, 9)]
    assert trainer.global_step == 11 and trainer.local_step == 11 and sched.last_epoch == 11
    # a refresh wherever a multiple of update_extra_interval is crossed: pre-step values 0 (front), 3 (group 1..3), 6 (group 5..7), 9
    # (group 9..10)
    assert len(refreshes) == 4
    # one multi-view SD engine, at views_per_step: the group of 2 (and the one guided view of group 1..3, steps 2..4 against
    # diff_iters 4) ran their guidance view by view
    assert cs.guidance_views == 3 and scene["guidance"]._view_engine.views == 3
    assert len(trainer.stats["loss"]) == 1 and np.isfinite(trainer.stats["loss"][0])
    for name in ("1.png", "1_gt.png", "1_depth.png"):
        assert os.path.isfile(tmp_path / "images" / name), name


def test_full_size_step_views_at_four_views():
    """one full-size seeded SD-2.0 step_views at G = 4 (128^2 renders): finite gradients; the G-view engines' workspace is reported"""
    sc = build_scene(full_size_sd=True)
    gd = sc["guidance"]
    opt = make_opt()
    cs = make_step(sc, opt)
    cs.optimizer.step = lambda *a, **k: None
    datas = [view(40.0), view(-50.0), view(120.0), view(20.0, large=True)]
    res = cs.step_views(datas, 2000, t=500)
    torch.cuda.synchronize()
    assert np.isfinite(res["loss"].item())
    grads = [p.grad for p in cs.model.parameters() if p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads) and any(float(g.abs().max()) > 0 for g in grads)
    eng = gd.views_engine(4)
    print(f"full-size SD-2.0: constructor engine {gd.engine.nbytes / 2 ** 30:.2f} GiB, 4-view engine {eng.nbytes / 2 ** 30:.2f} GiB, "
          f"peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    assert eng.nbytes > gd.engine.nbytes
