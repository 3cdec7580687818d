"""The coarse loop (nerf/coarse.py, csrc/coarse.cu) on the GPU: the loss kernel against oracle/coarse_ref.py and torch autograd of the
reference expressions; one iteration of each branch against `eager_train_step`, a literal restatement of nerf/utils.py:461-574 +
:977-986 on this package's drop-ins with the reference's two backwards; no host synchronisation inside `step`; repeatability; and
`train_one_epoch` end to end.  Fixtures: a sphere-occupancy field with a "trained-like" table (as bench.py builds it), the tiny SD
configuration of the SD tests, native CLIP, a seeded synthetic RGBA reference and depth prior."""
import argparse
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import camera_rays, make_table, sphere_bitfield  # noqa: E402
from oracle import coarse_ref as cr  # noqa: E402
from oracle import sd_ref  # noqa: E402
from test_coarse_oracle_cpu import _case, reference_terms, torch_pearson  # noqa: E402

pytestmark = pytest.mark.gpu

co = importlib.import_module("make-it-3d_b200.nerf.coarse")
nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
sd_mod = importlib.import_module("make-it-3d_b200.nerf.sd")
clip_mod = importlib.import_module("make-it-3d_b200.nerf.clip")
Adan = importlib.import_module("make-it-3d_b200.optimizer").Adan

HW = 128


def _rel(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def make_opt(**kw):
    o = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1, lambda_smooth=1,
                           lambda_orient=1e-2, lambda_opacity=1e-3, lambda_entropy=1, lambda_img=1e3, lambda_depth=1, lambda_clip=1,
                           max_depth=10.0, max_steps=512, dt_gamma=0, albedo_iters=1000, diff_iters=400, guidance_scale=10,
                           update_extra_interval=16, fp16=False)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def make_model(opt):
    torch.manual_seed(0)
    m = nt.NeRFNetwork(opt)
    with torch.no_grad():
        m.encoder.params.copy_(torch.from_numpy(make_table(m.encoder.params.numel(), 3, 0.5)))
    m = m.cuda().train()
    m.density_bitfield = torch.from_numpy(sphere_bitfield(0.2)).cuda()
    return m


def make_adan(model):
    return Adan(model.get_params(1e-3), eps=1e-8, weight_decay=2e-5, max_grad_norm=5.0, clip_grad_norm=10)


def view(phi, front=False, large=False):
    ro, rd, sc = camera_rays(HW, radius=1.0 if front else 1.2, theta=90.0 if front else 75.0, phi=phi)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()[None]
    return dict(rays_o=cu(ro), rays_d=cu(rd), depth_scale=cu(sc), H=HW, W=HW, is_front=front, is_large=large)


def build_scene(full_size_sd=False):
    """the shared inputs: reference RGBA, depth prior and mask, guidance (tiny SD, or seeded full-size SD-2.0), CLIP, text"""
    dev = "cuda"
    g = torch.Generator().manual_seed(0)
    yy, xx = torch.meshgrid(torch.arange(512, dtype=torch.float64), torch.arange(512, dtype=torch.float64), indexing="ij")
    obj = ((yy - 256) ** 2 + (xx - 256) ** 2) < 120 ** 2
    ref = torch.rand(1, 4, 512, 512, generator=g)
    ref[:, 3] = obj.float()
    prior = (0.1 + 0.9 * (1 - ((yy - 256) ** 2 + (xx - 256) ** 2).sqrt() / 200).clamp(0, 1)) * obj + (~obj).double()
    if full_size_sd:
        guidance = sd_mod.StableDiffusion(dev)
    else:
        ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
        guidance = sd_mod.StableDiffusion(dev, unet_cfg=dict(ucfg, latent_hw=32), vae_cfg=dict(vcfg, image_hw=256))
    text_z = [torch.randn(2, 77, guidance.unet_cfg["cross_dim"], generator=g).to(dev) for _ in range(2)]
    return dict(ref=ref.to(dev), prior=prior.to(dev), depth_mask=(~obj).to(dev), guidance=guidance, clip=clip_mod.CLIP(dev),
                text_z=text_z, tokens=torch.randint(1, 49000, (2, 77), generator=g).to(dev))


@pytest.fixture(scope="module")
def scene():
    return build_scene()


def make_step(sc, opt, model=None):
    model = model or make_model(opt)
    return co.CoarseStep(model, sc["guidance"], sc["clip"], make_adan(model), opt, sc["ref"], sc["prior"], sc["depth_mask"],
                         sc["text_z"], sc["tokens"])


# ---- the reference iteration (nerf/utils.py:461-574 + :977-986), restated on the drop-ins ----

def img_clip_loss(clip, rgb1, rgb2):
    z1 = clip_mod._EncodeImage.apply(rgb1, clip.engine, 1, 1)
    z2 = clip_mod._EncodeImage.apply(rgb2, clip.engine, 1, 0)
    z1, z2 = z1 / z1.norm(dim=-1, keepdim=True), z2 / z2.norm(dim=-1, keepdim=True)
    return -(z1 * z2).sum(-1).mean()


def img_text_clip_loss(clip, rgb, tokens):
    z1 = clip_mod._EncodeImage.apply(rgb, clip.engine, 1, 1)
    z1 = z1 / z1.norm(dim=-1, keepdim=True)
    zt = clip.encode_text(tokens)
    zt = zt / zt.norm(dim=-1, keepdim=True)
    return -(z1 * zt).sum(-1).mean()


def eager_train_step(model, optimizer, opt, sc, data, global_step, shading, bg_color, light_d, t=None, noise=None, eps_posterior=None):
    """one reference iteration with its two render backwards on SDS steps; returns (loss, {name: clipped grad of the step})"""
    optimizer.zero_grad()
    rays_o, rays_d, depth_scale = data['rays_o'], data['rays_d'], data['depth_scale']
    B, N = rays_o.shape[:2]
    H, W = data['H'], data['W']
    ambient_ratio = 1.0 if shading == 'albedo' else 0.1
    ref_imgs = sc["ref"]
    bg_img = bg_color.expand(1, 512, 512, 3).permute(0, 3, 1, 2).contiguous()
    gt_rgb = ref_imgs[:, :3, :, :] * ref_imgs[:, 3:, :, :] + bg_img * (1 - ref_imgs[:, 3:, :, :])
    kw = dict(vars(opt))
    kw.update(depth_scale=depth_scale, bg_color=bg_color, staged=False, perturb=True, ambient_ratio=ambient_ratio, shading=shading,
              force_all_rays=True, light_d=light_d)
    outputs = model.render(rays_o, rays_d, **kw)
    pred_rgb = outputs['image'].reshape(B, H, W, 3).permute(0, 3, 1, 2).contiguous()
    pred_depth = outputs['depth'].reshape(B, H, W, 1).permute(0, 3, 1, 2).contiguous()
    pred_ws = outputs['weights_sum'].reshape(B, 1, H, W)
    k = 1 if data['is_large'] else 0
    text_z, text = sc["text_z"][k], sc["tokens"][k:k + 1]
    if global_step < opt.diff_iters or data['is_front']:
        loss = 0
    else:
        loss, _ = sc["guidance"].train_step(text_z, pred_rgb, clip_model=sc["clip"], ref_text=text, islarge=data['is_large'], ref_rgb=gt_rgb,
                                            guidance_scale=opt.guidance_scale, t=t, noise=noise, eps_posterior=eps_posterior, defer=False)
    loss_opacity = (pred_ws ** 2).mean()
    loss = loss + (opt.lambda_opacity * loss_opacity * 10 if data['is_large'] else opt.lambda_opacity * loss_opacity)
    alphas = pred_ws.clamp(1e-5, 1 - 1e-5)
    loss_entropy = (- alphas * torch.log2(alphas) - (1 - alphas) * torch.log2(1 - alphas)).mean()
    loss = loss + (opt.lambda_entropy * loss_entropy if global_step < opt.diff_iters else opt.lambda_entropy * loss_entropy * 10)
    loss_orient = outputs['loss_orient']
    loss = loss + opt.lambda_orient * loss_orient
    loss = loss + (opt.lambda_orient * loss_orient if global_step < opt.diff_iters else opt.lambda_orient * loss_orient * 10)
    loss = loss + opt.lambda_smooth * outputs['loss_smooth']
    pred_rgb = F.interpolate(pred_rgb, (512, 512), mode='bilinear', align_corners=True)
    pred_depth = F.interpolate(pred_depth, (512, 512), mode='bilinear', align_corners=True)
    if data['is_front']:
        loss_ref = opt.lambda_img * torch.nn.L1Loss()(pred_rgb, gt_rgb)
        x = torch.nan_to_num(pred_depth.squeeze()).reshape(-1)
        m = (~sc["depth_mask"]).reshape(-1) == 1
        loss_depth = opt.lambda_depth * (1 - torch_pearson(x[m].double(), sc["prior"].reshape(-1)[m]))
        loss_ref += loss_depth
    else:
        loss_ref = opt.lambda_clip * img_clip_loss(sc["clip"], pred_rgb, gt_rgb) + opt.lambda_clip * img_text_clip_loss(sc["clip"], pred_rgb, text)
    loss = loss + loss_ref
    loss.backward()
    optimizer.step()
    # after the step: Adan's clip_grad_norm scales .grad in place, as it does on the native side
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    return loss.detach(), grads


# ---- tests ----

@pytest.mark.parametrize("hw", [(HW, HW), (37, 53)])
def test_loss_kernel_matches_oracle_and_torch_autograd(hw):
    h, w = hw
    image, depth, ws, ref, bg, prior, depth_mask = _case(h, w, seed=11, nonfinite=True, at_bounds=True)
    prior = prior + 0.5 * F.interpolate(depth.reshape(1, 1, h, w).nan_to_num(0, 0, 0), (512, 512), mode='bilinear',
                                        align_corners=True)[0, 0].double() * (~depth_mask)
    mask_u8 = (~depth_mask).to(torch.uint8)
    gen = torch.Generator().manual_seed(3)
    g_pred = torch.randn(1, 3, 512, 512, generator=gen) * 1e-3
    cu = lambda t: t.cuda()
    for front in (True, False):
        ti, td, tw = (cu(t).requires_grad_() for t in (image, depth, ws))
        terms, pred512, gt512 = co.coarse_losses(ti, td, tw, h, w, cu(ref), cu(bg), cu(prior), cu(mask_u8), front)
        g_terms = torch.tensor([0.7, -1.3, 2.1, -0.9], device="cuda")
        torch.autograd.backward([terms, pred512], [g_terms, cu(g_pred)])
        args = (image.numpy(), depth.numpy(), ws.numpy(), h, w, ref.numpy(), bg.numpy(), prior.numpy(), mask_u8.numpy(), front)
        o_terms, o_pred, o_gt = cr.forward(*args)
        got = terms.detach().double().cpu().numpy()
        for k in range(4):
            assert abs(got[k] - o_terms[k]) <= 1e-5 * max(abs(o_terms[k]), 1e-2 if k == 3 else 0.0), (k, got[k], o_terms[k])
        assert np.array_equal(gt512.cpu().double().numpy(), o_gt)
        want_pred = F.interpolate(cu(image).reshape(1, h, w, 3).permute(0, 3, 1, 2), (512, 512), mode='bilinear', align_corners=True)
        assert float((pred512 - want_pred).abs().max()) <= 1e-6
        gi, gd, gw = cr.backward(*args, g_terms.double().cpu().numpy(), g_pred.double().numpy())
        assert _rel(ti.grad.cpu(), torch.from_numpy(gi)) <= 1e-5
        assert _rel(tw.grad.cpu(), torch.from_numpy(gw)) <= 1e-5
        if front:
            assert _rel(td.grad.cpu(), torch.from_numpy(gd)) <= 1e-5
        else:
            assert float(td.grad.abs().max()) == 0.0
        # torch autograd of the reference expressions on the GPU
        ri, rd_, rw = (cu(t).requires_grad_() for t in (image, depth, ws))
        rterms, rpred, _ = reference_terms(ri, rd_, rw, h, w, cu(ref), cu(bg), cu(prior), cu(depth_mask), front)
        total = sum(g.double() * t.double() for g, t in zip(g_terms, rterms)) + (cu(g_pred) * rpred).sum().double()
        total.backward()
        for k, t in enumerate(rterms):
            assert abs(got[k] - t.item()) <= 1e-5 * max(abs(t.item()), 1e-2 if k == 3 else 0.0), k
        assert _rel(ti.grad, ri.grad) <= 1e-5 and _rel(tw.grad, rw.grad) <= 1e-5
        if front:
            assert _rel(td.grad, rd_.grad) <= 1e-5


def test_loss_kernel_empty_mask_gives_nan_and_no_depth_gradient_and_is_bitwise_repeatable():
    image, depth, ws, ref, bg, prior, depth_mask = _case(32, 24, seed=12, mask_kind="empty")
    mask_u8 = (~depth_mask).to(torch.uint8).cuda()
    runs = []
    for _ in range(2):
        ti, td, tw = (t.cuda().requires_grad_() for t in (image, depth, ws))
        terms, pred512, gt512 = co.coarse_losses(ti, td, tw, 32, 24, ref.cuda(), bg.cuda(), prior.cuda(), mask_u8, True)
        (terms[:3].sum() + terms[3].nan_to_num(0) + pred512.square().mean()).backward()
        runs.append((terms.detach().clone(), ti.grad, td.grad, tw.grad))
    assert torch.isnan(runs[0][0][3]) and float(runs[0][2].abs().max()) == 0.0
    for a, b in zip(*runs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))


BRANCHES = {                      # global_step, view, t, shading
    "front": (2000, dict(phi=0.0, front=True), None, "albedo"),
    "sds": (2000, dict(phi=40.0), 500, "lambertian"),
    "denoise": (2000, dict(phi=-50.0), 300, "albedo"),
    "before_diff_iters": (100, dict(phi=60.0), None, "albedo"),
    "large": (2000, dict(phi=20.0, large=True), 300, "textureless"),
}


@pytest.mark.parametrize("branch", list(BRANCHES))
def test_one_iteration_matches_the_reference_step(scene, branch):
    global_step, vkw, t, shading = BRANCHES[branch]
    opt = make_opt()
    cs = make_step(scene, opt)
    model_b = make_model(opt)
    adan_b = make_adan(model_b)
    data = view(**vkw)
    bg = torch.tensor([0.3, 0.6, 0.2], device="cuda")
    light = torch.tensor([0.0, 0.6, 0.8], device="cuda")
    g = torch.Generator().manual_seed(5)
    noise, eps = torch.randn(1, 4, 32, 32, generator=g).cuda(), torch.randn(1, 4, 32, 32, generator=g).cuda()
    torch.manual_seed(123)
    res = cs.step(data, global_step, shading=shading, bg_color=bg, t=t, noise=noise, eps_posterior=eps, light_d=light)
    grads_a = {n: p.grad.clone() for n, p in cs.model.named_parameters()}      # clipped in place by Adan's step
    torch.manual_seed(123)
    loss_b, grads_b = eager_train_step(model_b, adan_b, opt, scene, data, global_step, shading, bg, light, t=t, noise=noise, eps_posterior=eps)
    torch.cuda.synchronize()
    # non-front views: CLIP encodes [pred512, gt512] in one batch where the reference encodes each image on its own; the fp16-storage
    # tile plans of the two batch sizes round differently, so the CLIP value agrees to 1e-4 and the gradient it feeds back through the
    # image tower to its fp16 floor (3e-3); front views hold the loss to 1e-5 and the gradients to 1e-4 (summation order)
    tol, tol_grad = (1e-5, 1e-4) if vkw.get("front") else (1e-4, 3e-3)
    assert abs(res["loss"].item() - loss_b.item()) <= tol * abs(loss_b.item()), (res["loss"].item(), loss_b.item())
    assert set(res) == {"loss", "opacity", "entropy", "orient", "smooth"} | ({"l1", "depth"} if vkw.get("front") else {"clip", "guidance"})
    for n, gb in grads_b.items():
        if n == "encoder.params":
            continue
        assert _rel(grads_a[n], gb) <= tol_grad, (n, _rel(grads_a[n], gb))
    table_a, table_b = grads_a["encoder.params"], grads_b["encoder.params"]
    sample = torch.randint(0, table_b.numel(), (1 << 18,), generator=torch.Generator().manual_seed(0)).cuda()
    assert float(table_b[sample].abs().max()) > 0
    # the table gradient is accumulated with fp32 atomics in the field backward, in arrival order
    assert _rel(table_a[sample], table_b[sample]) <= max(5e-4, tol_grad), _rel(table_a[sample], table_b[sample])
    for (n, pa), (_, pb) in zip(cs.model.named_parameters(), model_b.named_parameters()):
        gb = grads_b[n]
        sel = gb.abs() > 1e-2 * gb.abs().max()
        assert float((pa.detach() - pb.detach())[sel].abs().max()) <= 1e-6, (n, float((pa.detach() - pb.detach())[sel].abs().max()))


def test_step_never_synchronises(scene):
    opt = make_opt()
    cs = make_step(scene, opt)
    views = [view(0.0, front=True), view(40.0), view(20.0, large=True)]
    for d, t in zip(views, (None, 300, 500)):              # warm-up: engine planning and workspaces may synchronise
        cs.step(d, 2000, t=t)
    views.append(view(-30.0))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for d, t in zip(views, (None, 300, 500, None)):
            res = cs.step(d, 2000, t=t)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert np.isfinite(res["loss"].item())


def test_identical_steps_are_bitwise_identical(scene):
    """the loss kernel's forward and its gradients into the render are bitwise repeatable; so is every loss term of the step (the
    field backward then accumulates with fp32 atomics, so parameter gradients are compared to summation order above)"""
    out = []
    for _ in range(2):
        opt = make_opt()
        cs = make_step(scene, opt)
        torch.manual_seed(7)
        r1 = cs.step(view(0.0, front=True), 2000, bg_color=torch.full((3,), 0.5, device="cuda"), light_d=torch.tensor([0.0, 0.0, 1.0], device="cuda"))
        out.append({k: v.item() for k, v in r1.items()})
    assert out[0] == out[1]


def test_train_one_epoch_end_to_end(scene, tmp_path):
    opt = make_opt(diff_iters=4, albedo_iters=2, update_extra_interval=4)
    model = make_model(opt)
    adan = make_adan(model)
    sched = torch.optim.lr_scheduler.LambdaLR(adan, lambda it: 1.0)
    logs = []
    calls = []
    orig = model.update_extra_state
    model.update_extra_state = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    trainer = argparse.Namespace(model=model, guidance=scene["guidance"], clip_model=scene["clip"], optimizer=adan, opt=opt,
                                 ref_imgs=scene["ref"], depth_prediction=scene["prior"], depth_mask=scene["depth_mask"],
                                 text_z=scene["text_z"], clip_text_tokens=scene["tokens"], global_step=0, epoch=1, workspace=str(tmp_path),
                                 img_path=str(tmp_path / "images"), log=logs.append, stats={"loss": []}, lr_scheduler=sched,
                                 scheduler_update_every_step=True, fp16=False, ema=None, world_size=1)
    loader = [view(0.0 if i % 4 == 0 else 45.0 * i, front=i % 4 == 0, large=i == 5) for i in range(8)]
    co.train_one_epoch(trainer, loader)
    assert trainer.global_step == 8 and trainer.local_step == 8
    assert len(calls) == 2                                   # global_step 0 and 4
    assert sched.last_epoch == 8
    assert len(trainer.stats["loss"]) == 1 and np.isfinite(trainer.stats["loss"][0])
    assert logs[0].startswith("==> Start Training") and logs[-1].startswith("==> Finished Epoch 1")
    for name in ("1.png", "1_gt.png", "1_depth.png", "1_ref_depth_mask.png"):
        assert os.path.isfile(tmp_path / "images" / name), name
    assert adan.clip_grad_norm == 10
