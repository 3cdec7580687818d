"""The refine loop (nerf/refine.py, csrc/refine.cu) on the GPU: the image-loss kernel against the unit-colour render, MaxPool2d and
oracle/refine_ref.py; the Adam launch against torch.optim.Adam; one iteration of each branch against `eager_iteration`, a literal
restatement of nerf/utils.py:840-894 on this package's drop-ins and torch glue; no host synchronisation inside `step`; run-to-run
repeatability; and `refine()` end to end on a synthetic mvimg folder.  The guidance is the tiny SD configuration of the SD tests."""
import argparse
import importlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys  # noqa: E402

sys.path.insert(0, ROOT)
from oracle import refine_ref as rr  # noqa: E402
from oracle import sd_ref, views_ref as vr  # noqa: E402

pytestmark = pytest.mark.gpu

S = 800
rf = importlib.import_module("make-it-3d_b200.nerf.refine")
ru = importlib.import_module("make-it-3d_b200.nerf.refine_utils")
unet_mod = importlib.import_module("make-it-3d_b200.nerf.unet")
clip_mod = importlib.import_module("make-it-3d_b200.nerf.clip")
cx_mod = importlib.import_module("make-it-3d_b200.nerf.contextual_loss")
sd_mod = importlib.import_module("make-it-3d_b200.nerf.sd")


# ---- the reference loop body (nerf/utils.py:840-894), restated on the drop-ins ----

class Eager:
    """the reference's refine state: four point leaves, bg_feat, the U-Net and torch.optim.Adam over the six groups"""

    def __init__(self, rs, unet):
        pc = rs.p_cano
        pts = rs.points.detach()
        self.all_v = rs.all_v
        self.colour_cano = torch.nn.Parameter(pts[:pc, :3].clone())
        self.feat_cano = torch.nn.Parameter(pts[:pc, 3:].clone())
        self.colour_novel = torch.nn.Parameter(pts[pc:, :3].clone())
        self.feat_novel = torch.nn.Parameter(pts[pc:, 3:].clone())
        self.origin_cano, self.origin_novel = rs.origin[:pc].clone(), rs.origin[pc:].clone()
        self.bg_feat = torch.nn.Parameter(torch.ones(1, 19, 1, 1, device="cuda"))
        self.unet = unet
        self.K = rs.K
        params = [{'params': [self.colour_novel], 'lr': 0.001}, {'params': [self.colour_cano], 'lr': 0.001},
                  {'params': [self.feat_novel], 'lr': 0.001}, {'params': [self.feat_cano], 'lr': 0.001},
                  {'params': [self.bg_feat], 'lr': 0.001}, {'params': unet.parameters(), 'lr': 0.001}]
        self.opt = torch.optim.Adam(params, betas=(0.9, 0.99), eps=1e-15)

    def leaves(self):
        return [self.colour_cano, self.feat_cano, self.colour_novel, self.feat_novel]

    def all_v_color(self):
        return torch.cat((torch.cat((self.colour_cano, self.feat_cano), -1), torch.cat((self.colour_novel, self.feat_novel), -1)), 0)


def img_clip_loss(clip, rgb1, rgb2):
    """Trainer.img_clip_loss (nerf/utils.py:436-443): each image encoded on its own, the reference's resize / normalise included"""
    z1 = clip_mod._EncodeImage.apply(rgb1, clip.engine, 1, 1)
    z2 = clip_mod._EncodeImage.apply(rgb2, clip.engine, 1, 0)
    z1, z2 = z1 / z1.norm(dim=-1, keepdim=True), z2 / z2.norm(dim=-1, keepdim=True)
    return -(z1 * z2).sum(-1).mean()


def eager_iteration(e, w2c, is_front, guidance, text_z, clip, cx, gt, gt_mask, tokens, t=None, noise=None, eps_posterior=None):
    """one reference iteration; returns (loss value, {name: grad before the step})"""
    all_v_color = e.all_v_color()
    pred_list = [ru.render_point(e.all_v, all_v_color, S >> j, S >> j, e.K[j], w2c, (S >> j, S >> j), rf.RADIUS, rf.PPP, bg_feat=e.bg_feat)
                 for j in range(3)]
    pred_rgb = e.unet(pred_list)
    pred_mask = ru.render_point(e.all_v, torch.ones_like(e.all_v), S, S, e.K[0], w2c, (S, S), rf.RADIUS, rf.PPP)
    pred_mask_dilate = torch.nn.MaxPool2d(5, 1, 2)(pred_mask)
    if is_front:
        clip_loss = 1000 * torch.nn.L1Loss()(pred_rgb * gt_mask, gt * gt_mask)
    else:
        clip_loss, _ = guidance.train_step(text_z, pred_rgb, clip_model=clip, ref_text=tokens, islarge=False, ref_rgb=gt, guidance_scale=5,
                                           t=t, noise=noise, eps_posterior=eps_posterior)
        clip_loss += 10 * img_clip_loss(clip, pred_rgb, gt)
        clip_loss += cx(pred_rgb, gt)
    bg_loss = 1e-3 * (1 - pred_rgb * (1 - pred_mask_dilate)).sum()
    reg_loss = torch.nn.MSELoss()(e.colour_novel, e.origin_novel) * 1e3 + torch.nn.MSELoss()(e.colour_cano, e.origin_cano) * 1e5
    loss = clip_loss + reg_loss + bg_loss
    e.opt.zero_grad()
    loss.backward()
    grads = {n: p.grad.clone() for n, p in zip(("colour_cano", "feat_cano", "colour_novel", "feat_novel"), e.leaves())}
    grads.update({"unet." + n: p.grad.clone() for n, p in e.unet.named_parameters()})
    e.opt.step()
    return loss.detach(), dict(bg=bg_loss.detach(), reg=reg_loss.detach()), grads


# ---- fixtures ----

@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    folder = str(tmp_path_factory.mktemp("scene") / "mvimg")
    gt, rgb_f, depth_f, mask_f, poses, K = vr.make_mvimg(folder, 5, S, seed=0)
    vc, cc, vn, cn = ru.load_views(gt, rgb_f, depth_f, mask_f, poses, S, S, K, 2, 8, folder, "cuda")
    import cv2
    alpha = cv2.erode((gt.max(-1) > 0.05).astype(np.float64), np.ones((5, 5), np.uint8), iterations=1)
    dev = "cuda"
    gen = torch.Generator().manual_seed(0)
    ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
    guidance = sd_mod.StableDiffusion(dev, unet_cfg=dict(ucfg, latent_hw=32), vae_cfg=dict(vcfg, image_hw=256))
    return dict(folder=folder, gt_np=gt, alpha=alpha, poses=poses, K=K, cloud=(vc, cc, vn, cn),
                gt=torch.tensor(gt, dtype=torch.float32).permute(2, 0, 1)[None].contiguous().to(dev),
                mask=torch.tensor(alpha, dtype=torch.float32)[None, None].to(dev),
                clip=clip_mod.CLIP(dev), cx=cx_mod.ContextualLoss(device=dev), guidance=guidance,
                text_z=torch.randn(2, 77, ucfg["cross_dim"], generator=gen).to(dev),
                tokens=torch.randint(1, 49000, (1, 77), generator=gen).to(dev))


def _unet(seed=0):
    torch.manual_seed(seed)
    return unet_mod.UNet(num_input_channels=19).cuda().train()


def _step(sc, unet, seed=0):
    vc, cc, vn, cn = sc["cloud"]
    return rf.RefineStep(vc, cc, vn, cn, sc["K"], unet, sc["cx"], sc["clip"], sc["guidance"], sc["text_z"], sc["gt"], sc["mask"],
                         sc["tokens"], seed=seed)


def _w2c(sc, i=None):
    """the front pose (i None) or view i of the mvimg poses, world2cam fp32 on the device"""
    if i is None:
        c2w, _, _ = rf.fix_poses(0, torch.Generator(), __import__("random").Random(0))
    else:
        c2w = torch.from_numpy(sc["poses"][i])
    return rf.world2cam_device(c2w, "cuda")


def _lat(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, 4, 32, 32, generator=g).cuda(), torch.randn(1, 4, 32, 32, generator=g).cuda()


# ---- tests ----

def test_image_losses_match_unit_render_maxpool_and_oracle(scene):
    vc, cc, vn, cn = scene["cloud"]
    all_v = torch.from_numpy(np.concatenate([vc, vn])).float().cuda()
    g = torch.Generator().manual_seed(1)
    feats = torch.rand(all_v.shape[0], 19, generator=g).cuda()
    K0 = rf.level_K(scene["K"], 0).cuda()
    for view in (None, 1):
        w2c = _w2c(scene, view)
        img, w0 = ru.render_point_weights(all_v, feats, S, S, K0, w2c, [S, S], rf.RADIUS, rf.PPP)
        assert torch.equal(img, ru.render_point(all_v, feats, S, S, K0, w2c, [S, S], rf.RADIUS, rf.PPP))
        unit = ru.render_point(all_v, torch.ones_like(all_v), S, S, K0, w2c, [S, S], rf.RADIUS, rf.PPP)
        pred = torch.rand(1, 3, S, S, generator=g).cuda().requires_grad_()
        for front in (True, False):
            bg, l1, cover, dil = rf.image_losses(pred, w0, scene["gt"], scene["mask"], front)
            for c in range(3):
                assert torch.equal(cover, unit[0, c])
            assert torch.equal(dil, F.max_pool2d(unit, 5, 1, 2)[0, 0])
            pred.grad = None
            (bg + l1).backward()
            p64, d64 = pred.detach().double().cpu().numpy(), rr.dilate(rr.coverage(w0.double().cpu().numpy()))
            vb, gb = rr.bg_loss(p64, d64)
            assert abs(bg.item() - vb) <= 1e-6 * abs(vb)
            want = gb
            if front:
                vl, gl = rr.masked_l1(p64, scene["gt"].double().cpu().numpy(), scene["mask"].double().cpu().numpy())
                assert abs(l1.item() - vl) <= 1e-6 * abs(vl)
                want = gb + gl
            else:
                assert l1.item() == 0.0
            err = np.abs(pred.grad.double().cpu().numpy() - want).max()
            assert err <= 1e-6 * np.abs(want).max(), err


def test_adam_matches_torch_optim_within_one_ulp():
    """three steps with the same gradients: every updated parameter within 1 fp32 ulp of torch.optim.Adam's (foreach path)"""
    g = torch.Generator().manual_seed(2)
    pc, pn = 1500, 2600
    pts = torch.rand(pc + pn, 19, generator=g).cuda()
    pts[:, 3:] = torch.randn(pc + pn, 16, generator=g).cuda()
    origin = (pts[:, :3] + 0.01 * torch.randn(pc + pn, 3, generator=g).cuda()).contiguous()
    extra = [torch.randn(64, 19, 3, 3, generator=g).cuda(), torch.randn(13, generator=g).cuda()]
    mine = [pts.clone()] + [t.clone() for t in extra]
    adam = rf.Adam(mine, origin=origin, p_cano=pc, p_novel=pn)
    ref = [torch.nn.Parameter(t) for t in (pts[pc:, :3].clone(), pts[:pc, :3].clone(), pts[pc:, 3:].clone(), pts[:pc, 3:].clone())]
    ref_extra = [torch.nn.Parameter(t.clone()) for t in extra]
    opt = torch.optim.Adam([{'params': [p], 'lr': 1e-3} for p in ref] + [{'params': ref_extra, 'lr': 1e-3}], betas=(0.9, 0.99), eps=1e-15)
    for step in range(3):
        gp = torch.randn(pc + pn, 19, generator=g).cuda() * 1e-2
        ge = [torch.randn(t.shape, generator=g).cuda() for t in extra]
        adam.zero_grad()
        mine[0].grad.copy_(gp)
        for m, e in zip(mine[1:], ge):
            m.grad.copy_(e)
        reg = adam.step()
        opt.zero_grad()
        reg_ref = torch.nn.MSELoss()(ref[0], origin[pc:]) * 1e3 + torch.nn.MSELoss()(ref[1], origin[:pc]) * 1e5
        reg_ref.backward()
        for p, e in zip(ref, (gp[pc:, :3], gp[:pc, :3], gp[pc:, 3:], gp[:pc, 3:])):
            p.grad = e.clone() if p.grad is None else p.grad + e          # the features have no regulariser
        for p, e in zip(ref_extra, ge):
            p.grad = e.clone()
        opt.step()
        assert abs(reg.item() - reg_ref.item()) <= 1e-6 * reg_ref.item()
        got = [mine[0][pc:, :3], mine[0][:pc, :3], mine[0][pc:, 3:], mine[0][:pc, 3:]] + mine[1:]
        for a, b in zip(got, ref + ref_extra):
            b = b.detach()
            ulp = (torch.nextafter(b, torch.full_like(b, float("inf"))) - b).abs()
            assert bool(((a - b).abs() <= ulp).all()), float(((a - b).abs() / ulp).max())


@pytest.mark.parametrize("branch", ["front", "sds", "denoise"])
def test_one_iteration_matches_the_reference_loop(scene, branch):
    unet_a, unet_b = _unet(0), _unet(0)
    rs = _step(scene, unet_a)
    e = Eager(rs, unet_b)
    front = branch == "front"
    w2c = _w2c(scene, None if front else 3)
    t = {"front": None, "sds": 500, "denoise": 300}[branch]
    noise, eps = _lat(5)
    kw = dict(t=t, noise=noise, eps_posterior=eps)
    terms = rs.step(w2c, front, keep_colours=True, **kw)
    loss_ref, terms_ref, grads_ref = eager_iteration(e, w2c, front, scene["guidance"], scene["text_z"], scene["clip"], scene["cx"],
                                                     scene["gt"], scene["mask"], scene["tokens"], **kw)
    torch.cuda.synchronize()
    for k in ("bg", "reg"):
        assert abs(terms[k].item() - terms_ref[k].item()) <= 1e-5 * abs(terms_ref[k].item()), k
    assert abs(terms["loss"].item() - loss_ref.item()) <= 1e-5 * abs(loss_ref.item())
    # .grad of the four regions (the image-loss part; the regulariser part is added in the update, torch's expression here)
    pc = rs.p_cano
    before = rs.kept_colours
    reg_g = [((before[:pc, :3] - rs.origin[:pc]) * (2.0 / (3 * pc))) * 1e5, ((before[pc:, :3] - rs.origin[pc:]) * (2.0 / (3 * rs.p_novel))) * 1e3]
    g = rs.points.grad
    mine = {"colour_cano": g[:pc, :3] + reg_g[0], "feat_cano": g[:pc, 3:], "colour_novel": g[pc:, :3] + reg_g[1], "feat_novel": g[pc:, 3:]}
    mine.update({"unet." + n: p.grad for n, p in unet_a.named_parameters()})
    for n, ref in grads_ref.items():
        scale = float(ref.abs().max())
        assert float((mine[n] - ref).abs().max()) <= 1e-4 * scale + 1e-30, n
    for (n, a), (_, b) in zip(unet_a.named_buffers(), unet_b.named_buffers()):
        assert torch.allclose(a.double(), b.double(), rtol=1e-6, atol=1e-7), n
    # parameters after the update, where the gradient clears a floor (a near-zero gradient may flip sign and move by 2 lr)
    after = {"colour_cano": rs.points[:pc, :3], "feat_cano": rs.points[:pc, 3:], "colour_novel": rs.points[pc:, :3], "feat_novel": rs.points[pc:, 3:]}
    for (n, a), p in zip(after.items(), e.leaves()):
        ref = grads_ref[n]
        sel = ref.abs() > 1e-3 * ref.abs().max()
        assert float((a.detach() - p.detach())[sel].abs().max()) <= 1e-6, n
    for (n, a), (_, b) in zip(unet_a.named_parameters(), unet_b.named_parameters()):
        ref = grads_ref["unet." + n]
        sel = ref.abs() > 1e-3 * ref.abs().max()
        if bool(sel.any()):
            assert float((a.detach() - b.detach())[sel].abs().max()) <= 1e-6, n


def test_step_never_synchronises(scene):
    rs = _step(scene, _unet(1))
    noise, eps = _lat(6)
    w_front, w_side = _w2c(scene, None), _w2c(scene, 2)
    rs.step(w_front, True)                                   # warm-up: engine planning may synchronise
    rs.step(w_side, False, t=300, noise=noise, eps_posterior=eps)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for args in ((w_front, True, {}), (w_side, False, dict(t=300, noise=noise, eps_posterior=eps)), (w_side, False, dict(t=500)),
                     (w_side, False, {})):
            terms = rs.step(args[0], args[1], **args[2])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert np.isfinite(terms["loss"].item())


def test_iterations_are_bitwise_repeatable(scene):
    runs = []
    noise, eps = _lat(7)
    for _ in range(2):
        unet = _unet(2)
        rs = _step(scene, unet, seed=3)
        out = [rs.step(_w2c(scene, None), True), rs.step(_w2c(scene, 1), False, t=300, noise=noise, eps_posterior=eps),
               rs.step(_w2c(scene, 4), False, t=500)]
        runs.append((rs.points.detach().clone(), [p.detach().clone() for p in unet.parameters()],
                     [b.clone() for b in unet.buffers()], [{k: v.item() for k, v in o.items()} for o in out]))
    a, b = runs
    assert torch.equal(a[0], b[0])
    assert all(torch.equal(x, y) for x, y in zip(a[1], b[1]))
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    assert a[3] == b[3]


def test_refine_end_to_end(scene, tmp_path):
    import cv2
    folder = str(tmp_path / "run_mvimg")
    gt, *_ = vr.make_mvimg(folder, 4, S, seed=1)
    rgba = np.concatenate([gt, (gt.max(-1, keepdims=True) > 0.05)], -1)
    ref_path = str(tmp_path / "ref.png")
    cv2.imwrite(ref_path, np.round(rgba[:, :, [2, 1, 0, 3]] * 255).astype(np.uint8))
    opt = argparse.Namespace(text="a thing", ref_path=ref_path, fov=40.0, H=S, W=S, radius_range=[1, 1.5], theta_range=[45, 105],
                             phi_range=[-180, 180])
    trainer = argparse.Namespace(opt=opt, guidance=scene["guidance"], clip_model=scene["clip"], text_z=[scene["text_z"]],
                                 clip_text_tokens=scene["tokens"])
    c2w = [vr.pr.lookat_c2w(1.2, 70.0, a).astype(np.float32) for a in (0.0, 90.0)]
    rs = rf.refine(trainer, folder, 3, [{"poses": torch.from_numpy(p)[None]} for p in c2w])
    out = folder.replace("mvimg", "refine")
    names = ["vertices_cano.npy", "vertices_color_cano.npy", "vertices_novel.npy", "vertices_color_novel.npy", "train/0.png",
             "results/render_unet_0000.png", "results/render_unet_0001.png"]
    names += [f"{tag}_{n}" for tag in ("0", "end") for n in ("v_unet.pt", "v_color_unet.pt", "bg_unet.pt", "unet.pth")]
    for n in names:
        assert os.path.isfile(os.path.join(out, n)), n
    ck = torch.load(os.path.join(out, "end_unet.pth"), weights_only=False)
    u = unet_mod.UNet(num_input_channels=19).cuda()
    u.load_state_dict(ck["model_state_dict"])
    pc, pn = rs.p_cano, rs.p_novel
    leaves = [torch.nn.Parameter(torch.zeros(*s, device="cuda")) for s in ((pn, 3), (pc, 3), (pn, 16), (pc, 16), (1, 19, 1, 1))]
    adam = torch.optim.Adam([{'params': [p], 'lr': 0.001} for p in leaves] + [{'params': u.parameters(), 'lr': 0.001}],
                            betas=(0.9, 0.99), eps=1e-15)
    adam.load_state_dict(ck["optimizer_state_dict"])
    assert leaves[4] not in adam.state and float(adam.state[leaves[0]]["step"]) == 3.0
    assert torch.equal(adam.state[leaves[1]]["exp_avg"], rs.opt.exp_avg[0][:pc, :3])
    colours = torch.load(os.path.join(out, "end_v_color_unet.pt"))
    assert colours.shape == (pc + pn, 19)
    # render(): the three renders through the U-Net in train mode, as composed by hand on a copy of the U-Net
    w2c = torch.from_numpy(np.linalg.inv(c2w[0].astype(np.float64)).astype(np.float32)).cuda()
    twin = unet_mod.UNet(num_input_channels=19).cuda().train()
    twin.load_state_dict(rs.unet.state_dict())
    imgs = [ru.render_point(rs.all_v, colours, S >> j, S >> j, rs.K[j], w2c, (S >> j, S >> j), rf.RADIUS, rf.PPP) for j in range(3)]
    with torch.no_grad():
        want = twin(imgs)
    assert torch.equal(rs.render(w2c, colours=colours), want)
