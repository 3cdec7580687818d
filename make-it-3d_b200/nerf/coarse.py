"""B12 seam: the coarse stage's training iteration (reference `Trainer.train_step` + the body of `Trainer.train_one_epoch`,
nerf/utils.py:461-574, :947-1027) on libmi3d.so.

* `coarse_losses(image, depth, weights_sum, h, w, ref_imgs, bg_color, depth_prior, mask, front)`: the per-iteration losses of
  csrc/coarse.cu as one autograd node -> (terms [4] = opacity, entropy, l1, pearson; pred512; gt512).
* `CoarseStep(model, guidance, clip_model, optimizer, opt, ref_imgs, depth_prediction, depth_mask, text_z, clip_text_tokens)`: the
  state of one coarse run.  `step(data, global_step, ...)` runs one iteration as one autograd graph with ONE backward (the SDS
  gradient enters as `StableDiffusion.train_step(defer=True)`'s surrogate instead of a second walk of the render graph), then one
  `Adan.step()` or `Adam.step()` (`--optim adan` / `adam|adamw`) with the Trainer's `clip_grad_norm(10)` folded in.  It returns
  the loss terms as device scalars and never synchronises the host.
* `CoarseStep.step_views(datas, global_step, ...)`: one iteration over G (<= 8) novel views: one multi-view render, the loss kernel per
  view, one batched guidance call (`StableDiffusion.train_step` on [G,3,H,W], U-Net at batch 2G), one backward, one optimizer step.
* `train_step(trainer, data)` / `train_one_epoch(trainer, loader, views_per_step=1)`: drop-ins for the two Trainer methods.  Swap them
  together: `train_step` already runs the backward and the update, so the reference's `train_one_epoch` must not run them again.
  `views_per_step` G > 1 groups consecutive novel-view items up to G per `step_views`; front items still run alone.  Memory stays
  bounded by G: StableDiffusion keeps one multi-view engine, at G, and a group with another number of guided views (cut short by a
  front item, the end of the epoch or diff_iters) runs its guidance view by view on the single-view engine.

What the iteration computes is the reference's: the render at data's H x W; bilinear upsampling (align_corners=True) of the image and
depth to 512^2; the gt composite on a random background; opacity (x10 on large views), entropy (x1 before diff_iters, x10 after),
orientation counted 1 + 1 before diff_iters and 1 + 10 after, smoothness; on front views lambda_img L1 + lambda_depth (1 - pearson);
on the others the guidance (skipped before diff_iters; text_z[1] / tokens[1] on large views) and lambda_clip (img_clip + img_text_clip)
on the upsampled render.  The denoise branch (t <= 400, not large) runs under no_grad: its CLIP value joins the loss without a gradient.

Differences, by design:
* `loss` is the reference's loss value; on SDS iterations the backward also carries the surrogate, whose value is not part of it;
* the Pearson coefficient is torchmetrics' formula in fp64 over the masked pixels without a boolean-mask compaction (no host sync);
* `train_one_epoch` accumulates the loss on the device and reads it once per epoch (the reference reads it every step), and prints
  nothing per step;
* `--fp16`, multi-GPU, CPU tensors and reference images other than 512^2 are refused with `Mi3dError`.

Several views per iteration (`step_views`, `views_per_step` G > 1).  View v of a group started at global_step counts as step
global_step + 1 + v for every per-step rule (opacity x10 on large views, entropy / orientation x1 or x10 around diff_iters, the guidance
skipped before diff_iters, text_z[1] / tokens[1] on large views).  The iteration's loss and gradient are the sum of the G single-view
iterations' (the definition SURVEY 8e uses for G ranks), followed by ONE optimizer step.  Where it departs from G reference iterations:
* one shading draw per group, at the first view's step (each view keeps the reference's marginal distribution, but the views of a
  group share it);
* one timestep t shared by the group's guidance;
* one optimizer step (and one gradient clip) instead of G;
* the density grid is refreshed at most once per group, when the group crosses a multiple of update_extra_interval.
"""
import ctypes as C
import os
import random

import torch
import torch.nn.functional as F

from .. import _lib as L
from ..optimizer import Adam, Adan
from .refine import _png
from .utils import safe_normalize

REF_HW = 512                     # the reference image and the upsample target (main.py:184, utils.py:551)
CLIP_GRAD_NORM = 10.0            # nn.utils.clip_grad_norm(model.parameters(), max_norm=10) (utils.py:984)


class _CoarseLosses(torch.autograd.Function):
    """terms [4], pred512, gt512 of one iteration (mi3d_coarse_losses); the backward is mi3d_coarse_losses_backward"""

    @staticmethod
    def forward(ctx, image, depth, ws, ref, bg, prior, mask, h, w, front):
        dev = image.device
        f32 = dict(dtype=torch.float32, device=dev)
        pred512 = torch.empty(1, 3, REF_HW, REF_HW, **f32)
        gt512 = torch.empty(1, 3, REF_HW, REF_HW, **f32)
        terms = torch.empty(4, **f32)
        lib = L.lib()
        work = torch.empty(lib.mi3d_coarse_losses_workspace_bytes(C.c_uint32(h), C.c_uint32(w)), dtype=torch.uint8, device=dev)
        L.check(lib.mi3d_coarse_losses(L.ptr(image), L.ptr(depth), L.ptr(ws), C.c_uint32(h), C.c_uint32(w), L.ptr(ref), L.ptr(bg),
                                       L.ptr(prior), L.ptr(mask), C.c_int(int(front)), L.ptr(pred512), L.ptr(gt512), L.ptr(terms),
                                       L.ptr(work), C.c_size_t(work.numel()), L.stream()), "coarse_losses")
        ctx.save_for_backward(ws, pred512, gt512, prior, mask, work)
        ctx.h, ctx.w, ctx.front = h, w, front
        ctx.mark_non_differentiable(gt512)
        ctx.set_materialize_grads(False)
        return terms, pred512, gt512

    @staticmethod
    def backward(ctx, g_terms, g_pred, _g_gt):
        ws, pred512, gt512, prior, mask, work = ctx.saved_tensors
        h, w = ctx.h, ctx.w
        dev = ws.device
        g_terms = torch.zeros(4, dtype=torch.float32, device=dev) if g_terms is None else L.f32c(g_terms)
        g_pred = L.f32c(g_pred) if g_pred is not None else None
        g_image = torch.empty(h * w, 3, dtype=torch.float32, device=dev)
        g_depth = torch.empty(h * w, dtype=torch.float32, device=dev)
        g_ws = torch.empty(h * w, dtype=torch.float32, device=dev)
        L.check(L.lib().mi3d_coarse_losses_backward(L.ptr(ws), C.c_uint32(h), C.c_uint32(w), L.ptr(pred512), L.ptr(gt512), L.ptr(prior),
                                                    L.ptr(mask), C.c_int(int(ctx.front)), L.ptr(g_terms), L.ptr(g_pred), L.ptr(work),
                                                    C.c_size_t(work.numel()), L.ptr(g_image), L.ptr(g_depth), L.ptr(g_ws), L.stream()),
                "coarse_losses_backward")
        return g_image, g_depth, g_ws, None, None, None, None, None, None, None


def coarse_losses(image, depth, weights_sum, h, w, ref_imgs, bg_color, depth_prior, mask, front):
    """(terms [4] = (mean ws^2, entropy, front ? L1 : 0, front ? pearson : 0), pred512 [1,3,512,512], gt512 [1,3,512,512]) of one
    h x w render.  image [h*w,3] (or any shape holding it ray-major), depth / weights_sum [h*w]; ref_imgs [1,4,512,512]; bg_color [3];
    depth_prior fp64 [512,512]; mask uint8 [512,512] (nonzero: the pixels of the depth term).  All on the GPU."""
    L.require_cuda(image, depth, weights_sum, ref_imgs, bg_color, depth_prior, mask)
    h, w = int(h), int(w)
    if h < 2 or w < 2:
        raise L.Mi3dError(f"coarse_losses: the render must be at least 2 x 2, got {h} x {w}")
    image, depth, weights_sum = L.f32c(image).reshape(-1, 3), L.f32c(depth).reshape(-1), L.f32c(weights_sum).reshape(-1)
    if image.shape[0] != h * w or depth.numel() != h * w or weights_sum.numel() != h * w:
        raise L.Mi3dError(f"coarse_losses: image [{h * w},3], depth and weights_sum [{h * w}] expected, got {tuple(image.shape)}, "
                          f"{tuple(depth.shape)}, {tuple(weights_sum.shape)}")
    if tuple(ref_imgs.shape) != (1, 4, REF_HW, REF_HW):
        raise L.Mi3dError(f"coarse_losses: the reference image must be RGBA [1,4,{REF_HW},{REF_HW}], got {tuple(ref_imgs.shape)}")
    if depth_prior.dtype != torch.float64 or depth_prior.numel() != REF_HW * REF_HW or mask.dtype != torch.uint8 or mask.numel() != REF_HW * REF_HW:
        raise L.Mi3dError(f"coarse_losses: depth prior fp64 and mask uint8 [{REF_HW},{REF_HW}] expected")
    bg = L.f32c(bg_color).reshape(3)
    return _CoarseLosses.apply(image, depth, weights_sum, L.f32c(ref_imgs), bg, depth_prior.contiguous(), mask.contiguous(), h, w,
                               bool(front))


def pick_shading(global_step, is_front, albedo_iters):
    """the reference's shading draw (utils.py:470-483) -> (shading, ambient_ratio)"""
    if global_step < albedo_iters or is_front:
        return 'albedo', 1.0
    rand = random.random()
    if rand > 0.5:
        return 'albedo', 1.0
    if rand > 0.4:
        return 'textureless', 0.1
    return 'lambertian', 0.1


class CoarseStep:
    """state and iteration of the coarse stage (nerf/utils.py:461-574 + :977-986); see the module docstring"""

    def __init__(self, model, guidance, clip_model, optimizer, opt, ref_imgs, depth_prediction, depth_mask, text_z, clip_text_tokens):
        if getattr(opt, "fp16", False):
            raise L.Mi3dError("the coarse step runs in fp32 only (--fp16's autocast + GradScaler is not built)")
        for name, t in (("ref_imgs", ref_imgs), ("depth_prediction", depth_prediction), ("depth_mask", depth_mask),
                        ("clip_text_tokens", clip_text_tokens)):
            if not torch.is_tensor(t) or not t.is_cuda:
                raise L.Mi3dError(f"CoarseStep: {name} must be a CUDA tensor (there is no CPU path)")
        if tuple(ref_imgs.shape) != (1, 4, REF_HW, REF_HW):
            raise L.Mi3dError(f"CoarseStep: the reference image must be RGBA [1,4,{REF_HW},{REF_HW}] (main.py:184), got {tuple(ref_imgs.shape)}")
        if depth_prediction.numel() != REF_HW * REF_HW or depth_mask.numel() != REF_HW * REF_HW:
            raise L.Mi3dError(f"CoarseStep: depth_prediction and depth_mask must hold {REF_HW} x {REF_HW} values")
        if not isinstance(optimizer, (Adan, Adam)):
            raise L.Mi3dError("CoarseStep: the optimizer must be this package's Adan or Adam (optimizer.Adan / optimizer.Adam)")
        if optimizer.clip_grad_norm == 0.0:
            optimizer.clip_grad_norm = CLIP_GRAD_NORM            # the Trainer's clip_grad_norm(model.parameters(), 10), folded in
        elif optimizer.clip_grad_norm != CLIP_GRAD_NORM:
            raise L.Mi3dError(f"CoarseStep: {type(optimizer).__name__}(clip_grad_norm={optimizer.clip_grad_norm}) given; "
                              f"the Trainer clips at {CLIP_GRAD_NORM}")
        tokens = clip_text_tokens.to(torch.long)
        if tokens.dim() != 2 or tokens.shape[0] != len(text_z):
            raise L.Mi3dError(f"CoarseStep: clip_text_tokens must be [{len(text_z)},77] int64, one row per text entry; got {tuple(tokens.shape)}")
        self.model, self.guidance, self.clip, self.optimizer, self.opt = model, guidance, clip_model, optimizer, opt
        self.ref = L.f32c(ref_imgs)
        self.prior = depth_prediction.reshape(REF_HW, REF_HW).to(torch.float64).contiguous()
        self.mask = (depth_mask.reshape(REF_HW, REF_HW) == 0).to(torch.uint8).contiguous()      # ~depth_mask (utils.py:556)
        self.text_z, self.tokens = text_z, tokens.contiguous()
        self.last = None
        # step_views: the number of guided views whose guidance runs as one batch (the size StableDiffusion keeps its one multi-view
        # engine at; train_one_epoch sets views_per_step); other sizes run view by view.  None: every size is batched.
        self.guidance_views = None

    def step(self, data, global_step, *, shading=None, bg_color=None, t=None, noise=None, eps_posterior=None, noises=None, light_d=None,
             step_seed=None):
        """one iteration on the loader batch `data` (rays_o, rays_d, depth_scale, H, W, is_front, is_large) at global_step.  The
        keyword arguments inject the random draws (shading name, background [3], guidance t / noise / eps_posterior, march jitter
        noises [N], light direction [3]; step_seed keys the smoothness perturbation by sample position, as in step_views).  Returns {'loss', 'opacity', 'entropy', 'orient', 'smooth', and 'l1', 'depth' (front) or
        'clip', 'guidance'} as device scalars (l1 = lambda_img L1, depth = lambda_depth (1 - pearson), clip = lambda_clip (img + text),
        guidance = the denoise branch's CLIP value, 0 otherwise).  `last` keeps pred512, gt512, the depth, weights_sum and the
        denoised image of this iteration for the PNG dumps."""
        opt, gd = self.opt, self.guidance
        is_front, is_large = bool(data['is_front']), bool(data['is_large'])
        H, W = int(data['H']), int(data['W'])
        if shading is None:
            shading, ambient_ratio = pick_shading(global_step, is_front, opt.albedo_iters)
        else:
            ambient_ratio = 1.0 if shading == 'albedo' else 0.1
        rays_o, rays_d = data['rays_o'], data['rays_d']
        L.require_cuda(rays_o, rays_d)
        dev = rays_o.device
        self.optimizer.zero_grad()
        if bg_color is None:
            bg_color = torch.rand(3, device=dev)                                       # utils.py:491, on the device
        if light_d is None:
            light_d = safe_normalize(rays_o.reshape(-1, 3)[0] + torch.randn(3, device=dev))   # renderer.py:496-499, on the device
        kw = dict(vars(opt))
        kw.update(depth_scale=data['depth_scale'], bg_color=bg_color, staged=False, perturb=True, ambient_ratio=ambient_ratio,
                  shading=shading, force_all_rays=True, light_d=light_d, noises=noises)
        if step_seed is not None:
            kw.update(step_seed=step_seed)
        out = self.model.render(rays_o, rays_d, **kw)
        terms, pred512, gt512 = coarse_losses(out['image'], out['depth'], out['weights_sum'], H, W, self.ref, bg_color, self.prior,
                                              self.mask, is_front)
        k = 1 if is_large else 0
        text_z, tokens = self.text_z[k], self.tokens[k:k + 1]
        surrogate, de_imgs, gval = None, None, None
        if not (global_step < opt.diff_iters or is_front):
            if t is None:
                t = int(torch.randint(gd.min_step, gd.max_step + 1, [1]).item())      # train_step's draw, CPU generator: no sync
            pred_rgb = out['image'].reshape(1, H, W, 3).permute(0, 3, 1, 2)            # a view: the graph holds no copy
            gkw = dict(ref_rgb=gt512, noise=noise, ref_text=tokens, clip_model=self.clip, guidance_scale=opt.guidance_scale, t=t,
                       eps_posterior=eps_posterior)
            if not is_large and t / gd.num_train_timesteps <= 0.4:
                with torch.no_grad():
                    g, de_imgs = gd.train_step(text_z, pred_rgb.detach(), islarge=False, **gkw)
                gval = g if torch.is_tensor(g) else pred512.new_full((), float(g))
            else:
                surrogate, _ = gd.train_step(text_z, pred_rgb, islarge=is_large, defer=True, **gkw)
                gval = pred512.new_zeros(())
        loss = 0 if gval is None else gval
        if opt.lambda_opacity > 0:
            loss = loss + (opt.lambda_opacity * terms[0] * 10 if is_large else opt.lambda_opacity * terms[0])
        if opt.lambda_entropy > 0:
            loss = loss + (opt.lambda_entropy * terms[1] if global_step < opt.diff_iters else opt.lambda_entropy * terms[1] * 10)
        zero = pred512.new_zeros(())
        orient, smooth = out.get('loss_orient', zero), out.get('loss_smooth', zero)
        if opt.lambda_orient > 0 and 'loss_orient' in out:
            loss = loss + opt.lambda_orient * orient
            loss = loss + (opt.lambda_orient * orient if global_step < opt.diff_iters else opt.lambda_orient * orient * 10)
        if opt.lambda_smooth > 0 and 'loss_smooth' in out:
            loss = loss + opt.lambda_smooth * smooth
        if is_front:
            l1 = opt.lambda_img * terms[2]
            dep = opt.lambda_depth * (1 - terms[3])
            loss_ref = l1 + dep
            res = dict(l1=l1.detach(), depth=dep.detach())
        else:
            img_l, text_l = self.clip.losses(pred512, gt512, tokens)
            loss_ref = opt.lambda_clip * img_l + opt.lambda_clip * text_l
            res = dict(clip=loss_ref.detach(), guidance=gval.detach() if gval is not None else zero)
        loss = loss + loss_ref
        (loss if surrogate is None else loss + surrogate).backward()
        self.optimizer.step()
        res.update(loss=loss.detach(), opacity=terms[0].detach(), entropy=terms[1].detach(), orient=orient.detach(),
                   smooth=smooth.detach())
        self.last = dict(pred512=pred512.detach(), gt512=gt512, depth=out['depth'].detach(), H=H, W=W,
                         weights_sum=out['weights_sum'].detach().reshape(1, 1, H, W), denoised=de_imgs)
        return res

    def step_views(self, datas, global_step, *, shading=None, bg_color=None, t=None, noise=None, eps_posterior=None, noises=None,
                   light_d=None, step_seed=None):
        """one iteration over the G novel-view loader batches `datas` (same H x W, none is_front); view v counts as step
        global_step + 1 + v (see the module docstring).  Injectable draws as in `step`, batched: bg_color [G,3], light_d [G,3], noises
        [G*H*W], noise / eps_posterior [G,4,h,w]; one shading and one t for the group.  Returns the same keys as `step`, each the sum
        over the views; `last_views` keeps each view's `last` dict (`last` is the final view's).  G = 1 is `step`."""
        G = len(datas)
        if G == 1:
            pick = lambda x: x[0] if x is not None else None
            return self.step(datas[0], global_step + 1, shading=shading, bg_color=pick(bg_color), t=t, noise=noise, eps_posterior=eps_posterior,
                             noises=noises, light_d=pick(light_d), step_seed=step_seed)
        opt, gd = self.opt, self.guidance
        H, W = int(datas[0]['H']), int(datas[0]['W'])
        if not 1 <= G <= L.MAX_VIEWS or any(bool(d['is_front']) or (int(d['H']), int(d['W'])) != (H, W) for d in datas):
            raise L.Mi3dError(f"step_views takes 1..{L.MAX_VIEWS} novel (not is_front) views of one size; got {G}")
        steps = [global_step + 1 + v for v in range(G)]
        large = [bool(d['is_large']) for d in datas]
        if shading is None:
            shading, ambient_ratio = pick_shading(steps[0], False, opt.albedo_iters)
        else:
            ambient_ratio = 1.0 if shading == 'albedo' else 0.1
        rays_o = torch.cat([d['rays_o'].reshape(1, H * W, 3) for d in datas])
        rays_d = torch.cat([d['rays_d'].reshape(1, H * W, 3) for d in datas])
        depth_scale = torch.cat([d['depth_scale'].reshape(1, H * W) for d in datas])
        L.require_cuda(rays_o, rays_d)
        dev = rays_o.device
        self.optimizer.zero_grad()
        if bg_color is None:
            bg_color = torch.rand(G, 3, device=dev)
        if light_d is None:
            light_d = safe_normalize(rays_o[:, 0] + torch.randn(G, 3, device=dev))
        kw = dict(vars(opt))
        kw.update(depth_scale=depth_scale, bg_color=bg_color, staged=False, perturb=True, ambient_ratio=ambient_ratio, shading=shading,
                  force_all_rays=True, light_d=light_d, noises=noises)
        if step_seed is not None:
            kw.update(step_seed=step_seed)
        out = self.model.render(rays_o, rays_d, **kw)
        per_view = [coarse_losses(out['image'][v], out['depth'][v], out['weights_sum'][v], H, W, self.ref, bg_color[v], self.prior, self.mask, False)
                    for v in range(G)]
        zero = out['image'].new_zeros(())
        # guidance: one batched call over the views at or past diff_iters
        gv = [v for v in range(G) if steps[v] >= opt.diff_iters]
        surrogate, gval, de_imgs = None, zero, [None] * G
        if gv:
            if t is None:
                t = int(torch.randint(gd.min_step, gd.max_step + 1, [1]).item())      # train_step's draw, CPU generator: no sync
            # views picked by slices (a list index would copy the index to the device and synchronise)
            sub = lambda x: (x if len(gv) == G else torch.cat([x[v:v + 1] for v in gv])) if x is not None else None
            pred_rgb = sub(out['image']).reshape(len(gv), H, W, 3).permute(0, 3, 1, 2)
            ks = [1 if large[v] else 0 for v in gv]
            gkw = dict(ref_rgb=torch.cat([per_view[v][2] for v in gv]), noise=sub(noise), ref_text=torch.cat([self.tokens[k:k + 1] for k in ks]),
                       clip_model=self.clip, guidance_scale=opt.guidance_scale, t=t, eps_posterior=sub(eps_posterior))
            if len(gv) > 1 and self.guidance_views in (None, len(gv)):
                te = self.text_z[ks[0]] if len(set(ks)) == 1 else torch.cat([self.text_z[k][:1] for k in ks] + [self.text_z[k][1:] for k in ks])
                surrogate, imgs = gd.train_step(te, pred_rgb, islarge=[large[v] for v in gv], defer=True, **gkw)
                g = gd.last['denoise']
                gval = g if torch.is_tensor(g) else zero + float(g)
                for i, v in enumerate(gv):
                    de_imgs[v] = imgs[i]
            else:
                # view by view on the constructor's engine, exactly as `step` calls it (one guided view, or a group size the multi-view
                # engine is not kept at: planning one per size would hold a 10-34 GiB engine for every size met)
                for i, v in enumerate(gv):
                    one = dict(gkw, ref_rgb=gkw['ref_rgb'][i:i + 1], ref_text=gkw['ref_text'][i:i + 1],
                               noise=gkw['noise'][i:i + 1] if noise is not None else None,
                               eps_posterior=gkw['eps_posterior'][i:i + 1] if eps_posterior is not None else None)
                    if not large[v] and t / gd.num_train_timesteps <= 0.4:
                        with torch.no_grad():
                            g, de_imgs[v] = gd.train_step(self.text_z[ks[i]], pred_rgb[i:i + 1].detach(), islarge=False, **one)
                        gval = gval + (g if torch.is_tensor(g) else float(g))
                    else:
                        sv, _ = gd.train_step(self.text_z[ks[i]], pred_rgb[i:i + 1], islarge=large[v], defer=True, **one)
                        surrogate = sv if surrogate is None else surrogate + sv
        loss, res, clip_surrogate = gval, dict(clip=zero, opacity=zero, entropy=zero, orient=zero, smooth=zero), zero
        self.last_views = []
        for v in range(G):
            terms, pred512, gt512 = per_view[v]
            before = steps[v] < opt.diff_iters
            if opt.lambda_opacity > 0:
                loss = loss + (opt.lambda_opacity * terms[0] * 10 if large[v] else opt.lambda_opacity * terms[0])
            if opt.lambda_entropy > 0:
                loss = loss + (opt.lambda_entropy * terms[1] if before else opt.lambda_entropy * terms[1] * 10)
            orient = out['loss_orient'][v] if 'loss_orient' in out else zero
            smooth = out['loss_smooth'][v] if 'loss_smooth' in out else zero
            if opt.lambda_orient > 0 and 'loss_orient' in out:
                loss = loss + opt.lambda_orient * orient
                loss = loss + (opt.lambda_orient * orient if before else opt.lambda_orient * orient * 10)
            if opt.lambda_smooth > 0 and 'loss_smooth' in out:
                loss = loss + opt.lambda_smooth * smooth
            k = 1 if large[v] else 0
            img_l, text_l = self.clip.losses(pred512, gt512, self.tokens[k:k + 1])
            loss_ref = opt.lambda_clip * img_l + opt.lambda_clip * text_l
            # the CLIP backward runs now, while this view's tape is the CLIP engine's: in the one backward below the G views' image
            # towers would each have to be run forward again first.  Its gradient joins as a surrogate, like the SDS gradient.
            (g_pred,) = torch.autograd.grad(loss_ref, pred512)
            clip_surrogate = clip_surrogate + (g_pred * pred512).sum()
            loss = loss + loss_ref.detach()
            for name, val in (('clip', loss_ref), ('opacity', terms[0]), ('entropy', terms[1]), ('orient', orient), ('smooth', smooth)):
                res[name] = res[name] + val.detach()
            self.last_views.append(dict(pred512=pred512.detach(), gt512=gt512, depth=out['depth'][v].detach(), H=H, W=W,
                                        weights_sum=out['weights_sum'][v].detach().reshape(1, 1, H, W), denoised=de_imgs[v]))
        (loss + clip_surrogate if surrogate is None else loss + clip_surrogate + surrogate).backward()
        self.optimizer.step()
        res.update(loss=loss.detach(), guidance=gval.detach())
        self.last = self.last_views[-1]
        return res


def _coarse_step(trainer):
    cs = getattr(trainer, "_coarse_step", None)
    if cs is None:
        if getattr(trainer, "fp16", False):
            raise L.Mi3dError("the coarse step runs in fp32 only (--fp16's autocast + GradScaler is not built)")
        tokens = getattr(trainer, "clip_text_tokens", None)
        if tokens is None:
            raise L.Mi3dError("the coarse step needs trainer.clip_text_tokens: the CLIP token ids of trainer.text ([2,77] int64; "
                              "there is no BPE tokenizer here)")
        cs = CoarseStep(trainer.model, trainer.guidance, trainer.clip_model, trainer.optimizer, trainer.opt, trainer.ref_imgs,
                        trainer.depth_prediction, trainer.depth_mask, trainer.text_z, tokens)
        trainer._coarse_step = cs
    return cs


def _save_pngs(trainer, cs, last=None, step=None):
    """the reference's dumps at global_step % 100 == 0 or == 1 (utils.py:565-571); save_image clamps to [0, 1].  last / step: a view
    of a multi-view iteration and its step number (default: cs.last at trainer.global_step)"""
    last, step, path = last or cs.last, trainer.global_step if step is None else step, trainer.img_path
    os.makedirs(path, exist_ok=True)
    with torch.no_grad():
        # the upsampled depth only feeds this dump (the loss kernel keeps its own copy), once per 100 steps
        depth = F.interpolate(last['depth'].reshape(1, 1, last['H'], last['W']), (REF_HW, REF_HW), mode='bilinear', align_corners=True)
        prior = (cs.prior * cs.mask)[None, None].float()
        for img, name in ((last['pred512'], f"{step}.png"), (last['gt512'], f"{step}_gt.png"), (depth, f"{step}_depth.png"),
                          (prior, f"{step}_ref_depth_mask.png"), (last['denoised'], f"{step}_denoise.png")):
            if img is not None:
                _png(img.expand(1, 3, *img.shape[-2:]).clamp(0, 1), os.path.join(path, name))


def train_step(trainer, data):
    """drop-in for Trainer.train_step (nerf/utils.py:461-574) that also runs the backward and the optimiser step (swap
    train_one_epoch with it).  Returns (pred_rgb512, pred_ws, loss) like the reference; loss is a detached device scalar."""
    cs = _coarse_step(trainer)
    res = cs.step(data, trainer.global_step)
    if trainer.global_step % 100 == 0 or trainer.global_step == 1:
        _save_pngs(trainer, cs)
    return cs.last['pred512'], cs.last['weights_sum'], res['loss']


def _dump_due(step):
    return step % 100 == 0 or step == 1


def train_one_epoch(trainer, loader, views_per_step=1):
    """drop-in for Trainer.train_one_epoch (nerf/utils.py:947-1027): density-grid update every update_extra_interval steps, one
    coarse iteration per batch, the scheduler step; the loss is summed on the device and read once, for stats["loss"] and the log.
    views_per_step G > 1: consecutive novel-view batches run G at a time through `CoarseStep.step_views` (a shorter group where a front
    view or the end of the epoch cuts it), front views alone through `step`; global_step, the scheduler and the density-grid refresh
    advance by views, so the step numbers and schedules are those of the one-view loop."""
    if getattr(trainer, "world_size", 1) > 1:
        raise L.Mi3dError("the coarse step is single-GPU (multi-GPU coarse training is not built)")
    G = int(views_per_step)
    if not 1 <= G <= L.MAX_VIEWS:
        raise L.Mi3dError(f"views_per_step must be in 1..{L.MAX_VIEWS}; got {views_per_step}")
    if G > 1:
        _coarse_step(trainer).guidance_views = G
    trainer.log(f"==> Start Training {trainer.workspace} Epoch {trainer.epoch}, lr={trainer.optimizer.param_groups[0]['lr']:.6f} ...")
    trainer.model.train()
    trainer.local_step = 0
    total = None

    def run(group):
        nonlocal total
        n, start = len(group), trainer.global_step
        if trainer.model.cuda_ray and any((start + v) % trainer.opt.update_extra_interval == 0 for v in range(n)):
            trainer.model.update_extra_state()
        trainer.local_step += n
        trainer.global_step += n
        if n == 1:
            _, _, loss = train_step(trainer, group[0])
        else:
            cs = _coarse_step(trainer)
            loss = cs.step_views(group, start)['loss']
            due = [v for v in range(n) if _dump_due(start + 1 + v)]
            if due:
                _save_pngs(trainer, cs, cs.last_views[due[0]], start + 1 + due[0])
        total = loss if total is None else total + loss
        if trainer.scheduler_update_every_step:
            for _ in range(n):
                trainer.lr_scheduler.step()

    group = []
    for data in loader:
        if G > 1 and not data['is_front']:
            group.append(data)
            if len(group) == G:
                run(group)
                group = []
            continue
        if group:
            run(group)
            group = []
        run([data])
    if group:
        run(group)
    if getattr(trainer, "ema", None) is not None:
        trainer.ema.update()
    average_loss = float(total) / trainer.local_step if trainer.local_step else 0.0
    trainer.stats["loss"].append(average_loss)
    if not trainer.scheduler_update_every_step:
        if isinstance(trainer.lr_scheduler, torch.optim.lr_scheduler.ReduceLROnPlateau):
            trainer.lr_scheduler.step(average_loss)
        else:
            trainer.lr_scheduler.step()
    trainer.log(f"==> Finished Epoch {trainer.epoch}. loss={average_loss:.4f}")
