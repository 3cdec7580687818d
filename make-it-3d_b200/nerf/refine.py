"""B11 seam: the refine stage's training loop (reference `Trainer.refine`, nerf/utils.py:747-944) on libmi3d.so.

* `RefineStep(vertices_cano, colours_cano, vertices_novel, colours_novel, K, unet, cx, clip, guidance, text_z, gt_rgb, gt_mask,
  clip_text_tokens, seed)`: the state of one refine run and its iteration.  The cloud's colours and features live in one contiguous
  fp32 leaf `points` [P,19] (cano rows first, then novel; columns 0-2 colours, 3-18 features), so the three renders read it without
  the reference's per-iteration `torch.cat`s.  `step(world2cam, is_front, t=None, noise=None, eps_posterior=None)` runs one iteration
  as one autograd graph with one backward, then one `mi3d_refine_adam` launch updates the cloud and every U-Net parameter.  It
  returns the loss terms as device scalars and never synchronises the host.
* `refine(trainer, load_dir, train_iters, test_poses)`: the body of `Trainer.refine` end to end (point clouds, loop, checkpoints,
  final renders).

What the iteration computes is the reference's: three renders at 800 / 400 / 200 through the train-mode U-Net; on front iterations
(every 4th) 1000 L1(pred m, gt m); otherwise the guidance step (t > 400: SDS, t <= 400: the denoise branch, whose CLIP value carries no
gradient), 10 img_clip_loss(pred, gt) and the contextual loss; always 1e-3 sum(1 - pred (1 - maxpool5(mask))) and the two colour
regularisers; Adam (0.9, 0.99), eps 1e-15, lr 1e-3 (the reference's scheduler is never stepped).

The SDS gradient never reaches the parameters in the reference: `guidance.train_step` back-propagates it into `.grad` (nerf/sd.py:171),
and then `point_optimizer.zero_grad()` (utils.py:892) clears it before `loss.backward()`; the branch's returned loss is 0.  So on
t > 400 iterations `step` draws t like `train_step` does and does not run the guidance at all: same parameters, same loss value, none
of the VAE encode, U-Net, and the two discarded render / U-Net backwards.  On t <= 400 the denoise branch runs as in the reference.

Differences, by design:
* the coverage mask comes from the scale-0 render's composite weights (bit-identical to rendering the cloud again with unit colours);
* the CLIP embedding of gt_rgb is computed once (the CLIP weights are frozen and gt_rgb never changes);
* `points.grad` holds the image-loss gradient; the regulariser gradient is added inside the Adam launch;
* the pose sampler draws from host generators (the reference draws from the CUDA generator), with the reference's distribution;
* the loop runs at 800 x 800 throughout (the reference's first iteration uses opt.H x opt.W, every later one 800; opt.H = opt.W = 800
  is required).
"""
import ctypes as C
import glob
import os
import random

import numpy as np
import torch

from .. import _lib as L
from .clip import _EncodeImage
from .refine_utils import load_views, render_point, render_point_weights

S0 = 800                                  # refine raster (nerf/utils.py:865)
RADIUS = 2.0 / 800.0 * 2.0                # 2 pixels at 800, in NDC (utils.py:765, 807)
PPP = 8                                   # points per pixel (utils.py:766)
LR, BETAS, EPS = 1e-3, (0.9, 0.99), 1e-15
REG_W_NOVEL, REG_W_CANO = 1e3, 1e5        # utils.py:887
N_FEAT = 16


def level_K(K, j):
    """the reference's K_ of level j (render size S0 / 2^j) from the S0 intrinsics, fp32: halving focal * w and 0.5 * w is exact"""
    k = np.array(K.detach().cpu().numpy() if torch.is_tensor(K) else K, dtype=np.float64).reshape(3, 3)
    k[:2] /= 2.0 ** j
    return torch.from_numpy(k).float()


class _ImageLosses(torch.autograd.Function):
    """losses [2] = (bg_loss, l1) of one iteration (mi3d_refine_image_losses); also returns the coverage and its dilation"""

    @staticmethod
    def forward(ctx, pred, weights, gt, mask, front, ws):
        S, ppp = weights.shape[0], weights.shape[2]
        dev = pred.device
        cover = torch.empty(S, S, dtype=torch.float32, device=dev)
        dil = torch.empty(S, S, dtype=torch.float32, device=dev)
        losses = torch.empty(2, dtype=torch.float32, device=dev)
        L.check(L.lib().mi3d_refine_image_losses(L.ptr(weights), C.c_uint32(S), C.c_uint32(ppp), L.ptr(pred), L.ptr(gt), L.ptr(mask),
                                                 C.c_int(int(front)), L.ptr(cover), L.ptr(dil), L.ptr(losses), L.ptr(ws),
                                                 C.c_size_t(ws.numel()), L.stream()), "refine_image_losses")
        ctx.save_for_backward(pred, gt, mask, dil)
        ctx.front = front
        ctx.mark_non_differentiable(cover, dil)
        return losses, cover, dil

    @staticmethod
    def backward(ctx, g, _gc, _gd):
        pred, gt, mask, dil = ctx.saved_tensors
        S = dil.shape[0]
        dpred = torch.empty_like(pred)
        L.check(L.lib().mi3d_refine_image_losses_backward(L.ptr(pred), L.ptr(gt), L.ptr(mask), L.ptr(dil), C.c_uint32(S), C.c_int(int(ctx.front)),
                                                          L.ptr(L.f32c(g)), L.ptr(dpred), L.stream()), "refine_image_losses_backward")
        return dpred, None, None, None, None, None


def image_losses(pred, weights, gt, mask, front):
    """(bg_loss, l1, coverage [S,S], dilated [S,S]) of nerf/utils.py:867-886 from the scale-0 composite weights [S,S,ppp]"""
    L.require_cuda(pred, weights, gt, mask)
    S = weights.shape[0]
    if tuple(pred.shape) != (1, 3, S, S) or tuple(gt.shape) != (1, 3, S, S) or tuple(mask.shape) != (1, 1, S, S):
        raise L.Mi3dError(f"image_losses: pred / gt [1,3,{S},{S}] and mask [1,1,{S},{S}] expected, got {tuple(pred.shape)}, "
                          f"{tuple(gt.shape)}, {tuple(mask.shape)}")
    nbytes = L.lib().mi3d_refine_image_losses_workspace_bytes(C.c_uint32(S))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=pred.device)
    losses, cover, dil = _ImageLosses.apply(L.f32c(pred), L.f32c(weights), L.f32c(gt), L.f32c(mask), bool(front), ws)
    return losses[0], losses[1], cover, dil


class Adam:
    """torch.optim.Adam(betas, eps, lr) over a fixed list of fp32 CUDA leaves as one mi3d_refine_adam launch.  With `origin`, leaf 0 is
    the [p_cano + p_novel, 19] cloud and the colour regularisers are added to its gradient.  The leaves' `.grad` tensors are allocated
    here once and zeroed by `zero_grad()`, so the device table of segments stays valid."""

    def __init__(self, params, origin=None, p_cano=0, p_novel=0, lr=LR, betas=BETAS, eps=EPS):
        self.params = list(params)
        for p in self.params:
            if p.dtype != torch.float32 or not p.is_cuda or not p.is_contiguous():
                raise L.Mi3dError("Adam: parameters must be contiguous fp32 CUDA tensors")
            p.grad = torch.zeros_like(p)
        self.exp_avg = [torch.zeros_like(p) for p in self.params]
        self.exp_avg_sq = [torch.zeros_like(p) for p in self.params]
        self.origin, self.p_cano, self.p_novel = origin, int(p_cano), int(p_novel)
        self.lr, self.betas, self.eps = lr, betas, eps
        self.steps = 0
        segs = (L.AdamSegment * len(self.params))()
        off = 0
        for s, p, m, v in zip(segs, self.params, self.exp_avg, self.exp_avg_sq):
            s.param, s.grad, s.exp_avg, s.exp_avg_sq = p.data_ptr(), p.grad.data_ptr(), m.data_ptr(), v.data_ptr()
            s.offset, s.n = off, p.numel()
            off += p.numel()
        self.total = off
        self.grad_ptrs = [p.grad.data_ptr() for p in self.params]
        dev = self.params[0].device
        self.table = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).to(dev)
        nbytes = L.lib().mi3d_refine_adam_workspace_bytes(C.c_ulonglong(off))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def zero_grad(self):
        torch._foreach_zero_([p.grad for p in self.params])

    def step(self):
        """one update; returns the regulariser value (DEVICE fp32 scalar, 0 without origin) of the parameters before it"""
        for p, g in zip(self.params, self.grad_ptrs):
            if p.grad is None or p.grad.data_ptr() != g:
                raise L.Mi3dError("Adam: a parameter's .grad was replaced (zero it with zero_grad(), do not set it to None)")
        self.steps += 1
        reg = torch.zeros(1, dtype=torch.float32, device=self.table.device)
        L.check(L.lib().mi3d_refine_adam(L.ptr(self.table), C.c_int(len(self.params)), C.c_ulonglong(self.total), C.c_double(self.lr),
                                         C.c_double(self.betas[0]), C.c_double(self.betas[1]), C.c_double(self.eps), C.c_int(self.steps),
                                         L.ptr(self.origin), C.c_uint32(self.p_cano), C.c_uint32(self.p_novel), C.c_double(REG_W_CANO),
                                         C.c_double(REG_W_NOVEL), L.ptr(reg), L.ptr(self.ws), C.c_size_t(self.ws.numel()), L.stream()),
                "refine_adam")
        return reg[0]


class RefineStep:
    """state and iteration of one refine run (nerf/utils.py:808-894); see the module docstring"""

    def __init__(self, vertices_cano, colours_cano, vertices_novel, colours_novel, K, unet, cx, clip, guidance, text_z, gt_rgb, gt_mask,
                 clip_text_tokens, seed=0):
        dev = gt_rgb.device
        L.require_cuda(gt_rgb, gt_mask)
        t = lambda a, dt: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).to(dev, dt)
        vc, vn = t(vertices_cano, torch.float64), t(vertices_novel, torch.float64)
        cc, cn = t(colours_cano, torch.float32), t(colours_novel, torch.float32)
        self.p_cano, self.p_novel = vc.shape[0], vn.shape[0]
        # all_v = torch.cat((vertices_cano, vertices_novel)).float() (utils.py:846), once
        self.all_v = torch.cat((vc, vn)).float().contiguous()
        gen = torch.Generator().manual_seed(int(seed))
        feat_cano = torch.randn(self.p_cano, N_FEAT, generator=gen)
        feat_novel = torch.randn(self.p_novel, N_FEAT, generator=gen)
        self.points = torch.cat((torch.cat((cc, feat_cano.to(dev)), -1), torch.cat((cn, feat_novel.to(dev)), -1))).contiguous().requires_grad_()
        self.origin = torch.cat((cc, cn)).contiguous()
        self.bg_feat = torch.nn.Parameter(torch.ones(1, 3 + N_FEAT, 1, 1, device=dev))     # passed to render_point, ignored there
        self.K = [level_K(K, j).to(dev) for j in range(3)]
        self.unet, self.cx, self.clip, self.guidance = unet, cx, clip, guidance
        self.text_z, self.clip_text_tokens = text_z, clip_text_tokens
        self.gt_rgb, self.gt_mask = L.f32c(gt_rgb), L.f32c(gt_mask)
        with torch.no_grad():
            z = _EncodeImage.apply(self.gt_rgb, clip.engine, 1, 0)
            self.z_gt = z / z.norm(dim=-1, keepdim=True)
        self.unet_params = list(unet.parameters())
        self.opt = Adam([self.points] + self.unet_params, origin=self.origin, p_cano=self.p_cano, p_novel=self.p_novel)
        self.kept_colours = None

    def _renders(self, feats, world2cam, weights=False):
        out, w0 = [], None
        for j in range(3):
            S = S0 >> j
            if j == 0 and weights:
                img, w0 = render_point_weights(self.all_v, feats, S, S, self.K[j], world2cam, [S, S], RADIUS, PPP)
            else:
                img = render_point(self.all_v, feats, S, S, self.K[j], world2cam, [S, S], RADIUS, PPP, bg_feat=self.bg_feat)
            out.append(img)
        return out, w0

    def clip_image_loss(self, pred):
        """img_clip_loss(pred, gt_rgb) of nerf/utils.py:436-443 against the cached gt embedding"""
        z = _EncodeImage.apply(pred, self.clip.engine, 1, 1 if (torch.is_grad_enabled() and pred.requires_grad) else 0)
        z = z / z.norm(dim=-1, keepdim=True)
        return -(z * self.z_gt).sum(-1).mean()

    def step(self, world2cam, is_front, t=None, noise=None, eps_posterior=None, keep_colours=False):
        """one iteration at the pose world2cam (DEVICE [4,4]); t / noise / eps_posterior inject the guidance's random draws.
        Returns {'loss', 'bg', 'reg', and 'l1' (front) or 'guidance', 'clip', 'cx'} as device scalars; 'loss' is the reference's
        loss value.  The drawn t is left in `last_t`.  keep_colours: keep a copy of the colours this iteration rendered
        (`kept_colours`), which is what the reference saves and renders after its last step."""
        self.opt.zero_grad()
        imgs, w0 = self._renders(self.points, world2cam, weights=True)
        pred = self.unet(imgs)
        self.last_pred = pred.detach()
        bg, l1, _, _ = image_losses(pred, w0, self.gt_rgb, self.gt_mask, is_front)
        if is_front:
            head = l1
            objective = l1 + bg
            terms = dict(l1=l1.detach())
        else:
            gd = self.guidance
            if t is None:
                t = int(torch.randint(gd.min_step, gd.max_step + 1, [1]).item())     # train_step's draw, CPU generator: no sync
            self.last_t = int(t)
            g = 0
            if self.last_t / gd.num_train_timesteps <= 0.4:
                # the denoise branch (islarge=False): its CLIP value is part of the loss and carries no gradient
                with torch.no_grad():
                    g, _ = gd.train_step(self.text_z, pred.detach(), ref_rgb=self.gt_rgb, noise=noise, islarge=False,
                                         ref_text=self.clip_text_tokens, clip_model=self.clip, guidance_scale=5, t=self.last_t,
                                         eps_posterior=eps_posterior)
            gval = g if torch.is_tensor(g) else pred.new_full((), float(g))        # a fill: no host-to-device copy
            clip_l = 10 * self.clip_image_loss(pred)
            cx_l = self.cx(pred, self.gt_rgb)
            head = (gval + clip_l) + cx_l
            objective = clip_l + cx_l + bg
            terms = dict(guidance=gval.detach(), clip=clip_l.detach(), cx=cx_l.detach())
        if keep_colours:
            self.kept_colours = self.points.detach().clone()
        objective.backward()
        reg = self.opt.step()
        terms.update(loss=((head.detach() + reg) + bg.detach()), bg=bg.detach(), reg=reg)
        return terms

    @torch.no_grad()
    def render(self, world2cam, colours=None):
        """[1,3,800,800]: the three renders through the U-Net as it is (train mode in the reference's final renders, utils.py:911)"""
        imgs, _ = self._renders((self.points if colours is None else colours).detach(), world2cam)
        return self.unet(imgs)

    def optimizer_state_dict(self):
        """torch.optim.Adam.state_dict() of the reference's six groups (colour_novel, colour_cano, feat_novel, feat_cano, bg_feat,
        unet.parameters()); bg_feat never has a gradient, so it has no state"""
        pc = self.p_cano
        regions = [(slice(pc, None), slice(0, 3)), (slice(0, pc), slice(0, 3)), (slice(pc, None), slice(3, None)), (slice(0, pc), slice(3, None))]
        pts = self.points.detach()
        leaves = [torch.nn.Parameter(pts[r].clone()) for r in regions]
        bg = torch.nn.Parameter(self.bg_feat.detach().clone())
        groups = [{"params": [p], "lr": LR} for p in leaves] + [{"params": [bg], "lr": LR}, {"params": self.unet_params, "lr": LR}]
        opt = torch.optim.Adam(groups, betas=BETAS, eps=EPS)
        if self.opt.steps:
            step = lambda: torch.tensor(float(self.opt.steps), dtype=torch.float32)
            m0, v0 = self.opt.exp_avg[0], self.opt.exp_avg_sq[0]
            for p, r in zip(leaves, regions):
                opt.state[p] = {"step": step(), "exp_avg": m0[r].clone(), "exp_avg_sq": v0[r].clone()}
            for p, m, v in zip(self.unet_params, self.opt.exp_avg[1:], self.opt.exp_avg_sq[1:]):
                opt.state[p] = {"step": step(), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        return opt.state_dict()

    def save(self, outdir, tag, colours=None):
        """the reference's checkpoint files {tag}_v_unet.pt, {tag}_v_color_unet.pt, {tag}_bg_unet.pt, {tag}_unet.pth (utils.py:896-909)"""
        torch.save(self.all_v, os.path.join(outdir, f"{tag}_v_unet.pt"))
        torch.save((self.points if colours is None else colours).detach().clone(), os.path.join(outdir, f"{tag}_v_color_unet.pt"))
        torch.save(self.bg_feat, os.path.join(outdir, f"{tag}_bg_unet.pt"))
        torch.save({"model_state_dict": self.unet.state_dict(), "optimizer_state_dict": self.optimizer_state_dict()},
                   os.path.join(outdir, f"{tag}_unet.pth"))


# ---- pose sampler: refine_utils.py:244-304 (fix_poses) on host generators ----

def _normalize(v):
    return v / torch.sqrt(torch.clamp(torch.sum(v * v, -1, keepdim=True), min=1e-20))


def fix_poses(index, gen, rnd, radius_range=(1, 1.5), theta_range=(0, 100), phi_range=(0, 360)):
    """(cam2world fp32 [4,4] on the host, is_front, is_large): fix_poses' distribution and front rule (every index % 4 == 0 is the
    fixed front view), drawing from the torch CPU generator `gen` and the random.Random `rnd`"""
    theta_range, phi_range = np.deg2rad(theta_range), np.deg2rad(phi_range)
    rand = lambda: torch.rand(1, generator=gen)
    if index % 4 == 0:
        radius = torch.ones(1)
        thetas = torch.ones(1) * (theta_range[1] - theta_range[0]) / 2 + theta_range[0]
        phis = torch.ones(1) * (phi_range[1] - phi_range[0]) / 2 + phi_range[0]
        is_front = True
    else:
        radius = rand() * (radius_range[1] - radius_range[0]) + radius_range[0]
        if phi_range[1] <= np.deg2rad(240.0) and phi_range[0] >= np.deg2rad(120.0):
            phis = rand() * (phi_range[1] - phi_range[0]) + phi_range[0]
        else:
            r = rnd.random()
            if r > 0.85:
                phis = rand() * (phi_range[1] - np.deg2rad(315.0)) + np.deg2rad(315.0)
            elif r > 0.7:
                phis = rand() * (np.deg2rad(45.0) - phi_range[0]) + phi_range[0]
            elif r > 0.5:
                phis = rand() * (np.deg2rad(315.0) - np.deg2rad(240.0)) + np.deg2rad(240.0)
            elif r > 0.3:
                phis = rand() * (np.deg2rad(120.0) - np.deg2rad(45.0)) + np.deg2rad(45.0)
            else:
                phis = rand() * (np.deg2rad(240.0) - np.deg2rad(120.0)) + np.deg2rad(120.0)
        is_front = False
        thetas = rand() * (theta_range[1] - theta_range[0]) + theta_range[0]
    p = float(phis)
    is_large = (0.0 <= p <= np.deg2rad(45)) or (np.deg2rad(315) <= p <= np.deg2rad(360))
    centers = torch.stack([radius * torch.sin(thetas) * torch.sin(phis), radius * torch.cos(thetas),
                           radius * torch.sin(thetas) * torch.cos(phis)], dim=-1)
    forward = _normalize(0 - centers)
    up = torch.tensor([[0.0, -1.0, 0.0]])
    right = _normalize(torch.cross(forward, up, dim=-1))
    up = _normalize(torch.cross(right, forward, dim=-1))
    pose = torch.eye(4, dtype=torch.float32)
    pose[:3, :3] = torch.stack((right, up, forward), dim=-1)[0]
    pose[:3, 3] = centers[0]
    return pose, is_front, is_large


def world2cam_device(cam2world, device):
    """torch.linalg.inv(cam2world) in fp32 on the device (utils.py:845) without a host synchronisation"""
    c2w = cam2world.to(torch.float32).pin_memory().to(device, non_blocking=True)
    return torch.linalg.inv_ex(c2w).inverse


def _png(img, path):
    """torchvision.utils.save_image of one [1,3,H,W] image in [0,1]"""
    import cv2
    a = img[0].mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()
    cv2.imwrite(path, np.ascontiguousarray(a[:, :, ::-1]))


def _read_rgba(path):
    """imageio.imread(path) / 255. as float64 RGBA"""
    import cv2
    im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if im is None or im.ndim != 3 or im.shape[2] != 4:
        raise L.Mi3dError(f"refine: {path} must be an RGBA image (its alpha is the reference mask)")
    return im[:, :, [2, 1, 0, 3]].astype(np.float64) / 255.0


def refine(trainer, load_dir, train_iters, test_poses, clip_text_tokens=None, seed=0, log_every=100):
    """Trainer.refine (nerf/utils.py:747-944) on the engines.  trainer supplies opt (text, ref_path, fov, H, W, radius_range,
    theta_range, phi_range), guidance (a StableDiffusion), clip_model (a nerf.clip.CLIP) and text_z; clip_text_tokens are the CLIP
    token ids of opt.text ([1,77] int64; default trainer.clip_text_tokens).  test_poses: the test loader (batches with 'poses') or
    [4,4] cam2world poses.  Writes what the reference writes under load_dir with "mvimg" replaced by "refine"; the mp4 only when
    imageio can be imported.  Returns the RefineStep."""
    import cv2

    from .contextual_loss import ContextualLoss
    from .unet import UNet
    opt = trainer.opt
    H, W = int(opt.H), int(opt.W)
    if (H, W) != (S0, S0):
        raise L.Mi3dError(f"refine runs at {S0} x {S0} (the reference renders at 800 from its second iteration on); got opt.H, opt.W = {H}, {W}")
    tokens = clip_text_tokens if clip_text_tokens is not None else getattr(trainer, "clip_text_tokens", None)
    if tokens is None:
        raise L.Mi3dError("refine: pass the CLIP token ids of the prompt (clip_text_tokens=[1,77] int64; there is no BPE tokenizer here)")
    device = torch.device("cuda")
    outputdir = load_dir.replace("mvimg", "refine")
    os.makedirs(outputdir, exist_ok=True)
    focal = 1 / (2 * np.tan(np.deg2rad(opt.fov) / 2))
    K = np.array([[focal * W, 0, 0.5 * W], [0, focal * H, 0.5 * H], [0, 0, 1]])
    cam2world_list = np.load(sorted(glob.glob(load_dir + "/*poses.npy"))[0])
    rgba = _read_rgba(opt.ref_path)
    gt_rgb = cv2.resize(rgba[:, :, :3], (H, W))
    depth_files = sorted(glob.glob(load_dir + "/*depth.png"))
    mask_files = sorted(glob.glob(load_dir + "/*mask.png"))
    rgb_files = sorted(glob.glob(load_dir + "/*rgb.png"))
    vc, cc, vn, cn = load_views(gt_rgb, rgb_files, depth_files, mask_files, cam2world_list, H, W, K, 2, PPP, outputdir, device)
    print("###### Save point cloud ######")
    np.save(outputdir + "/vertices_cano.npy", vc)
    np.save(outputdir + "/vertices_color_cano.npy", cc)
    np.save(outputdir + "/vertices_novel.npy", vn)
    np.save(outputdir + "/vertices_color_novel.npy", cn)

    print("###### Optimization with SDS loss ######")
    gt_mask = cv2.erode(cv2.resize(rgba[:, :, 3:], (H, W)), np.ones((5, 5), np.uint8), iterations=1)
    gt_mask = torch.Tensor(gt_mask)[None, None].to(device)
    gt = torch.Tensor(gt_rgb[None]).permute(0, 3, 1, 2).contiguous().to(device)
    train_outputdir = outputdir + "/train/"
    os.makedirs(train_outputdir, exist_ok=True)
    unet = UNet(num_input_channels=3 + 16).to(device)
    unet.train()
    cx = ContextualLoss(use_vgg=True, vgg_layer="relu5_4", device=device)
    tokens = torch.as_tensor(tokens).reshape(1, -1).to(device)
    rs = RefineStep(vc, cc, vn, cn, K, unet, cx, trainer.clip_model, trainer.guidance, trainer.text_z[0], gt, gt_mask, tokens, seed=seed)
    gen, rnd = torch.Generator().manual_seed(int(seed)), random.Random(int(seed))
    kw = dict(radius_range=opt.radius_range, theta_range=opt.theta_range, phi_range=opt.phi_range)
    for i in range(train_iters):
        c2w, is_front, _ = fix_poses(i, gen, rnd, **kw)
        last = i == train_iters - 1
        ckpt = i % 1000 == 0
        terms = rs.step(world2cam_device(c2w, device), is_front, keep_colours=ckpt or last)
        if i % 50 == 0:
            # the reference saves pred_rgb here, the image of this iteration's forward (before its update)
            _png(rs.last_pred, os.path.join(train_outputdir, f"{i}.png"))
        if ckpt:
            rs.save(outputdir, str(i), colours=rs.kept_colours)
        if i % log_every == 0 or last:
            print(f"refine {i}/{train_iters}: loss {float(terms['loss']):.4f}; reg_loss {float(terms['reg']):.4f}; "
                  f"bg_loss {float(terms['bg']):.4f}")
    final = rs.kept_colours
    rs.save(outputdir, "end", colours=final)

    print("###### Finel Refine Rendering ######")
    img_outdir = os.path.join(outputdir, "results")
    os.makedirs(img_outdir, exist_ok=True)
    frames = []
    for i, data in enumerate(test_poses):
        pose = data["poses"][0] if isinstance(data, dict) else data
        pose = pose.detach().cpu().numpy() if torch.is_tensor(pose) else np.asarray(pose)
        w2c = torch.from_numpy(np.linalg.inv(pose.astype(np.float64)).astype(np.float32)).to(device)
        pred = rs.render(w2c, colours=final)
        frames.append(np.array(pred[0].permute(1, 2, 0).cpu().numpy() * 255, dtype=np.uint8))
        _png(pred, img_outdir + f"/render_unet_{i:04d}.png")
    try:
        import imageio
    except ImportError:
        imageio = None
    if imageio is not None and frames:
        imageio.mimwrite(img_outdir + "/render_unet_img_clip.mp4", np.stack(frames, 0), fps=25, quality=8, macro_block_size=1)
    return rs
