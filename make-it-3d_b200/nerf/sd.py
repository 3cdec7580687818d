"""B3 seam: `StableDiffusion` guidance with the reference's constructor / method surface (nerf/sd.py:21-238) on libmi3d.so.

`train_step(text_embeddings, pred_rgb, ref_rgb=None, noise=None, islarge=False, ref_text=None, clip_model=None,
guidance_scale=10) -> (loss, imgs)` performs the SDS backward itself into pred_rgb's graph exactly like the reference
(nerf/sd.py:163-172) and returns (0, None) on that branch.  Everything between pred_rgb and the gradient runs in the
engine of csrc/sd_engine.cu (wgmma tile kernel + fused memory-bound kernels); there is no diffusers / cuDNN / cuBLAS
call and no CPU fallback.

Weights: parameters are enumerated by diffusers' state_dict names; real SD-2.x checkpoints load through
`load_diffusers_state_dict(unet_state, vae_state)` (which also pushes them into the engine); offline (no network, no weights on disk) they are seeded random tensors with PyTorch's default
initialisers -- which is what the benchmark and the parity tests use (`data: synthetic`).
SD-1.x (`sd_version='1.5'`, or `hf_key` of any SD-1.x checkpoint) runs on the same engine with its own topology (`sd15_unet_cfg`: 8 heads
of 40 / 80 / 160, cross dim 768, 1x1-conv proj_in / proj_out) and needs its checkpoint: pass `unet_state` / `vae_state` (diffusers'
`UNet2DConditionModel` / `AutoencoderKL` state_dict()s); there is no seeded SD-1.5 stand-in.  Its text encoder (OpenAI CLIP ViT-L/14,
quick-GELU) is created by `load_diffusers_state_dict(text_encoder_state=...)`.
The "denoise" side branch (nerf/sd.py:153-159: DDIM step t -> t-1, VAE decode, CLIP losses) is built on the same engine (`mi3d_sd_ddim_step`,
`mi3d_sd_decode`); the CLIP losses run on the caller-provided clip_model (the reference passes it in too) and are skipped without one.
A native `nerf.clip.CLIP` computes them on the CLIP engine (csrc/clip_engine.cu, aug included); any other model is called as before.
`get_text_embeds` runs the SD text encoder (nerf/sd_text.py, csrc/sd_text_engine.cu) once its weights are loaded with
`load_diffusers_state_dict(text_encoder_state=...)`; prompts given as strings go through the `tokenizer` passed to the constructor.
Without text-encoder weights it returns a deterministic stand-in keyed by the prompt strings.
"""
import ctypes as C
import hashlib
import math
import os

import torch
import torch.nn as nn

from .. import _lib as L
from .clip import CLIP
from .sd_text import TextEncoder, cfg_from_state_dict


class UNetCfg(C.Structure):
    _fields_ = [("in_ch", C.c_int), ("out_ch", C.c_int), ("n_levels", C.c_int), ("block_out", C.c_int * 4), ("layers_per_block", C.c_int),
                ("heads", C.c_int * 4), ("cross_dim", C.c_int), ("ctx_len", C.c_int), ("groups", C.c_int), ("latent_hw", C.c_int),
                ("batch", C.c_int), ("proj_conv", C.c_int)]


class VaeCfg(C.Structure):
    _fields_ = [("in_ch", C.c_int), ("latent_ch", C.c_int), ("n_levels", C.c_int), ("block_out", C.c_int * 4), ("layers_per_block", C.c_int),
                ("groups", C.c_int), ("image_hw", C.c_int), ("decoder", C.c_int)]


def sd20_unet_cfg(latent_hw=64):
    return dict(in_channels=4, out_channels=4, block_out=(320, 640, 1280, 1280), layers_per_block=2, heads=(5, 10, 20, 20),
                cross_dim=1024, groups=32, ctx_len=77, latent_hw=latent_hw)


def sd15_unet_cfg(latent_hw=64):
    """SD-1.x (stable-diffusion-v1-5 unet/config.json): 8 heads at every level (head_dim 40 / 80 / 160), cross dim 768 (OpenAI CLIP
    ViT-L/14 text features), 1x1-conv proj_in / proj_out (use_linear_projection false)"""
    return dict(sd20_unet_cfg(latent_hw), heads=(8, 8, 8, 8), cross_dim=768, proj_conv=True)


def is_sd1_unet_state(state):
    """an SD-1.x U-Net state_dict: its transformer projections are 1x1 convs [C, C, 1, 1]"""
    w = state.get("down_blocks.0.attentions.0.proj_in.weight") if state is not None else None
    return w is not None and w.dim() == 4


def sd_vae_cfg(image_hw=512):
    return dict(in_channels=3, latent_channels=4, block_out=(128, 256, 512, 512), layers_per_block=2, groups=32, image_hw=image_hw)


def _unet_struct(cfg):
    u = UNetCfg()
    u.in_ch, u.out_ch, u.n_levels = cfg["in_channels"], cfg["out_channels"], len(cfg["block_out"])
    for i, v in enumerate(cfg["block_out"]):
        u.block_out[i] = v
    for i, v in enumerate(cfg["heads"]):
        u.heads[i] = v
    u.layers_per_block, u.cross_dim, u.ctx_len, u.groups = cfg["layers_per_block"], cfg["cross_dim"], cfg["ctx_len"], cfg["groups"]
    u.latent_hw, u.batch = cfg["latent_hw"], 2
    u.proj_conv = 1 if cfg.get("proj_conv", False) else 0
    return u


def _vae_struct(cfg):
    v = VaeCfg()
    v.in_ch, v.latent_ch, v.n_levels = cfg["in_channels"], cfg["latent_channels"], len(cfg["block_out"])
    for i, c in enumerate(cfg["block_out"]):
        v.block_out[i] = c
    v.layers_per_block, v.groups, v.image_hw = cfg["layers_per_block"], cfg["groups"], cfg["image_hw"]
    v.decoder = 1 if cfg.get("decoder", True) else 0
    return v


def alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    """DDIMScheduler with SD's scheduler_config.json (scaled_linear), as used at nerf/sd.py:55,62."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class SDEngine(L.Engine):
    """The SD engine (mi3d_sd_create): U-Net and VAE launch lists planned in one workspace."""

    def __init__(self, unet_cfg, vae_cfg, device, graph_replay=True):
        self.u = _unet_struct(unet_cfg) if unet_cfg else None
        self.v = _vae_struct(vae_cfg) if vae_cfg else None
        # graph_replay=False keeps plain launches on the caller's stream (used by the parity tests as the A/B arm)
        super().__init__("sd", (C.byref(self.u) if self.u else None, C.byref(self.v) if self.v else None), device, graph_replay,
                         f"SD configuration unet={unet_cfg} vae={vae_cfg}")

    def partner(self, name, tensors):
        """the GEGLU proj weight is written together with its bias"""
        if not name.endswith("ff.net.0.proj.weight"):
            return None
        return tensors[name[:-len("weight")] + "bias"]


def _default_init(name, shape, gen):
    """PyTorch default initialisers keyed by the diffusers parameter name."""
    if name.endswith(".weight") and len(shape) == 1:          # norms
        return torch.ones(shape)
    if name.endswith(".bias") and ("norm" in name.split(".")[-2] or name.split(".")[-2] in ("conv_norm_out", "group_norm")):
        return torch.zeros(shape)
    if name.endswith(".weight"):
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        bound = 1.0 / math.sqrt(fan_in)
        return (torch.rand(shape, generator=gen) * 2 - 1) * bound
    return (torch.rand(shape, generator=gen) * 2 - 1) * 0.02   # biases


class _EncodeImgs(torch.autograd.Function):
    """latents = vae.encode(2*interp(pred_rgb)-1).latent_dist.sample() * 0.18215 with the posterior noise injected."""

    @staticmethod
    def forward(ctx, pred_rgb, eps, engine):
        pred_rgb = L.f32c(pred_rgb)
        L.require_cuda(pred_rgb, eps)
        B, Cc, H, W = pred_rgb.shape
        if B != 1 or Cc != 3:
            raise L.Mi3dError("encode_imgs expects pred_rgb [1,3,H,W]")
        hw = engine.v.image_hw // 8
        latents = torch.empty(1, 4, hw, hw, dtype=torch.float32, device=pred_rgb.device)
        with engine.on_stream():
            L.check(L.lib().mi3d_sd_encode(engine.h, L.ptr(pred_rgb), C.c_int(H), C.c_int(W), L.ptr(eps), L.ptr(latents), L.stream()), "sd_encode")
        ctx.engine, ctx.hw_in = engine, (H, W)
        ctx.save_for_backward(eps)
        return latents

    @staticmethod
    def backward(ctx, g):
        (eps,) = ctx.saved_tensors
        H, W = ctx.hw_in
        g = L.f32c(g)
        grad = torch.empty(1, 3, H, W, dtype=torch.float32, device=g.device)
        with ctx.engine.on_stream():
            L.check(L.lib().mi3d_sd_encode_backward(ctx.engine.h, L.ptr(g), L.ptr(eps), C.c_int(H), C.c_int(W), L.ptr(grad), L.stream()),
                    "sd_encode_backward")
        return grad, None, None


class StableDiffusion(nn.Module):
    def __init__(self, device, sd_version='2.0', hf_key=None, step_range=[0.2, 0.6], unet_cfg=None, vae_cfg=None, seed=0,
                 unet_state=None, vae_state=None, graph_replay=True, defer_backward=False, tokenizer=None):
        super().__init__()
        # tokenizer: a callable with CLIPTokenizer.__call__'s contract (e.g. CLIPTokenizer.from_pretrained(model_key, subfolder="tokenizer")),
        # used by get_text_embeds for prompts given as strings.  The text encoder itself is created when its weights are loaded.
        self.tokenizer = tokenizer
        self.text_encoder = None
        self.graph_replay = graph_replay
        # defer_backward (additive option, default off = the reference's behaviour): train_step does not call latents.backward
        # itself (nerf/sd.py:171) but returns the surrogate loss  sum(stopgrad(dL/d pred_rgb) * pred_rgb), whose gradient w.r.t.
        # pred_rgb IS the SDS gradient.  The Trainer adds it to its regularisers and its single loss.backward() (nerf/utils.py:983)
        # then walks the render graph ONCE instead of twice (the reference back-propagates through the retained render graph a
        # second time).  Parameter gradients are identical (linearity); only the returned loss value differs (0 in the reference).
        self.defer_backward = bool(defer_backward)
        self.device = torch.device(device)
        self.sd_version = sd_version
        # nerf/sd.py:29-37: '2.1' / '2.0' select stable-diffusion-2-1-base / 2-base, '1.5' stable-diffusion-v1-5, hf_key any other
        # checkpoint (BASELINE config 4 names SD-2.1-768).  All SD-2.x U-Nets share ONE topology (block_out 320/640/1280/1280, head_dim
        # 64, cross dim 1024, linear projections) and all SD-1.x U-Nets another (the same channels, 8 heads of 40 / 80 / 160, cross dim
        # 768, 1x1-conv projections); nerf/sd.py:124 always feeds 512x512 -> 64x64 latents, so each family runs on one engine plan.  An
        # hf_key checkpoint is SD-1.x when its unet_state has conv projections.  The 768 checkpoint's v-prediction output is consumed
        # as if it were epsilon, exactly like the reference does (it never reads prediction_type, nerf/sd.py:146-151).  SD-1.x needs its
        # checkpoint: the seeded stand-in exists for SD-2.0 only (the benchmark's synthetic workload), so a missing SD-1.5 unet_state
        # is an error rather than silently random weights.
        sd1 = unet_cfg is None and (sd_version == '1.5' or is_sd1_unet_state(unet_state))
        if sd1 and unet_state is None:
            raise ValueError('Stable-diffusion 1.5 needs its checkpoint: pass the U-Net / VAE state dicts (unet_state=, vae_state=: '
                             'diffusers UNet2DConditionModel / AutoencoderKL state_dict()s); there is no synthetic SD-1.5')
        if sd_version not in ('1.5', '2.0', '2.1') and hf_key is None and unet_cfg is None:
            raise ValueError(f'Stable-diffusion version {sd_version} not built (1.5 / 2.0 / 2.1 / hf_key of an SD-1.x or SD-2.x checkpoint; reference default 2.0, nerf/sd.py:33-34)')
        self.hf_key = hf_key
        self.unet_cfg = unet_cfg or (sd15_unet_cfg() if sd1 else sd20_unet_cfg())
        self.vae_cfg = vae_cfg or sd_vae_cfg()
        self.engine = SDEngine(self.unet_cfg, self.vae_cfg, self.device, graph_replay=graph_replay)
        gen = torch.Generator().manual_seed(seed)
        # parameter containers with diffusers names: unet.<name>, vae.<name>
        self.unet = nn.ParameterDict()
        self.vae = nn.ParameterDict()
        tensors = {}
        for name, shape in zip(self.engine.names, self.engine.shapes):
            if "#" in name:
                continue
            is_vae = name.split(".")[0] in ("encoder", "quant_conv", "decoder", "post_quant_conv")
            src = (vae_state if is_vae else unet_state)
            # tensors absent from a given state (e.g. an encoder-only VAE state) keep the seeded default initialisation
            t = src[name].detach().float() if (src is not None and name in src) else _default_init(name, shape, gen)
            p = nn.Parameter(t.to(self.device).contiguous(), requires_grad=False)
            (self.vae if is_vae else self.unet)[name.replace(".", "/")] = p
            tensors[name] = p.data
        self.engine.load(tensors)
        self.num_train_timesteps = 1000
        self.min_step = int(self.num_train_timesteps * float(step_range[0]))
        self.max_step = int(self.num_train_timesteps * float(step_range[1]))
        self.alphas = alphas_cumprod().to(self.device)
        self._t = torch.zeros(1, dtype=torch.long, device=self.device)

    def load_diffusers_state_dict(self, unet_state=None, vae_state=None, text_encoder_state=None):
        """copy tensors named like diffusers' UNet2DConditionModel / AutoencoderKL state_dict()s and push them to the engine;
        text_encoder_state (transformers' CLIPTextModel.state_dict()) goes into the SD text encoder, created on first use (quick-GELU
        when the U-Net is SD-1.x, exact GELU for SD-2.x)."""
        if text_encoder_state is not None:
            if self.text_encoder is None:
                act = "quick_gelu" if self.unet_cfg.get("proj_conv", False) else "gelu"
                self.text_encoder = TextEncoder(self.device, cfg=cfg_from_state_dict(text_encoder_state, hidden_act=act),
                                                state_dict=text_encoder_state, graph_replay=self.graph_replay)
            else:
                self.text_encoder.load_state_dict(text_encoder_state)
            if unet_state is None and vae_state is None:
                return
        with torch.no_grad():
            for store, sd in ((self.unet, unet_state), (self.vae, vae_state)):
                if sd is None:
                    continue
                for k, p in store.items():
                    p.copy_(sd[k.replace("/", ".")].to(p.device, torch.float32))
        self.reload()

    def reload(self):
        """push the current parameter values into the engine again (after load_state_dict)."""
        tensors = {k.replace("/", "."): v.data for k, v in list(self.unet.items()) + list(self.vae.items())}
        self.engine.load(tensors)

    def get_text_embeds(self, prompt, negative_prompt):
        """nerf/sd.py:68-85: [uncond, cond] text embeddings [2,77,D].  prompt / negative_prompt: a string, a list of one string, or
        int64 token ids [1,77] / [77].  With text-encoder weights loaded both run through the SD text encoder in one batch of 2;
        strings need the tokenizer (the prompt is truncated to 77 tokens, the negative prompt is not, as in the reference).
        Without them a deterministic stand-in keyed by the prompt strings keeps the call surface."""
        if self.text_encoder is None:
            D = self.unet_cfg["cross_dim"]
            out = []
            for s in (negative_prompt, prompt):
                s = s[0] if isinstance(s, (list, tuple)) else s
                # stable digest (python's hash() is salted per process: every rank would get different text conditioning)
                g = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(("mi3d:" + s).encode()).digest()[:4], "little"))
                out.append(torch.randn(1, 77, D, generator=g))
            return torch.cat(out).to(self.device)
        ids = torch.cat([self._token_ids(negative_prompt, truncation=False), self._token_ids(prompt, truncation=True)])
        with torch.no_grad():
            return self.text_encoder(ids)[0]

    def _token_ids(self, text, truncation):
        T = self.text_encoder.cfg["context_len"]
        if torch.is_tensor(text):
            ids = text
        else:
            if self.tokenizer is None:
                raise L.Mi3dError("get_text_embeds got a string but StableDiffusion has no tokenizer: pass tokenizer=CLIPTokenizer.from_pretrained("
                                  "model_key, subfolder='tokenizer') to the constructor, or pass int64 token ids [1,77]")
            kw = dict(padding="max_length", max_length=T, return_tensors="pt")
            if truncation:
                kw["truncation"] = True
            tok = self.tokenizer(text if isinstance(text, (list, tuple)) else [text], **kw)
            ids = tok.input_ids if hasattr(tok, "input_ids") else tok["input_ids"]
            ids = torch.as_tensor(ids)
        if ids.dtype != torch.long or ids.shape[-1] != T or ids.dim() not in (1, 2) or (ids.dim() == 2 and ids.shape[0] != 1):
            raise L.Mi3dError(f"text embeddings take one prompt's int64 token ids [1,{T}] or [{T}]; got {ids.dtype} {tuple(ids.shape)}")
        return ids.reshape(1, T).to(self.device)

    def encode_imgs(self, imgs, eps=None):
        """nerf/sd.py:212-220 (the 512x512 interpolation of :124 is folded in: pass the render-resolution image)."""
        hw = self.vae_cfg["image_hw"] // 8
        if eps is None:
            eps = torch.randn(1, 4, hw, hw, device=self.device)
        return _EncodeImgs.apply(imgs, L.f32c(eps), self.engine)

    def decode_latents(self, latents):
        """nerf/sd.py:201-210: (vae.decode(latents / 0.18215).sample / 2 + 0.5).clamp(0, 1) -> [1,3,S,S]; no gradient, like the reference"""
        latents = L.f32c(latents.detach())
        S = self.vae_cfg["image_hw"]
        imgs = torch.empty(1, 3, S, S, dtype=torch.float32, device=latents.device)
        with self.engine.on_stream():
            L.check(L.lib().mi3d_sd_decode(self.engine.h, L.ptr(latents), L.ptr(imgs), L.stream()), "sd_decode")
        return imgs

    def ddim_prev_sample(self, noise_pred, latents_noisy, t_dev):
        """scheduler.set_timesteps(1000); scheduler.step(noise_pred, t, latents_noisy)['prev_sample'] (nerf/sd.py:154-155)"""
        noise_pred, latents_noisy = L.f32c(noise_pred), L.f32c(latents_noisy)
        out = torch.empty_like(latents_noisy)
        L.check(L.lib().mi3d_sd_ddim_step(L.ptr(noise_pred), L.ptr(latents_noisy), L.ptr(t_dev), L.ptr(self.alphas), L.ptr(out),
                                          C.c_int(out.numel()), L.stream()), "sd_ddim_step")
        return out

    @staticmethod
    def img_clip_loss(clip_model, rgb1, rgb2, aug=None):
        """nerf/sd.py:97-104 on a caller-provided CLIP model (openai `clip` is outside the hot path and not shipped here)"""
        aug = aug or (lambda x: x)
        z1, z2 = clip_model.encode_image(aug(rgb1)), clip_model.encode_image(aug(rgb2))
        z1, z2 = z1 / z1.norm(dim=-1, keepdim=True), z2 / z2.norm(dim=-1, keepdim=True)
        return -(z1 * z2).sum(-1).mean()

    @staticmethod
    def img_text_clip_loss(clip_model, rgb, text_tokens, aug=None):
        """nerf/sd.py:106-114; `text_tokens` = clip.tokenize(prompt) done by the caller (the tokenizer belongs to the clip package)"""
        aug = aug or (lambda x: x)
        z1 = clip_model.encode_image(aug(rgb))
        z1 = z1 / z1.norm(dim=-1, keepdim=True)
        zt = clip_model.encode_text(text_tokens)
        zt = zt / zt.norm(dim=-1, keepdim=True)
        return -(z1 * zt).sum(-1).mean()

    def _denoise_branch(self, noise_pred, latents_noisy, ref_rgb, ref_text, clip_model):
        """nerf/sd.py:153-159: one DDIM step, decode, CLIP losses.  Nothing here carries a gradient to the NeRF (imgs comes out of
        no_grad code in the reference too); without a clip_model the images are still produced (Trainer dumps them, utils.py:569)."""
        de_latents = self.ddim_prev_sample(noise_pred, latents_noisy, self._t)
        imgs = self.decode_latents(de_latents)
        loss = 0
        if isinstance(clip_model, CLIP):
            img_loss, text_loss = clip_model.losses(imgs, ref_rgb, ref_text)
            loss = 10 * img_loss + 10 * text_loss
        elif clip_model is not None:
            aug = getattr(self, "aug", None)
            loss = 10 * self.img_clip_loss(clip_model, imgs, ref_rgb, aug) + 10 * self.img_text_clip_loss(clip_model, imgs, ref_text, aug)
        return loss, imgs

    def unet_sds(self, latents, noise, t, text_embeddings, guidance_scale):
        """add_noise -> U-Net -> CFG -> SDS gradient (nerf/sd.py:138-170). t: device int64 [1]. Returns (noise_pred, grad)."""
        latents, noise, text_embeddings = L.f32c(latents.detach()), L.f32c(noise), L.f32c(text_embeddings)
        noise_pred = torch.empty_like(latents)
        grad = torch.empty_like(latents)
        with self.engine.on_stream():
            L.check(L.lib().mi3d_sd_unet_sds(self.engine.h, L.ptr(latents), L.ptr(noise), L.ptr(t), L.ptr(self.alphas), L.ptr(text_embeddings),
                                             C.c_float(float(guidance_scale)), L.ptr(noise_pred), L.ptr(grad), L.stream()), "sd_unet_sds")
        return noise_pred, grad

    def train_step(self, text_embeddings, pred_rgb, ref_rgb=None, noise=None, islarge=False, ref_text=None, clip_model=None,
                   guidance_scale=10, t=None, eps_posterior=None):
        """nerf/sd.py:117-174.  `noise` is accepted and ignored like the reference (:140) unless `t` is also injected
        (additive test hook: t, eps_posterior, noise make the step deterministic)."""
        loss, imgs = 0, None
        if t is None:
            t_host = int(torch.randint(self.min_step, self.max_step + 1, [1]).item())     # CPU generator: no device sync
            noise = None
        else:
            t_host = int(t)
        self._t.fill_(t_host)
        if self.defer_backward and not (not islarge and (t_host / self.num_train_timesteps) <= 0.4):
            with torch.no_grad():
                hw = self.vae_cfg["image_hw"] // 8
                eps = L.f32c(eps_posterior) if eps_posterior is not None else torch.randn(1, 4, hw, hw, device=self.device)
                rgb = L.f32c(pred_rgb.detach())
                H, W = rgb.shape[-2:]
                latents = torch.empty(1, 4, hw, hw, dtype=torch.float32, device=rgb.device)
                grad_rgb = torch.empty_like(rgb)
                if noise is None:
                    noise = torch.randn_like(latents)
                with self.engine.on_stream():
                    L.check(L.lib().mi3d_sd_encode(self.engine.h, L.ptr(rgb), C.c_int(H), C.c_int(W), L.ptr(eps), L.ptr(latents), L.stream()), "sd_encode")
                noise_pred, grad = self.unet_sds(latents, noise, self._t, text_embeddings, guidance_scale)
                with self.engine.on_stream():
                    L.check(L.lib().mi3d_sd_encode_backward(self.engine.h, L.ptr(grad), L.ptr(eps), C.c_int(H), C.c_int(W), L.ptr(grad_rgb), L.stream()),
                            "sd_encode_backward")
            self.last = dict(latents=latents, noise_pred=noise_pred, grad=grad, t=t_host)
            return (grad_rgb * pred_rgb).sum(), None
        latents = self.encode_imgs(pred_rgb, eps_posterior)
        if noise is None:
            noise = torch.randn_like(latents)
        with torch.no_grad():
            noise_pred, grad = self.unet_sds(latents, noise, self._t, text_embeddings, guidance_scale)
            if not islarge and (t_host / self.num_train_timesteps) <= 0.4:
                # the "denoise" side branch (nerf/sd.py:153-159): no SDS backward on this step, exactly like the reference
                a = self.alphas[t_host]
                latents_noisy = a.sqrt() * latents.detach() + (1 - a).sqrt() * noise            # scheduler.add_noise (nerf/sd.py:141)
                if not self.vae_cfg.get("decoder", True):
                    return 0, None
                return self._denoise_branch(noise_pred, latents_noisy, ref_rgb, ref_text, clip_model)
        latents.backward(gradient=grad, retain_graph=True)
        self.last = dict(latents=latents.detach(), noise_pred=noise_pred, grad=grad, t=t_host)
        return loss, imgs
