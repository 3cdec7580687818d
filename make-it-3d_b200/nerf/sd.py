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
`produce_latents` / `prompt_to_img` (nerf/sd.py:176-238) sample with DDIM (eta 0) and classifier-free guidance on the device
(`mi3d_sd_sample`); `from_pretrained(local_dir, device)` loads a local diffusers directory; `python -m mi3d_b200.nerf.sd PROMPT --ckpt DIR`
is the reference's demo.
Batches of G views (2 <= G <= 8; the coarse stage's several views per iteration): `encode_imgs`, `unet_sds` and `train_step` take
pred_rgb / latents [G,...] and run on a second engine planned for G views (U-Net batch 2G, VAE encoder batch G) on first use; its
weights are the same parameter tensors.  ONE such engine is kept (33.5 GiB at G = 8, full size): a batch of another size replaces it.  The G views share one timestep; each takes the SDS or the denoise branch on its own.
"""
import ctypes as C
import hashlib
import json
import math
import os

import numpy as np
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
                ("groups", C.c_int), ("image_hw", C.c_int), ("decoder", C.c_int), ("batch", C.c_int)]


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


def _unet_struct(cfg, views=1):
    u = UNetCfg()
    u.in_ch, u.out_ch, u.n_levels = cfg["in_channels"], cfg["out_channels"], len(cfg["block_out"])
    for i, v in enumerate(cfg["block_out"]):
        u.block_out[i] = v
    for i, v in enumerate(cfg["heads"]):
        u.heads[i] = v
    u.layers_per_block, u.cross_dim, u.ctx_len, u.groups = cfg["layers_per_block"], cfg["cross_dim"], cfg["ctx_len"], cfg["groups"]
    u.latent_hw, u.batch = cfg["latent_hw"], 2 * views
    u.proj_conv = 1 if cfg.get("proj_conv", False) else 0
    return u


def _vae_struct(cfg, views=1):
    v = VaeCfg()
    v.in_ch, v.latent_ch, v.n_levels = cfg["in_channels"], cfg["latent_channels"], len(cfg["block_out"])
    for i, c in enumerate(cfg["block_out"]):
        v.block_out[i] = c
    v.layers_per_block, v.groups, v.image_hw = cfg["layers_per_block"], cfg["groups"], cfg["image_hw"]
    v.decoder = 1 if cfg.get("decoder", True) else 0
    v.batch = views
    return v


def alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    """DDIMScheduler with SD's scheduler_config.json (scaled_linear), as used at nerf/sd.py:55,62."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


# ---------------------------------------------------------------------------------------------------------------------------------
# DDIM sampling schedule (produce_latents, nerf/sd.py:176-199) and diffusers checkpoint configs
# ---------------------------------------------------------------------------------------------------------------------------------
NUM_TRAIN_TIMESTEPS = 1000
# SD's scheduler defaults (scheduler_config.json of every SD-1.x / SD-2.x checkpoint but SD-2.1-768's prediction_type)
SD_SCHEDULER = dict(steps_offset=1, set_alpha_to_one=False, prediction_type="epsilon", timestep_spacing="leading")
PREDICTION_TYPES = {"epsilon": 0, "v_prediction": 1}


class SDSchedule(C.Structure):
    """mi3d_sd_schedule: one DDIM step of mi3d_sd_sample"""
    _fields_ = [("t", C.c_longlong), ("alpha_t", C.c_float), ("alpha_prev", C.c_float)]


def ddim_timesteps(n, spacing="leading", steps_offset=1, T=NUM_TRAIN_TIMESTEPS):
    """DDIMScheduler.set_timesteps(n).timesteps (int64, descending) for timestep_spacing 'leading' / 'trailing' / 'linspace'"""
    if not isinstance(n, int) or not 1 <= n <= T:
        raise L.Mi3dError(f"num_inference_steps must be an integer in 1..{T}; got {n!r}")
    if spacing == "leading":
        ts = (np.arange(0, n) * (T // n)).round()[::-1].astype(np.int64) + int(steps_offset)
    elif spacing == "trailing":
        ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
    elif spacing == "linspace":
        ts = np.linspace(0, T - 1, n).round()[::-1].astype(np.int64)
    else:
        raise L.Mi3dError(f"timestep_spacing must be 'leading', 'trailing' or 'linspace'; got {spacing!r}")
    if ts.min() < 0 or ts.max() >= T:
        raise L.Mi3dError(f"{n} steps with {spacing!r} spacing and steps_offset {steps_offset} give timesteps outside 0..{T - 1}")
    return np.ascontiguousarray(ts)


def ddim_schedule(n, spacing="leading", steps_offset=1, set_alpha_to_one=False, alphas=None, T=NUM_TRAIN_TIMESTEPS):
    """the mi3d_sd_schedule table (a numpy record array): t_i, alphas_cumprod[t_i] and alpha_prev_i = alphas_cumprod[t_i - T // n], or
    final_alpha_cumprod (1 with set_alpha_to_one, else alphas_cumprod[0]) when t_i - T // n < 0"""
    a = (alphas_cumprod(T) if alphas is None else alphas).detach().cpu().float().numpy()
    ts = ddim_timesteps(n, spacing, steps_offset, T)
    prev = ts - T // n
    final = np.float32(1.0) if set_alpha_to_one else a[0]
    tab = np.zeros(n, dtype=np.dtype([("t", "<i8"), ("alpha_t", "<f4"), ("alpha_prev", "<f4")]))
    tab["t"], tab["alpha_t"] = ts, a[ts]
    tab["alpha_prev"] = np.where(prev >= 0, a[np.maximum(prev, 0)], final)
    assert tab.dtype.itemsize == C.sizeof(SDSchedule)
    return tab


def _heads(cfg, n_levels):
    h = cfg["attention_head_dim"]           # diffusers' name; SD's configs store the head COUNT in it
    h = [h] * n_levels if isinstance(h, int) else list(h)
    if len(h) != n_levels:
        raise L.Mi3dError(f"attention_head_dim {cfg['attention_head_dim']} does not match {n_levels} levels")
    return tuple(int(x) for x in h)


def unet_cfg_from_config(cfg):
    """diffusers' unet/config.json -> the engine's U-Net configuration (sd20_unet_cfg / sd15_unet_cfg form)"""
    if cfg.get("in_channels", 4) != 4 or cfg.get("out_channels", 4) != 4:
        raise L.Mi3dError(f"only 4-channel latent U-Nets are supported; got in_channels={cfg.get('in_channels')} (inpainting and "
                          f"depth-conditioned checkpoints take more) out_channels={cfg.get('out_channels')}")
    bo = tuple(int(x) for x in cfg["block_out_channels"])
    if not 1 <= len(bo) <= 4 or not isinstance(cfg.get("cross_attention_dim"), int):
        raise L.Mi3dError(f"unsupported U-Net topology: block_out_channels {bo}, cross_attention_dim {cfg.get('cross_attention_dim')}")
    out = dict(in_channels=4, out_channels=4, block_out=bo, layers_per_block=int(cfg["layers_per_block"]), heads=_heads(cfg, len(bo)),
               cross_dim=int(cfg["cross_attention_dim"]), groups=int(cfg.get("norm_num_groups", 32)), ctx_len=77,
               latent_hw=int(cfg["sample_size"]))
    if not cfg.get("use_linear_projection", False):
        out["proj_conv"] = True                  # SD-1.x: 1x1-conv proj_in / proj_out
    return out


def vae_cfg_from_config(cfg):
    """diffusers' vae/config.json -> the engine's VAE configuration (sd_vae_cfg form)"""
    if float(cfg.get("scaling_factor", 0.18215)) != 0.18215:
        raise L.Mi3dError(f"the VAE's scaling_factor is {cfg['scaling_factor']}; nerf/sd.py scales latents by 0.18215")
    if cfg.get("in_channels", 3) != 3 or cfg.get("latent_channels", 4) != 4:
        raise L.Mi3dError("only 3-channel images and 4-channel latents are supported")
    return dict(in_channels=3, latent_channels=4, block_out=tuple(int(x) for x in cfg["block_out_channels"]),
                layers_per_block=int(cfg["layers_per_block"]), groups=int(cfg.get("norm_num_groups", 32)), image_hw=int(cfg["sample_size"]))


def scheduler_from_config(cfg):
    """scheduler/scheduler_config.json -> the DDIM settings the sampler reads (DDIMScheduler's defaults for absent keys).  The betas
    must be SD's scaled_linear 0.00085 / 0.012 over 1000 steps: the SDS path's `alphas` are built from them."""
    betas = (cfg.get("beta_schedule", "linear"), float(cfg.get("beta_start", 0.0001)), float(cfg.get("beta_end", 0.02)),
             int(cfg.get("num_train_timesteps", 1000)))
    if betas != ("scaled_linear", 0.00085, 0.012, 1000) or cfg.get("trained_betas") is not None or cfg.get("rescale_betas_zero_snr", False):
        raise L.Mi3dError(f"unsupported beta schedule {betas} (trained_betas={cfg.get('trained_betas')}, rescale_betas_zero_snr="
                          f"{cfg.get('rescale_betas_zero_snr', False)}): SD's is scaled_linear 0.00085 / 0.012 over 1000 steps")
    if cfg.get("clip_sample", True) or cfg.get("thresholding", False):
        raise L.Mi3dError("clip_sample / thresholding are not supported (SD's scheduler configs turn both off)")
    out = dict(steps_offset=int(cfg.get("steps_offset", 0)), set_alpha_to_one=bool(cfg.get("set_alpha_to_one", True)),
               prediction_type=cfg.get("prediction_type", "epsilon"), timestep_spacing=cfg.get("timestep_spacing", "leading"))
    if out["prediction_type"] not in PREDICTION_TYPES:
        raise L.Mi3dError(f"prediction_type must be one of {sorted(PREDICTION_TYPES)}; got {out['prediction_type']!r}")
    ddim_timesteps(1, out["timestep_spacing"], out["steps_offset"])
    return out


_ST_DTYPES = {"F32": torch.float32, "F16": torch.float16, "BF16": torch.bfloat16, "F64": torch.float64, "I64": torch.int64,
              "I32": torch.int32}


def read_safetensors(path):
    """name -> CPU tensor from a .safetensors file (an 8-byte little-endian header size, a JSON header, then the raw tensors)"""
    out = {}
    with open(path, "rb") as f:
        n = int.from_bytes(f.read(8), "little")
        header = json.loads(f.read(n))
        for name, meta in header.items():
            if name == "__metadata__":
                continue
            if meta["dtype"] not in _ST_DTYPES:
                raise L.Mi3dError(f"{path}: tensor {name} has unsupported dtype {meta['dtype']}")
            b, e = meta["data_offsets"]
            buf = bytearray(e - b)                  # each tensor is read straight into its own buffer: one host copy of the file
            f.seek(8 + n + b)
            if f.readinto(buf) != e - b:
                raise L.Mi3dError(f"{path}: tensor {name} runs past the end of the file")
            t = torch.frombuffer(buf, dtype=_ST_DTYPES[meta["dtype"]]) if e > b else torch.empty(0, dtype=_ST_DTYPES[meta["dtype"]])
            out[name] = t.reshape(meta["shape"])
    return out


def _read_weights(folder, stem):
    """<folder>/<stem>.safetensors, else <stem>.fp16.safetensors; .bin-only folders are refused (pickle files are not read)"""
    for name in (stem + ".safetensors", stem + ".fp16.safetensors"):
        p = os.path.join(folder, name)
        if os.path.exists(p):
            return read_safetensors(p)
    raise L.Mi3dError(f"no {stem}[.fp16].safetensors in {folder} (.bin checkpoints are not supported)")


def _read_json(path):
    if not os.path.exists(path):
        raise L.Mi3dError(f"{path} is missing: from_pretrained needs a local diffusers directory")
    with open(path) as f:
        return json.load(f)


class SDEngine(L.Engine):
    """The SD engine (mi3d_sd_create): U-Net and VAE launch lists planned in one workspace, for `views` views per SDS step (U-Net
    batch 2 * views, VAE encoder batch views)."""

    def __init__(self, unet_cfg, vae_cfg, device, graph_replay=True, views=1):
        self.views = views
        self.u = _unet_struct(unet_cfg, views) if unet_cfg else None
        self.v = _vae_struct(vae_cfg, views) if vae_cfg else None
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
        if B != engine.views or Cc != 3:
            raise L.Mi3dError(f"encode_imgs expects pred_rgb [{engine.views},3,H,W]")
        hw = engine.v.image_hw // 8
        latents = torch.empty(B, 4, hw, hw, dtype=torch.float32, device=pred_rgb.device)
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
        grad = torch.empty(g.shape[0], 3, H, W, dtype=torch.float32, device=g.device)
        with ctx.engine.on_stream():
            L.check(L.lib().mi3d_sd_encode_backward(ctx.engine.h, L.ptr(g), L.ptr(eps), C.c_int(H), C.c_int(W), L.ptr(grad), L.stream()),
                    "sd_encode_backward")
        return grad, None, None


class StableDiffusion(nn.Module):
    def __init__(self, device, sd_version='2.0', hf_key=None, step_range=[0.2, 0.6], unet_cfg=None, vae_cfg=None, seed=0,
                 unet_state=None, vae_state=None, graph_replay=True, defer_backward=False, tokenizer=None, strict=False):
        super().__init__()
        # strict: every registry tensor must come from unet_state / vae_state and no other key is accepted (from_pretrained); by
        # default absent tensors keep the seeded initialisation.  A tensor whose shape differs from the registry's is always refused.
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
            if src is not None and name in src and tuple(src[name].shape) != tuple(shape):
                raise L.Mi3dError(f"{name}: shape {tuple(src[name].shape)} in the state dict, the engine's configuration has {tuple(shape)}")
            if strict and (src is None or name not in src):
                raise L.Mi3dError(f"{name} is missing from the {'VAE' if is_vae else 'U-Net'} state dict")
            t = src[name].detach().float() if (src is not None and name in src) else _default_init(name, shape, gen)
            p = nn.Parameter(t.to(self.device).contiguous(), requires_grad=False)
            (self.vae if is_vae else self.unet)[name.replace(".", "/")] = p
            tensors[name] = p.data
        if strict:
            unexpected = sorted(set(unet_state or {}).union(vae_state or {}) - set(tensors))
            if unexpected:
                raise L.Mi3dError(f"{len(unexpected)} tensors of the state dicts have no place in the engine's configuration, e.g. {unexpected[:4]}")
        self.engine.load(tensors)
        self.num_train_timesteps = 1000
        self.min_step = int(self.num_train_timesteps * float(step_range[0]))
        self.max_step = int(self.num_train_timesteps * float(step_range[1]))
        self.alphas = alphas_cumprod().to(self.device)
        self._t = torch.zeros(1, dtype=torch.long, device=self.device)
        # the sampler's DDIM settings (scheduler_config.json; from_pretrained reads them).  train_step never reads them: like the
        # reference it consumes a v-prediction U-Net's output as epsilon.
        for k, v in SD_SCHEDULER.items():
            setattr(self, k, v)
        self._schedules = {}          # (n, scheduler settings) -> device mi3d_sd_schedule table
        self._size_engines = {}       # image size -> SDEngine planned on first use by produce_latents / decode_latents
        self._view_engine = None      # the one SDEngine for G > 1 views per SDS step, planned on first use (views_engine)

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
        tensors = self._tensors()
        for eng in [self.engine] + list(self._size_engines.values()) + ([self._view_engine] if self._view_engine else []):
            eng.load(tensors)

    def _tensors(self):
        return {k.replace("/", "."): v.data for k, v in list(self.unet.items()) + list(self.vae.items())}

    def _engine_for(self, size, part):
        """the engine whose `part` ("unet" or "vae") is planned for size x size images: the constructor's at its own size, else one
        planned on first use per size and loaded from the same parameter tensors"""
        if (self.unet_cfg["latent_hw"] * 8 if part == "unet" else self.vae_cfg["image_hw"]) == size:
            return self.engine
        eng = self._size_engines.get(size)
        if eng is None:
            try:
                eng = SDEngine(dict(self.unet_cfg, latent_hw=size // 8), dict(self.vae_cfg, image_hw=size), self.device, graph_replay=self.graph_replay)
            except L.Mi3dError as e:
                raise L.Mi3dError(f"no SD engine plan for {size}x{size} images") from e
            eng.load(self._tensors())
            self._size_engines[size] = eng
        return eng

    def views_engine(self, G):
        """the engine of G-view SDS steps: the constructor's for G = 1, else the one multi-view engine (U-Net batch 2G, VAE encoder batch
        G, no decoder: denoise-branch views decode one at a time on the constructor's engine), loaded from the same tensors.  Only one is
        kept, so memory stays bounded by the largest batch in use: asking for another G frees the current one (an autograd node that still
        holds it keeps it until its backward ran) and plans the new one.  Callers that mix batch sizes should run the odd ones view by
        view instead (CoarseStep.step_views does)."""
        if G == 1:
            return self.engine
        if not 1 <= G <= L.MAX_VIEWS:
            raise L.Mi3dError(f"a batched SDS step takes 1..{L.MAX_VIEWS} views; got {G}")
        if self._view_engine is None or self._view_engine.views != G:
            self._view_engine = None                      # released before the new workspace is allocated
            eng = SDEngine(self.unet_cfg, dict(self.vae_cfg, decoder=False), self.device, graph_replay=self.graph_replay, views=G)
            eng.load(self._tensors())
            self._view_engine = eng
        return self._view_engine

    def _schedule(self, n):
        key = (n, self.timestep_spacing, self.steps_offset, self.set_alpha_to_one)
        tab = self._schedules.get(key)
        if tab is None:
            rec = ddim_schedule(n, self.timestep_spacing, self.steps_offset, self.set_alpha_to_one)
            tab = torch.from_numpy(rec.view(np.uint8).copy()).to(self.device)
            self._schedules[key] = tab
        return tab

    def produce_latents(self, text_embeddings, height=512, width=512, num_inference_steps=50, guidance_scale=7.5, latents=None):
        """nerf/sd.py:176-199: DDIM (eta 0) with classifier-free guidance from x_T to x_0, on the device (mi3d_sd_sample).
        text_embeddings [2B,77,D] laid out [uncond x B, cond x B]; latents (x_T) [B,4,H/8,W/8], drawn with torch.randn when None
        (DDIM's init_noise_sigma is 1).  The B samples run in turn: each is independent in the reference's batch too.  Square sizes
        only, H a multiple of 64.  Returns fp32 [B,4,H/8,W/8]."""
        if height != width or height <= 0 or height % 64:
            raise L.Mi3dError(f"produce_latents takes square sizes with H a multiple of 64; got {height}x{width}")
        D, hw = self.unet_cfg["cross_dim"], height // 8
        te = text_embeddings
        if not torch.is_tensor(te) or te.dim() != 3 or te.shape[0] == 0 or te.shape[0] % 2 or tuple(te.shape[1:]) != (77, D):
            raise L.Mi3dError(f"text_embeddings must be [2B,77,{D}] ([uncond x B, cond x B]); got {tuple(getattr(te, 'shape', ()))}")
        B = te.shape[0] // 2
        if latents is None:
            latents = torch.randn((B, 4, hw, hw), device=self.device)
        elif tuple(latents.shape) != (B, 4, hw, hw):
            raise L.Mi3dError(f"latents must be [{B},4,{hw},{hw}] for {B} prompt(s) at {height}x{width}; got {tuple(latents.shape)}")
        L.require_cuda(te, latents)
        sched = self._schedule(num_inference_steps)
        eng = self._engine_for(height, "unet")
        ptype = PREDICTION_TYPES[self.prediction_type]
        te = L.f32c(te.detach())
        out = latents.detach().to(torch.float32).clone(memory_format=torch.contiguous_format)
        with eng.on_stream():
            for b in range(B):
                ctx = torch.stack([te[b], te[B + b]])
                L.check(L.lib().mi3d_sd_sample(eng.h, L.ptr(out[b]), L.ptr(sched), C.c_int(num_inference_steps), C.c_int(ptype), L.ptr(ctx),
                                               C.c_float(float(guidance_scale)), L.stream()), "sd_sample")
        return out

    def prompt_to_img(self, prompts, negative_prompts='', height=512, width=512, num_inference_steps=50, guidance_scale=7.5, latents=None):
        """nerf/sd.py:222-238: get_text_embeds per prompt -> produce_latents -> decode_latents -> imgs [B,3,H,W] in [0,1].  prompts /
        negative_prompts: a string or int64 token ids [1,77] / [77], or a list of them (strings need the tokenizer)."""
        one = lambda p: [p] if isinstance(p, str) or torch.is_tensor(p) else list(p)
        prompts, negs = one(prompts), one(negative_prompts)
        if len(negs) == 1:
            negs = negs * len(prompts)
        if len(negs) != len(prompts):
            raise L.Mi3dError(f"{len(prompts)} prompts but {len(negs)} negative prompts")
        embeds = [self.get_text_embeds(p, n) for p, n in zip(prompts, negs)]
        text_embeds = torch.cat([e[:1] for e in embeds] + [e[1:] for e in embeds])
        latents = self.produce_latents(text_embeds, height=height, width=width, latents=latents, num_inference_steps=num_inference_steps,
                                       guidance_scale=guidance_scale)
        return self.decode_latents(latents)

    @classmethod
    def from_pretrained(cls, local_dir, device, step_range=[0.2, 0.6], graph_replay=True, defer_backward=False):
        """A local diffusers directory (nothing is downloaded): unet/ and vae/ config.json + diffusion_pytorch_model[.fp16].safetensors,
        text_encoder/ config.json + model[.fp16].safetensors, scheduler/scheduler_config.json, and tokenizer/ through transformers'
        CLIPTokenizer when transformers imports (without it prompts must be token ids).  The engine is planned at 512 x 512, the size
        train_step feeds (nerf/sd.py:124); other sampling sizes are planned on first use."""
        sub = lambda *p: os.path.join(local_dir, *p)
        unet_cfg = dict(unet_cfg_from_config(_read_json(sub("unet", "config.json"))), latent_hw=64)
        vae_cfg = dict(vae_cfg_from_config(_read_json(sub("vae", "config.json"))), image_hw=512)
        sched = scheduler_from_config(_read_json(sub("scheduler", "scheduler_config.json")))
        te_cfg = _read_json(sub("text_encoder", "config.json"))
        unet_state, vae_state = _read_weights(sub("unet"), "diffusion_pytorch_model"), _read_weights(sub("vae"), "diffusion_pytorch_model")
        te_state = _read_weights(sub("text_encoder"), "model")
        tokenizer = None
        if os.path.isdir(sub("tokenizer")):
            try:
                from transformers import CLIPTokenizer
            except ImportError:
                CLIPTokenizer = None
            if CLIPTokenizer is not None:
                tokenizer = CLIPTokenizer.from_pretrained(sub("tokenizer"))
        sd1 = unet_cfg.get("proj_conv", False)
        self = cls(device, sd_version="1.5" if sd1 else "2.0", hf_key=os.path.abspath(local_dir), step_range=step_range, unet_cfg=unet_cfg,
                   vae_cfg=vae_cfg, unet_state=unet_state, vae_state=vae_state, graph_replay=graph_replay, defer_backward=defer_backward,
                   tokenizer=tokenizer, strict=True)
        for k, v in sched.items():
            setattr(self, k, v)
        act = te_cfg.get("hidden_act", "quick_gelu")
        self.text_encoder = TextEncoder(self.device, cfg=cfg_from_state_dict(te_state, hidden_act=act), state_dict=te_state, graph_replay=graph_replay)
        return self

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
        """nerf/sd.py:212-220 (the 512x512 interpolation of :124 is folded in: pass the render-resolution image).  imgs [G,3,H,W]:
        G images at once on the G-view engine."""
        hw = self.vae_cfg["image_hw"] // 8
        G = imgs.shape[0]
        if eps is None:
            eps = torch.randn(G, 4, hw, hw, device=self.device)
        return _EncodeImgs.apply(imgs, L.f32c(eps), self.views_engine(G))

    def decode_latents(self, latents):
        """nerf/sd.py:201-210: (vae.decode(latents / 0.18215).sample / 2 + 0.5).clamp(0, 1) -> [B,3,S,S]; no gradient, like the reference.
        latents [B,4,h,w] with h = w a multiple of 8: the engine's own size, or another one planned on first use (S = 8h)."""
        latents = L.f32c(latents.detach())
        if latents.dim() != 4 or latents.shape[1] != 4 or latents.shape[2] != latents.shape[3] or latents.shape[2] % 8:
            raise L.Mi3dError(f"decode_latents takes square latents [B,4,h,h] with h a multiple of 8; got {tuple(latents.shape)}")
        S = latents.shape[2] * 8
        eng = self._engine_for(S, "vae")
        imgs = torch.empty(latents.shape[0], 3, S, S, dtype=torch.float32, device=latents.device)
        with eng.on_stream():
            for b in range(latents.shape[0]):
                L.check(L.lib().mi3d_sd_decode(eng.h, L.ptr(latents[b]), L.ptr(imgs[b]), L.stream()), "sd_decode")
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
        """add_noise -> U-Net -> CFG -> SDS gradient (nerf/sd.py:138-170). t: device int64 [1]. Returns (noise_pred, grad).
        latents / noise [G,4,h,w] of G views at the one timestep t; text_embeddings [2G,77,D] laid out [uncond x G, cond x G]."""
        latents, noise, text_embeddings = L.f32c(latents.detach()), L.f32c(noise), L.f32c(text_embeddings)
        G = latents.shape[0]
        if noise.numel() != latents.numel() or text_embeddings.dim() != 3 or text_embeddings.shape[0] != 2 * G:
            raise L.Mi3dError(f"unet_sds: latents and noise [G,4,h,w] and text_embeddings [2G,77,D] expected; got {tuple(latents.shape)}, "
                              f"{tuple(noise.shape)}, {tuple(text_embeddings.shape)}")
        eng = self.views_engine(G)
        noise_pred = torch.empty_like(latents)
        grad = torch.empty_like(latents)
        with eng.on_stream():
            L.check(L.lib().mi3d_sd_unet_sds(eng.h, L.ptr(latents), L.ptr(noise), L.ptr(t), L.ptr(self.alphas), L.ptr(text_embeddings),
                                             C.c_float(float(guidance_scale)), L.ptr(noise_pred), L.ptr(grad), L.stream()), "sd_unet_sds")
        return noise_pred, grad

    def train_step(self, text_embeddings, pred_rgb, ref_rgb=None, noise=None, islarge=False, ref_text=None, clip_model=None,
                   guidance_scale=10, t=None, eps_posterior=None, defer=None):
        """nerf/sd.py:117-174.  `noise` is accepted and ignored like the reference (:140) unless `t` is also injected
        (additive test hook: t, eps_posterior, noise make the step deterministic).  `defer` overrides the constructor's
        defer_backward for this call (None keeps it)."""
        defer = self.defer_backward if defer is None else bool(defer)
        if pred_rgb.shape[0] > 1:
            return self._train_step_views(text_embeddings, pred_rgb, ref_rgb, noise, islarge, ref_text, clip_model, guidance_scale, t,
                                          eps_posterior, defer)
        loss, imgs = 0, None
        if t is None:
            t_host = int(torch.randint(self.min_step, self.max_step + 1, [1]).item())     # CPU generator: no device sync
            noise = None
        else:
            t_host = int(t)
        self._t.fill_(t_host)
        if defer and not (not islarge and (t_host / self.num_train_timesteps) <= 0.4):
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
            self.last = dict(latents=latents, noise_pred=noise_pred, grad=grad, t=t_host, grad_rgb=grad_rgb)
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

    def _train_step_views(self, text_embeddings, pred_rgb, ref_rgb, noise, islarge, ref_text, clip_model, guidance_scale, t, eps_posterior,
                          defer):
        """train_step on G = pred_rgb.shape[0] views at one timestep: one encode, one U-Net pass at batch 2G and one encode backward on
        the G-view engine.  text_embeddings [2,77,D] (shared) or [2G,77,D] ([uncond x G, cond x G]); islarge a bool or G bools; noise /
        eps_posterior [G,4,h,w]; ref_rgb / ref_text one shared row or one per view.  Each view takes the reference's branch on its own:
        large views, or t > 0.4 T, the SDS gradient; the others the denoise branch (DDIM step, decode, CLIP), without a gradient.
        Returns (loss, imgs): loss = the denoise views' summed CLIP value (+ the SDS surrogate summed over the SDS views with defer),
        imgs = a list of G decoded images, None for SDS views.  Without defer the SDS gradient is back-propagated here, as at G = 1."""
        G, hw = pred_rgb.shape[0], self.vae_cfg["image_hw"] // 8
        large = [bool(islarge)] * G if isinstance(islarge, (bool, int)) else [bool(x) for x in islarge]
        te = L.f32c(text_embeddings)
        if len(large) != G or te.dim() != 3 or te.shape[0] not in (2, 2 * G):
            raise L.Mi3dError(f"train_step on {G} views: islarge takes a bool or {G} of them, text_embeddings [2,77,D] or [{2 * G},77,D]; got "
                              f"{len(large)} flags and {tuple(te.shape)}")
        if te.shape[0] == 2:
            te = torch.cat([te[:1].expand(G, -1, -1), te[1:].expand(G, -1, -1)]).contiguous()
        if t is None:
            t_host = int(torch.randint(self.min_step, self.max_step + 1, [1]).item())     # CPU generator: no device sync
            noise = None
        else:
            t_host = int(t)
        self._t.fill_(t_host)
        sds = [lg or t_host / self.num_train_timesteps > 0.4 for lg in large]
        eng = self.views_engine(G)
        rgb = L.f32c(pred_rgb.detach())
        H, W = rgb.shape[-2:]
        with torch.no_grad():
            eps = L.f32c(eps_posterior) if eps_posterior is not None else torch.randn(G, 4, hw, hw, device=self.device)
            latents = torch.empty(G, 4, hw, hw, dtype=torch.float32, device=rgb.device)
            with eng.on_stream():
                L.check(L.lib().mi3d_sd_encode(eng.h, L.ptr(rgb), C.c_int(H), C.c_int(W), L.ptr(eps), L.ptr(latents), L.stream()), "sd_encode")
            if noise is None:
                noise = torch.randn_like(latents)
            noise = L.f32c(noise)
            noise_pred, grad = self.unet_sds(latents, noise, self._t, te, guidance_scale)
            loss, imgs = 0, [None] * G
            if not all(sds):
                a = self.alphas[t_host]
                for v in range(G):
                    if sds[v]:
                        continue
                    grad[v].zero_()
                    if not self.vae_cfg.get("decoder", True):
                        continue
                    latents_noisy = a.sqrt() * latents[v:v + 1] + (1 - a).sqrt() * noise[v:v + 1]     # scheduler.add_noise (nerf/sd.py:141)
                    pick = lambda x: x[v:v + 1] if torch.is_tensor(x) and x.dim() > 0 and x.shape[0] == G else x
                    lv, imgs[v] = self._denoise_branch(noise_pred[v:v + 1], latents_noisy, pick(ref_rgb), pick(ref_text), clip_model)
                    loss = loss + lv
            grad_rgb = None
            if any(sds):
                grad_rgb = torch.empty_like(rgb)
                with eng.on_stream():
                    L.check(L.lib().mi3d_sd_encode_backward(eng.h, L.ptr(grad), L.ptr(eps), C.c_int(H), C.c_int(W), L.ptr(grad_rgb), L.stream()),
                            "sd_encode_backward")
        self.last = dict(latents=latents, noise_pred=noise_pred, grad=grad, t=t_host, sds=sds, denoise=loss, grad_rgb=grad_rgb)
        if grad_rgb is not None and pred_rgb.requires_grad:
            if defer:
                loss = loss + (grad_rgb * pred_rgb).sum()
            else:
                torch.autograd.backward(pred_rgb, grad_rgb, retain_graph=True)
        return loss, imgs


def main(argv=None):
    """nerf/sd.py:241-268: `python -m mi3d_b200.nerf.sd PROMPT --ckpt DIR` writes test_bench/<workspace>/<prompt>_<seed>.png for seeds
    0..--seeds-1 (the reference's default of 0 writes nothing)"""
    import argparse
    parser = argparse.ArgumentParser(description="text-to-image with a local diffusers Stable Diffusion checkpoint")
    parser.add_argument('prompt', type=str)
    parser.add_argument('--ckpt', required=True, type=str, help="local diffusers directory (unet/, vae/, text_encoder/, scheduler/, tokenizer/)")
    parser.add_argument('--negative', default='', type=str)
    parser.add_argument('--workspace', default='', type=str)
    parser.add_argument('--sd_version', type=str, default='2.0', choices=['1.5', '2.0'], help="stable diffusion version")
    parser.add_argument('-H', type=int, default=512)
    parser.add_argument('-W', type=int, default=512)
    parser.add_argument('--seeds', type=int, default=0)
    parser.add_argument('--steps', type=int, default=50)
    opt = parser.parse_args(argv)

    workspace = os.path.join('test_bench', opt.workspace)
    os.makedirs(workspace, exist_ok=True)
    sd = StableDiffusion.from_pretrained(opt.ckpt, torch.device('cuda'))
    if (opt.sd_version == '1.5') != bool(sd.unet_cfg.get("proj_conv", False)):
        raise L.Mi3dError(f"--sd_version {opt.sd_version} does not match {opt.ckpt}, an SD-{'1.x' if sd.unet_cfg.get('proj_conv') else '2.x'} U-Net")
    for seed in range(opt.seeds):
        torch.manual_seed(seed)
        np.random.seed(seed)
        imgs = sd.prompt_to_img(opt.prompt, opt.negative, opt.H, opt.W, opt.steps, guidance_scale=7.5)
        img = (imgs[0].permute(1, 2, 0).clamp(0, 1) * 255 + 0.5).to(torch.uint8).cpu().numpy()    # torchvision save_image's rounding
        path = os.path.join(workspace, opt.prompt.replace(" ", "_") + f'_{seed}.png')
        try:
            from PIL import Image
            Image.fromarray(img).save(path)
        except ImportError:
            import cv2
            cv2.imwrite(path, img[..., ::-1])
        print(path)


if __name__ == '__main__':
    main()
