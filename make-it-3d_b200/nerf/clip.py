"""B4 seam: openai CLIP ViT (`clip.load("ViT-B/16")`, nerf/utils.py:248) for the per-step CLIP losses, on libmi3d.so.

`CLIP(device, cfg=None, state_dict=None, seed=0, graph_replay=True)` is an `nn.Module` whose frozen parameters carry openai's
state_dict names (`model.state_dict()` keys are openai's; `load_openai_state_dict(clip.load(...)[0].state_dict())` loads real weights).
Everything between the image / token ids and the features runs in the engine of csrc/clip_engine.cu (tile GEMM, fused attention,
fused memory-bound kernels); there is no CPU or eager-PyTorch fallback.

* `encode_image(image)`: drop-in for openai's method: `[B,3,224,224]` already augmented -> `[B,embed_dim]`, with an input gradient.
* `encode_text(tokens)`: `[B,77]` int64 (`clip.tokenize` ids; the tokenizer is not part of this package) -> `[B,embed_dim]`, no gradient.
* `losses(rgb, ref_rgb, tokens) -> (img_loss, text_loss)`: the reference's `img_clip_loss(rgb, ref_rgb)` and
  `img_text_clip_loss(rgb, prompt)` (nerf/utils.py:436-453) with the reference's `aug` applied natively (bilinear resize to 224,
  align_corners=False, no antialiasing, then CLIP's Normalize).  `rgb` and `ref_rgb` are encoded in one batched pass and the
  backward runs once, for `rgb` only; the reference encodes `rgb` twice, which gives the same values and, by linearity, the same
  gradient.  No gradient flows to `ref_rgb`.  Normalisation, dot products and the mean stay in torch on the `[B,embed_dim]` features.
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from .. import _lib as L


class ClipCfg(C.Structure):
    _fields_ = [("image_res", C.c_int), ("patch", C.c_int), ("width", C.c_int), ("layers", C.c_int), ("heads", C.c_int),
                ("embed_dim", C.c_int), ("context_len", C.c_int), ("vocab", C.c_int), ("text_width", C.c_int), ("text_layers", C.c_int),
                ("text_heads", C.c_int), ("max_batch", C.c_int)]


def vit_b16_cfg():
    """openai CLIP ViT-B/16"""
    return dict(image_res=224, patch=16, width=768, layers=12, heads=12, embed_dim=512,
                context_len=77, vocab=49408, text_width=512, text_layers=12, text_heads=8)


def _cfg_struct(cfg, max_batch):
    s = ClipCfg()
    for k, _ in ClipCfg._fields_:
        setattr(s, k, int(max_batch if k == "max_batch" else cfg[k]))
    return s


class ClipEngine(L.Engine):
    """The CLIP engine (mi3d_clip_create): image and text towers planned in one workspace."""

    def __init__(self, cfg, device, graph_replay=True, max_batch=2):
        self.cfg = _cfg_struct(cfg, max_batch)
        super().__init__("clip", (C.byref(self.cfg),), device, graph_replay, f"CLIP configuration {cfg}")
        self.tape_id = 0          # bumped by every image forward: each one replaces the engine's tape

    def encode_image(self, img, aug, need_grad):
        img = L.f32c(img)
        L.require_cuda(img)
        B, ch, H, W = img.shape
        if ch != 3:
            raise L.Mi3dError("encode_image expects [B,3,H,W]")
        feats = torch.empty(B, self.cfg.embed_dim, dtype=torch.float32, device=img.device)
        with self.on_stream():
            L.check(L.lib().mi3d_clip_encode_image(self.h, L.ptr(img), C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(int(aug)),
                                                   C.c_int(int(need_grad)), L.ptr(feats), L.stream()), "clip_encode_image")
        self.tape_id += 1
        return feats

    def encode_image_backward(self, dfeats, n_grad, H, W):
        dfeats = L.f32c(dfeats)
        dimg = torch.empty(n_grad, 3, H, W, dtype=torch.float32, device=dfeats.device)
        with self.on_stream():
            L.check(L.lib().mi3d_clip_encode_image_backward(self.h, L.ptr(dfeats), C.c_int(n_grad), L.ptr(dimg), L.stream()),
                    "clip_encode_image_backward")
        return dimg

    def encode_text(self, tokens):
        L.require_cuda(tokens)
        tokens = tokens.to(torch.long).contiguous()
        if tokens.dim() != 2 or tokens.shape[1] != self.cfg.context_len:
            raise L.Mi3dError(f"encode_text expects int64 [B,{self.cfg.context_len}] token ids")
        feats = torch.empty(tokens.shape[0], self.cfg.embed_dim, dtype=torch.float32, device=tokens.device)
        with self.on_stream():
            L.check(L.lib().mi3d_clip_encode_text(self.h, L.ptr(tokens), C.c_int(tokens.shape[0]), L.ptr(feats), L.stream()),
                    "clip_encode_text")
        return feats


class _EncodeImage(torch.autograd.Function):
    """feats = encode_image(aug(image)); the input gradient covers the first n_grad images (the rest get zeros)."""

    @staticmethod
    def forward(ctx, image, engine, aug, n_grad):
        feats = engine.encode_image(image, aug, n_grad > 0)
        ctx.engine, ctx.aug, ctx.n_grad, ctx.tape_id = engine, aug, n_grad, engine.tape_id
        if n_grad > 0:
            ctx.save_for_backward(image)
        return feats

    @staticmethod
    def backward(ctx, g):
        (image,) = ctx.saved_tensors
        eng, n = ctx.engine, ctx.n_grad
        if eng.tape_id != ctx.tape_id:
            # a later image forward replaced the engine's tape: rebuild it (same inputs, same result)
            eng.encode_image(image, ctx.aug, True)
        B, _, H, W = image.shape
        dimg = eng.encode_image_backward(g[:n], n, H, W)
        if n < B:
            dimg = torch.cat([dimg, dimg.new_zeros(B - n, 3, H, W)])
        return dimg.to(image.dtype), None, None, None


class CLIP(nn.Module):
    def __init__(self, device, cfg=None, state_dict=None, seed=0, graph_replay=True, max_batch=2):
        super().__init__()
        self.device = torch.device(device)
        self.cfg = dict(cfg or vit_b16_cfg())
        self.engine = ClipEngine(self.cfg, self.device, graph_replay=graph_replay, max_batch=max_batch)
        gen = torch.Generator().manual_seed(seed)
        for name, shape in zip(self.engine.names, self.engine.shapes):
            if "#" in name:
                continue
            t = state_dict[name].detach().float() if (state_dict is not None and name in state_dict) else _default_init(name, shape, gen, self.cfg)
            *path, leaf = name.split(".")
            m = self
            for part in path:
                if part not in m._modules:
                    m.add_module(part, nn.Module())
                m = m._modules[part]
            m.register_parameter(leaf, nn.Parameter(t.reshape(shape).to(self.device).contiguous(), requires_grad=False))
        self.reload()

    def load_openai_state_dict(self, sd):
        """copy tensors named like openai CLIP's state_dict() (fp16 or fp32) and push them to the engine"""
        own = dict(self.named_parameters())
        with torch.no_grad():
            for k, p in own.items():
                p.copy_(sd[k].to(p.device, torch.float32).reshape(p.shape))
        self.reload()
        return self

    def reload(self):
        """push the current parameter values into the engine again (after load_state_dict)"""
        self.engine.load({k: p.data for k, p in self.named_parameters()})

    def encode_image(self, image):
        """openai CLIP.encode_image: image [B,3,res,res], already augmented -> [B,embed_dim]"""
        need = torch.is_grad_enabled() and image.requires_grad
        return _EncodeImage.apply(image, self.engine, 0, image.shape[0] if need else 0)

    def encode_text(self, tokens):
        """openai CLIP.encode_text: token ids [B,77] -> [B,embed_dim]; no gradient"""
        return self.engine.encode_text(tokens)

    def losses(self, rgb, ref_rgb, tokens):
        """(img_clip_loss(rgb, ref_rgb), img_text_clip_loss(rgb, tokens)) of nerf/utils.py:436-453, aug included"""
        n = rgb.shape[0]
        need = torch.is_grad_enabled() and rgb.requires_grad
        if rgb.shape[1:] == ref_rgb.shape[1:] and n + ref_rgb.shape[0] <= self.engine.cfg.max_batch:
            z = _EncodeImage.apply(torch.cat([rgb, ref_rgb.detach().to(rgb.dtype)]), self.engine, 1, n if need else 0)
            z1, z2 = z[:n], z[n:]
        else:
            # different sizes: two passes, the one with the tape last
            z2 = _EncodeImage.apply(ref_rgb.detach(), self.engine, 1, 0)
            z1 = _EncodeImage.apply(rgb, self.engine, 1, n if need else 0)
        zt = self.encode_text(tokens)
        z1 = z1 / z1.norm(dim=-1, keepdim=True)
        z2 = z2 / z2.norm(dim=-1, keepdim=True)
        zt = zt / zt.norm(dim=-1, keepdim=True)
        return -(z1 * z2).sum(-1).mean(), -(z1 * zt).sum(-1).mean()


def _default_init(name, shape, gen, cfg):
    """seeded stand-in weights (no CLIP weights exist offline): openai's initialisers in spirit"""
    if name.endswith(".weight") and len(shape) == 1:           # LayerNorms
        return torch.ones(shape)
    if len(shape) == 0:                                         # logit_scale
        return torch.full((), math.log(1 / 0.07))
    if name.endswith(".bias"):
        return torch.zeros(shape)
    if name == "token_embedding.weight":
        return torch.randn(shape, generator=gen) * 0.02
    if name == "positional_embedding":
        return torch.randn(shape, generator=gen) * 0.01
    fan_in = shape[0] if name.endswith(("proj", "projection", "embedding")) else math.prod(shape[1:])
    return torch.randn(shape, generator=gen) * fan_in ** -0.5
