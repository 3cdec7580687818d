"""fp32 torch restatement of openai CLIP's ViT model (clip/model.py: VisionTransformer, the text Transformer, encode_image,
encode_text), keyed by openai's state_dict names, plus the reference's `aug` and its two CLIP losses (nerf/utils.py:323-326,
436-453; nerf/sd.py:49-52, 97-114).  Test infrastructure only (CPU, fp32).

`aug` is `Resize((224, 224))` + `Normalize(CLIP mean, std)` as torchvision 0.11 applied it to a tensor (the version matching the
reference's pinned torch 1.10): bilinear, align_corners=False, NO antialiasing.  Modern torchvision antialiases tensors by default;
that is not what the reference computes.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def vit_b16_config():
    """clip.load("ViT-B/16") (nerf/utils.py:248)"""
    return dict(image_res=224, patch=16, width=768, layers=12, heads=12, embed_dim=512,
                context_len=77, vocab=49408, text_width=512, text_layers=12, text_heads=8)


def tiny_config():
    return dict(image_res=64, patch=16, width=128, layers=2, heads=2, embed_dim=128,
                context_len=77, vocab=49408, text_width=128, text_layers=2, text_heads=2)


def aug(x, res=224):
    x = F.interpolate(x, (res, res), mode="bilinear", align_corners=False, antialias=False)
    mean = torch.tensor(CLIP_MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


class QuickGELU(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d, heads, causal_len=None):
        super().__init__()
        self.attn = nn.MultiheadAttention(d, heads)
        self.ln_1 = nn.LayerNorm(d)
        self.mlp = nn.Sequential()
        self.mlp.add_module("c_fc", nn.Linear(d, 4 * d))
        self.mlp.add_module("gelu", QuickGELU())
        self.mlp.add_module("c_proj", nn.Linear(4 * d, d))
        self.ln_2 = nn.LayerNorm(d)
        self.causal_len = causal_len

    def forward(self, x):                                  # x [T, B, d] (openai's sequence-first layout)
        mask = None
        if self.causal_len is not None:
            mask = torch.full((self.causal_len, self.causal_len), float("-inf"), dtype=x.dtype, device=x.device).triu_(1)
        h = self.ln_1(x)
        x = x + self.attn(h, h, h, need_weights=False, attn_mask=mask)[0]
        return x + self.mlp(self.ln_2(x))


class Transformer(nn.Module):
    def __init__(self, d, layers, heads, causal_len=None):
        super().__init__()
        self.resblocks = nn.Sequential(*[ResidualAttentionBlock(d, heads, causal_len) for _ in range(layers)])

    def forward(self, x):
        return self.resblocks(x)


class VisionTransformer(nn.Module):
    def __init__(self, res, patch, width, layers, heads, out_dim):
        super().__init__()
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch, stride=patch, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((res // patch) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = Transformer(width, layers, heads)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, out_dim))      # [in, out]: x @ proj

    def forward(self, x):
        x = self.conv1(x)
        x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
        cls = self.class_embedding + torch.zeros(x.shape[0], 1, x.shape[-1], dtype=x.dtype, device=x.device)
        x = torch.cat([cls, x], dim=1) + self.positional_embedding
        x = self.ln_pre(x)
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        return self.ln_post(x[:, 0, :]) @ self.proj


class CLIPRef(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        c = cfg
        self.cfg = dict(cfg)
        self.visual = VisionTransformer(c["image_res"], c["patch"], c["width"], c["layers"], c["heads"], c["embed_dim"])
        self.transformer = Transformer(c["text_width"], c["text_layers"], c["text_heads"], causal_len=c["context_len"])
        self.token_embedding = nn.Embedding(c["vocab"], c["text_width"])
        self.positional_embedding = nn.Parameter(torch.empty(c["context_len"], c["text_width"]))
        self.ln_final = nn.LayerNorm(c["text_width"])
        self.text_projection = nn.Parameter(torch.empty(c["text_width"], c["embed_dim"]))
        self.logit_scale = nn.Parameter(torch.ones([]) * math.log(1 / 0.07))

    def encode_image(self, image):
        return self.visual(image)

    def encode_text(self, text):
        x = self.token_embedding(text) + self.positional_embedding
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        x = self.ln_final(x)
        return x[torch.arange(x.shape[0]), text.argmax(dim=-1)] @ self.text_projection


def default_init(model, seed=0):
    """Seeded initialisation in the spirit of openai's CLIP.initialize_parameters (no weights exist offline).  LayerNorms get some
    spread so every normalisation carries signal."""
    g = torch.Generator().manual_seed(seed)
    c = model.cfg
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() == 1 and (".ln_" in name or name.startswith("ln_") or "ln_final" in name or "ln_pre" in name or "ln_post" in name):
                if name.endswith("weight"):
                    p.copy_(torch.rand(p.shape, generator=g) * 0.4 + 0.8)
                else:
                    p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * 0.1)
            elif name == "logit_scale":
                p.fill_(math.log(1 / 0.07))
            elif p.dim() == 1:                       # biases, class embedding
                std = c["width"] ** -0.5 if "class_embedding" in name else 0.02
                p.copy_(torch.randn(p.shape, generator=g) * std)
            else:
                fan_in = p[0].numel() if not name.endswith(("proj", "text_projection", "positional_embedding")) else p.shape[0]
                if name.endswith("token_embedding.weight"):
                    std = 0.02
                elif name.endswith("positional_embedding"):
                    std = 0.01 if not name.startswith("visual") else c["width"] ** -0.5
                else:
                    std = fan_in ** -0.5
                p.copy_(torch.randn(p.shape, generator=g) * std)
    return model


def img_clip_loss(model, rgb1, rgb2, aug_fn=aug):
    """nerf/utils.py:436-443"""
    image_z_1 = model.encode_image(aug_fn(rgb1))
    image_z_2 = model.encode_image(aug_fn(rgb2))
    image_z_1 = image_z_1 / image_z_1.norm(dim=-1, keepdim=True)
    image_z_2 = image_z_2 / image_z_2.norm(dim=-1, keepdim=True)
    return - (image_z_1 * image_z_2).sum(-1).mean()


def img_text_clip_loss(model, rgb, text_tokens, aug_fn=aug):
    """nerf/utils.py:445-453, with clip.tokenize(prompt) done by the caller"""
    image_z_1 = model.encode_image(aug_fn(rgb))
    image_z_1 = image_z_1 / image_z_1.norm(dim=-1, keepdim=True)
    text_z = model.encode_text(text_tokens)
    text_z = text_z / text_z.norm(dim=-1, keepdim=True)
    return - (image_z_1 * text_z).sum(-1).mean()


def make_tokens(lengths, context_len=77, vocab=49408, seed=0):
    """clip.tokenize-shaped ids: SOT (vocab-2), words, EOT (vocab-1) at position length-1, zero padding"""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros(len(lengths), context_len, dtype=torch.long)
    for i, n in enumerate(lengths):
        out[i, 0] = vocab - 2
        if n > 2:
            out[i, 1:n - 1] = torch.randint(1, vocab - 2, (n - 2,), generator=g)
        out[i, n - 1] = vocab - 1
    return out
