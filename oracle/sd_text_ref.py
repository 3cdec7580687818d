"""fp32 torch restatement of the Stable Diffusion 2 text encoder: transformers' `CLIPTextModel` as SD-2.x ships it (OpenCLIP ViT-H/14's
text tower truncated to 23 layers), keyed by transformers' state_dict names, returning `last_hidden_state` (what nerf/sd.py:68-85 reads
as `text_encoder(ids)[0]`).  Test infrastructure only (CPU, fp32).

Pre-LN blocks: x += out_proj(attn(LN1(x))), x += fc2(gelu(fc1(LN2(x)))); attention is causal with 64-wide heads, q scaled by 1/8, and
no padding mask; final_layer_norm is applied to every position.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


def sd2_text_config():
    """text_encoder/config.json of stable-diffusion-2-base, 2-1-base and 2-1 (the same encoder)"""
    return dict(width=1024, layers=23, heads=16, context_len=77, vocab=49408)


def tiny_config():
    return dict(width=128, layers=2, heads=2, context_len=77, vocab=49408)


class Attention(nn.Module):
    def __init__(self, d, heads):
        super().__init__()
        self.heads = heads
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(d, d) for _ in range(4))

    def forward(self, x):                                   # x [B, T, d]
        B, T, d = x.shape
        split = lambda t: t.view(B, T, self.heads, d // self.heads).transpose(1, 2)
        q, k, v = split(self.q_proj(x)), split(self.k_proj(x)), split(self.v_proj(x))
        s = (q * (d // self.heads) ** -0.5) @ k.transpose(-1, -2)
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=x.device).triu(1), float("-inf"))
        o = F.softmax(s, dim=-1) @ v
        return self.out_proj(o.transpose(1, 2).reshape(B, T, d))


class Mlp(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.fc1, self.act, self.fc2 = nn.Linear(d, 4 * d), nn.GELU(), nn.Linear(4 * d, d)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class Layer(nn.Module):
    def __init__(self, d, heads):
        super().__init__()
        self.self_attn = Attention(d, heads)
        self.layer_norm1 = nn.LayerNorm(d)
        self.mlp = Mlp(d)
        self.layer_norm2 = nn.LayerNorm(d)

    def forward(self, x):
        x = x + self.self_attn(self.layer_norm1(x))
        return x + self.mlp(self.layer_norm2(x))


class Embeddings(nn.Module):
    def __init__(self, vocab, d, T):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, d)
        self.position_embedding = nn.Embedding(T, d)

    def forward(self, ids):
        return self.token_embedding(ids) + self.position_embedding.weight[:ids.shape[1]]


class Encoder(nn.Module):
    def __init__(self, d, layers, heads):
        super().__init__()
        self.layers = nn.ModuleList(Layer(d, heads) for _ in range(layers))


class TextModel(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.embeddings = Embeddings(c["vocab"], c["width"], c["context_len"])
        self.encoder = Encoder(c["width"], c["layers"], c["heads"])
        self.final_layer_norm = nn.LayerNorm(c["width"])


class TextEncoderRef(nn.Module):
    """`TextEncoderRef(cfg)(ids)[0]` = `CLIPTextModel(ids)[0]`: ids int64 [B, T] -> last_hidden_state [B, T, width]"""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = dict(cfg)
        self.text_model = TextModel(self.cfg)

    def forward(self, ids):
        x = self.text_model.embeddings(ids)
        for layer in self.text_model.encoder.layers:
            x = layer(x)
        return (self.text_model.final_layer_norm(x),)


def default_init(model, seed=0):
    """Seeded weights in the spirit of CLIP's initialisers (no SD-2 weights exist offline).  LayerNorms get some spread so every
    normalisation carries signal."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "layer_norm" in name:
                if name.endswith("weight"):
                    p.copy_(torch.rand(p.shape, generator=g) * 0.4 + 0.8)
                else:
                    p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * 0.1)
            elif name.endswith("token_embedding.weight"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif name.endswith("position_embedding.weight"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.01)
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            else:
                p.copy_(torch.randn(p.shape, generator=g) * p.shape[1] ** -0.5)
    return model


def make_ids(lengths, pad=0, context_len=77, vocab=49408, seed=0):
    """CLIPTokenizer-shaped ids: BOS (49406), words, EOS (49407) at position length-1, then `pad` (SD-2's tokenizer pads with id 0,
    openai's CLIP-L tokenizer with 49407).  A length above context_len is truncated to it, the EOS kept last, as truncation=True does."""
    g = torch.Generator().manual_seed(seed)
    out = torch.full((len(lengths), context_len), pad, dtype=torch.long)
    for i, n in enumerate(lengths):
        n = min(n, context_len)
        out[i, 0] = vocab - 2
        if n > 2:
            out[i, 1:n - 1] = torch.randint(1, vocab - 2, (n - 2,), generator=g)
        out[i, n - 1] = vocab - 1
    return out


def num_params(cfg):
    """parameter count from the shapes: embeddings + layers x (4 attention linears, 2 MLP linears, 2 LayerNorms) + final LayerNorm"""
    C, L = cfg["width"], cfg["layers"]
    per_layer = 4 * (C * C + C) + (4 * C * C + 4 * C) + (4 * C * C + C) + 4 * C
    return cfg["vocab"] * C + cfg["context_len"] * C + L * per_layer + 2 * C


def gemm_flops(cfg, B):
    """FLOPs of one encoder call's matrix products at B sequences of context_len tokens (2 per multiply-add): the linears over
    every token, plus Q K^T and P V over the full (unmasked) context of every head."""
    C, L, T = cfg["width"], cfg["layers"], cfg["context_len"]
    linear = 2 * B * T * (3 * C * C + C * C + 4 * C * C + 4 * C * C)
    attn = 2 * 2 * B * T * T * C
    return L * (linear + attn)

