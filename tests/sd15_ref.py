"""Test infrastructure: the SD-1.5 forms of the fp32 oracles, built from oracle/sd_ref.py and oracle/sd_text_ref.py as they stand.

* U-Net (`sd15_unet(cfg)`): diffusers' UNet2DConditionModel with `use_linear_projection: false`: every Transformer2DModel's
  proj_in / proj_out is a 1x1 Conv2d [C, C, 1, 1] applied to the feature map, proj_in before the token reshape and proj_out after
  the reshape back, as diffusers orders them.  `sd15_unet_config()`: stable-diffusion-v1-5's unet/config.json (attention_head_dim 8,
  i.e. 8 heads at every level, cross_attention_dim 768).
* Text encoder (`sd15_text_encoder(cfg)`): transformers' CLIPTextModel with hidden_act "quick_gelu" (OpenAI CLIP ViT-L/14's text
  tower, SD-1.x's text_encoder); `sd15_text_config()` is its config.json.

The state_dict names are those of the SD-2 forms; only the projection shapes and the activation differ.
"""
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import sd_ref, sd_text_ref  # noqa: E402


def sd15_unet_config():
    return dict(sd_ref.sd20_unet_config(), heads=(8, 8, 8, 8), cross_dim=768)


class ConvProjTransformer2DModel(sd_ref.Transformer2DModel):
    """Transformer2DModel with 1x1-conv projections on the [B, C, H, W] feature map"""

    def forward(self, x, ctx):
        B, C, H, W = x.shape
        h = self.proj_in(self.norm(x)).permute(0, 2, 3, 1).reshape(B, H * W, C)
        for blk in self.transformer_blocks:
            h = blk(h, ctx)
        return self.proj_out(h.reshape(B, H, W, C).permute(0, 3, 1, 2)) + x


def conv_projections(unet):
    """turn every transformer of an oracle U-Net into the conv-projection form (fresh Conv2d weights, PyTorch's default init)"""
    for m in unet.modules():
        if type(m) is sd_ref.Transformer2DModel:
            C = m.proj_in.in_features
            m.proj_in, m.proj_out = nn.Conv2d(C, C, 1), nn.Conv2d(C, C, 1)
            m.__class__ = ConvProjTransformer2DModel
    return unet


def sd15_unet(cfg=None):
    return conv_projections(sd_ref.UNet2DConditionModel(cfg or sd15_unet_config()))


def sd15_text_config():
    """text_encoder/config.json of stable-diffusion-v1-5"""
    return dict(width=768, layers=12, heads=12, context_len=77, vocab=49408)


class QuickGELU(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


def sd15_text_encoder(cfg=None):
    """TextEncoderRef with quick-GELU in every MLP (the activation holds no parameters: the state_dict is unchanged)"""
    model = sd_text_ref.TextEncoderRef(cfg or sd15_text_config())
    for layer in model.text_model.encoder.layers:
        layer.mlp.act = QuickGELU()
    return model
