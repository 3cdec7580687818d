"""CPU: oracle/clip_ref.py (the fp32 restatement of openai CLIP the GPU tests compare against) pinned against transformers' independently
written CLIPModel at the ViT-B/16 configuration, its `aug` against torchvision, and the ctypes mirror of mi3d_clip_cfg against the header."""
import ctypes
import importlib
import os
import subprocess

import pytest
import torch

from oracle import clip_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hf_state(sd, cfg):
    """openai state_dict -> transformers CLIPModel state_dict"""
    out = {"logit_scale": sd["logit_scale"],
           "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
           "vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
           "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
           "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
           "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"], "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
           "visual_projection.weight": sd["visual.proj"].t(),
           "text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
           "text_projection.weight": sd["text_projection"].t()}
    for src, dst, n in (("visual.transformer", "vision_model.encoder", cfg["layers"]), ("transformer", "text_model.encoder", cfg["text_layers"])):
        for i in range(n):
            a, b = f"{src}.resblocks.{i}", f"{dst}.layers.{i}"
            for k, (w, bias) in enumerate(zip(sd[a + ".attn.in_proj_weight"].chunk(3), sd[a + ".attn.in_proj_bias"].chunk(3))):
                out[f"{b}.self_attn.{'qkv'[k]}_proj.weight"], out[f"{b}.self_attn.{'qkv'[k]}_proj.bias"] = w, bias
            for o, h in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                         ("mlp.c_proj", "mlp.fc2")):
                out[f"{b}.{h}.weight"], out[f"{b}.{h}.bias"] = sd[f"{a}.{o}.weight"], sd[f"{a}.{o}.bias"]
    return out


@pytest.fixture(scope="module")
def vit_b16():
    torch.manual_seed(0)
    cfg = clip_ref.vit_b16_config()
    return cfg, clip_ref.default_init(clip_ref.CLIPRef(cfg), seed=1).eval()


def test_oracle_matches_transformers_clip_vit_b16(vit_b16):
    transformers = pytest.importorskip("transformers")
    cfg, model = vit_b16
    c = cfg
    hf_cfg = transformers.CLIPConfig(
        text_config=dict(vocab_size=c["vocab"], hidden_size=c["text_width"], intermediate_size=4 * c["text_width"], num_hidden_layers=c["text_layers"],
                         num_attention_heads=c["text_heads"], max_position_embeddings=c["context_len"], hidden_act="quick_gelu",
                         layer_norm_eps=1e-5, eos_token_id=2),
        vision_config=dict(hidden_size=c["width"], intermediate_size=4 * c["width"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                           image_size=c["image_res"], patch_size=c["patch"], hidden_act="quick_gelu", layer_norm_eps=1e-5),
        projection_dim=c["embed_dim"])
    hf = transformers.CLIPModel(hf_cfg).eval()
    missing, unexpected = hf.load_state_dict(_hf_state(model.state_dict(), cfg), strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    assert sum(p.numel() for p in hf.parameters()) == sum(p.numel() for p in model.parameters()) == 149_620_737
    g = torch.Generator().manual_seed(2)
    img = clip_ref.aug(torch.rand(2, 3, 512, 512, generator=g))
    tok = clip_ref.make_tokens([5, 77], seed=3)
    with torch.no_grad():
        fi, ft = model.encode_image(img), model.encode_text(tok)
        hi = hf.visual_projection(hf.vision_model(pixel_values=img).pooler_output)
        ht = hf.text_projection(hf.text_model(input_ids=tok).pooler_output)
    ei, et = float((fi - hi).norm() / hi.norm()), float((ft - ht).norm() / ht.norm())
    print(f"oracle vs transformers: image features rel {ei:.2e}, text features rel {et:.2e}")
    assert ei <= 1e-5 and et <= 1e-5


def test_oracle_aug_is_torchvision_resize_without_antialias_and_normalize():
    T = pytest.importorskip("torchvision.transforms")
    g = torch.Generator().manual_seed(4)
    for hw in ((512, 512), (128, 128), (300, 200)):
        x = torch.rand(1, 3, *hw, generator=g)
        want = T.Compose([T.Resize((224, 224), antialias=False), T.Normalize(clip_ref.CLIP_MEAN, clip_ref.CLIP_STD)])(x)
        assert torch.equal(clip_ref.aug(x), want), hw


def test_clip_cfg_ctypes_mirror_matches_the_header(tmp_path):
    cls = importlib.import_module("make-it-3d_b200.nerf.clip").ClipCfg
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(mi3d_clip_cfg));']
    src += [f'  printf("{f} %zu\\n", offsetof(mi3d_clip_cfg, {f}));' for f, *_ in cls._fields_]
    src += ['  return 0;', '}']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, *_ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f
