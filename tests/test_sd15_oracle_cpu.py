"""CPU: the SD-1.5 oracles (tests/sd15_ref.py: the quick-GELU text encoder and the conv-projection U-Net built on oracle/) that the
GPU tests compare against, pinned against transformers' independently written CLIPTextModel (quick-GELU) and against the
linear-projection U-Net; and the host side of the SD-1.5 configuration (ctypes structs, workspace queries, the checkpoint requirement)."""
import ctypes
import importlib
import math

import pytest
import torch

import sd15_ref
from oracle import sd_ref, sd_text_ref


def test_text_oracle_matches_transformers_clip_text_model_at_the_sd15_config():
    transformers = pytest.importorskip("transformers")
    c = sd15_ref.sd15_text_config()
    torch.manual_seed(0)
    model = sd_text_ref.default_init(sd15_ref.sd15_text_encoder(c), seed=1).eval()
    hf_cfg = transformers.CLIPTextConfig(vocab_size=c["vocab"], hidden_size=c["width"], intermediate_size=4 * c["width"],
                                         num_hidden_layers=c["layers"], num_attention_heads=c["heads"], max_position_embeddings=c["context_len"],
                                         hidden_act="quick_gelu", layer_norm_eps=1e-5)
    hf = transformers.CLIPTextModel(hf_cfg).eval()
    sd = model.state_dict()
    hf_names = {k for k in hf.state_dict() if not k.endswith("position_ids")}
    assert hf_names == set(sd) and len(sd) == 196
    assert sum(p.numel() for p in hf.parameters()) == sum(p.numel() for p in model.parameters()) == sd_text_ref.num_params(c) == 123_060_480
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    lengths = (2, 11, 40, 77, 90)
    ids = torch.cat([sd_text_ref.make_ids(lengths, pad=c["vocab"] - 1, seed=2), sd_text_ref.make_ids((5, 30), pad=0, seed=3)])
    with torch.no_grad():
        got = model(ids)[0]
        want = hf(input_ids=ids).last_hidden_state
        gelu = sd_text_ref.TextEncoderRef(c)
        gelu.load_state_dict(sd)
        other = gelu(ids)[0]
    assert got.shape == (7, 77, c["width"])
    for i in range(ids.shape[0]):
        e = float((got[i] - want[i]).norm() / want[i].norm())
        print(f"prompt {i}: oracle vs transformers last_hidden_state rel {e:.2e}")
        assert e <= 1e-5, (i, e)
    # the activation matters: the exact-GELU tower with the same weights is far away
    assert float((other - want).norm() / want.norm()) > 1e-3


def test_sd15_unet_oracle_has_the_diffusers_parameters():
    with torch.device("meta"):
        sd15, sd20 = sd15_ref.sd15_unet(), sd_ref.UNet2DConditionModel(sd_ref.sd20_unet_config())
    assert sum(p.numel() for p in sd15.parameters()) == 859_520_964
    assert sum(p.numel() for p in sd20.parameters()) == 865_910_724
    s15, s20 = sd15.state_dict(), sd20.state_dict()
    assert list(s15) == list(s20)                                          # the same names, in the same order
    proj = [k for k in s15 if k.endswith(("proj_in.weight", "proj_out.weight"))]
    assert len(proj) == 32
    for k in proj:
        C = s15[k].shape[0]
        assert tuple(s15[k].shape) == (C, C, 1, 1) and tuple(s20[k].shape) == (C, C), k
    assert tuple(s15["down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight"].shape) == (320, 768)
    assert all(tuple(s15[k].shape) == tuple(s20[k].shape) for k in s15 if k not in proj and "attn2.to_k" not in k and "attn2.to_v" not in k)


def _conv_state(state):
    return {k: (v.view(*v.shape, 1, 1) if k.endswith(("proj_in.weight", "proj_out.weight")) else v) for k, v in state.items()}


def test_conv_projection_equals_linear_projection_with_reshaped_weights():
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(1)
    # one transformer in float64: the two orders of the same sums agree far below the bound
    lin = sd_ref.Transformer2DModel(128, 4, 96, 32).double().eval()
    conv = sd15_ref.conv_projections(sd_ref.Transformer2DModel(128, 4, 96, 32)).double().eval()
    conv.load_state_dict(_conv_state(lin.state_dict()))
    x = torch.randn(2, 128, 8, 8, generator=gen, dtype=torch.float64)
    ctx = torch.randn(2, 77, 96, generator=gen, dtype=torch.float64)
    with torch.no_grad():
        a, b = lin(x, ctx), conv(x, ctx)
    e = float((a - b).norm() / a.norm())
    print(f"Transformer2DModel conv vs linear projections (float64) rel {e:.2e}")
    assert e <= 1e-6
    # the whole tiny U-Net in float32: every transformer of the down, mid and up blocks takes the conv path
    cfg = dict(sd_ref.tiny_unet_config(), heads=(2, 2, 4))
    lin = sd_ref.UNet2DConditionModel(cfg).eval()
    conv = sd15_ref.conv_projections(sd_ref.UNet2DConditionModel(cfg)).eval()
    conv.load_state_dict(_conv_state(lin.state_dict()))
    x = torch.randn(2, 4, 16, 16, generator=gen)
    ctx = torch.randn(2, 77, cfg["cross_dim"], generator=gen)
    with torch.no_grad():
        a, b = lin(x, torch.tensor([500]), ctx), conv(x, torch.tensor([500]), ctx)
    e = float((a - b).double().norm() / a.double().norm())
    print(f"tiny U-Net conv vs linear projections (float32) rel {e:.2e}")
    assert e <= 1e-5


def _sd():
    return importlib.import_module("make-it-3d_b200.nerf.sd")


def test_sd15_python_configuration():
    sdm = _sd()
    c = sdm.sd15_unet_cfg()
    assert c["heads"] == (8, 8, 8, 8) and c["cross_dim"] == 768 and c["proj_conv"] is True
    assert [b // h for b, h in zip(c["block_out"], c["heads"])] == [40, 80, 160, 160]
    assert {k: v for k, v in c.items() if k != "proj_conv"} == dict(sdm.sd20_unet_cfg(), heads=(8, 8, 8, 8), cross_dim=768)
    assert sdm._unet_struct(c).proj_conv == 1 and sdm._unet_struct(sdm.sd20_unet_cfg()).proj_conv == 0
    s15 = {"down_blocks.0.attentions.0.proj_in.weight": torch.zeros(320, 320, 1, 1)}
    s20 = {"down_blocks.0.attentions.0.proj_in.weight": torch.zeros(320, 320)}
    assert sdm.is_sd1_unet_state(s15) and not sdm.is_sd1_unet_state(s20) and not sdm.is_sd1_unet_state(None)
    # no seeded SD-1.5: the checkpoint is required, and refused before any device work
    with pytest.raises(ValueError, match="state dicts"):
        sdm.StableDiffusion("cpu", sd_version="1.5")
    with pytest.raises(ValueError, match="state dicts"):
        sdm.StableDiffusion("cpu", sd_version="1.5", hf_key="runwayml/stable-diffusion-v1-5", vae_state={})


def test_text_cfg_activation():
    st = importlib.import_module("make-it-3d_b200.nerf.sd_text")
    L = importlib.import_module("make-it-3d_b200._lib")
    ref = sd_text_ref.TextEncoderRef(sd_text_ref.tiny_config())
    assert st.cfg_from_state_dict(ref.state_dict())["hidden_act"] == "gelu"
    c = st.cfg_from_state_dict(ref.state_dict(), hidden_act="quick_gelu")
    assert c == dict(width=128, layers=2, heads=2, context_len=77, vocab=49408, hidden_act="quick_gelu")
    with pytest.raises(L.Mi3dError):
        st.cfg_from_state_dict(ref.state_dict(), hidden_act="relu")
    assert st.sd15_text_cfg() == dict(width=768, layers=12, heads=12, context_len=77, vocab=49408, hidden_act="quick_gelu")
    assert st.sd2_text_cfg()["hidden_act"] == "gelu"


def test_workspace_queries_accept_sd15_and_reject_other_head_dims(mi3d):
    sdm, st = _sd(), importlib.import_module("make-it-3d_b200.nerf.sd_text")
    lib = mi3d.lib()
    lib.mi3d_sd_workspace_bytes.restype = ctypes.c_size_t
    lib.mi3d_sd_text_workspace_bytes.restype = ctypes.c_size_t
    lib.mi3d_sd_text_act_workspace_bytes.restype = ctypes.c_size_t
    ws = lambda cfg: lib.mi3d_sd_workspace_bytes(ctypes.byref(sdm._unet_struct(cfg)), None)
    w15, w20 = ws(sdm.sd15_unet_cfg()), ws(sdm.sd20_unet_cfg())
    # the same channels; SD-1.5's cross projections are narrower (768 inputs) and its proj weights the same size
    print(f"U-Net workspace: SD-1.5 {w15 / 2 ** 20:.1f} MiB, SD-2.0 {w20 / 2 ** 20:.1f} MiB")
    assert w15 > 0 and w20 > 0 and abs(w15 - w20) < 0.05 * w20
    for heads in ((8, 8, 8, 8), (5, 10, 20, 20)):
        assert ws(dict(sdm.sd15_unet_cfg(), heads=heads, block_out=(384, 640, 1280, 1280))) == 0      # head_dim 48 / 76.8
    assert ws(dict(sdm.sd20_unet_cfg(), heads=(4, 10, 20, 20))) > 0                               # head_dim 80 at level 0 is built too

    cfg = st.SdTextCfg(*(dict(sd15_ref.sd15_text_config(), max_batch=2)[f] for f, _ in st.SdTextCfg._fields_))
    tws = lambda act: lib.mi3d_sd_text_act_workspace_bytes(ctypes.byref(cfg), ctypes.c_int(act))
    full = tws(1)
    weights = 12 * 12 * 768 * 768 * 2 + (49408 + 77) * 768 * 4
    assert weights < full < weights + 64 * 2 ** 20, full
    # the activation changes the epilogue, not the plan's buffers; the plain entry point is the exact-GELU one
    assert tws(0) == full == lib.mi3d_sd_text_workspace_bytes(ctypes.byref(cfg))
    assert tws(2) == 0 and tws(-1) == 0
    assert math.isclose(sd_text_ref.num_params(sd15_ref.sd15_text_config()), 123_060_480)
