"""The lifecycle every planned engine shares (include/mi3d.h, "Planned engines"): the generic mi3d_engine_* accessors reach each of the
seven engines, an index out of range is refused cleanly, and an engine's own entry points refuse another engine's handle with
MI3D_ERR_ARG before any device work."""
import ctypes as C
import importlib
import math

import pytest
import torch

from oracle import clip_ref, sd_ref, sd_text_ref

pytestmark = pytest.mark.gpu


def _m(name):
    return importlib.import_module("make-it-3d_b200." + name)


def _blip2_small_cfg():
    return dict(image_size=56, patch=14, vision_width=704, vision_layers=2, vision_heads=8, vision_mlp=1024,
                qformer_width=128, qformer_layers=3, qformer_heads=2, qformer_ffn=256, cross_attention_frequency=2,
                num_query_tokens=32, opt_width=320, opt_layers=2, opt_heads=4, opt_ffn=640, vocab=1000, max_positions=128,
                image_token_index=998, bos_token_id=2, eos_token_id=50)


@pytest.fixture(scope="module")
def engines():
    sd = _m("nerf.sd")
    return {
        "sd": sd.SDEngine(dict(sd_ref.tiny_unet_config(), latent_hw=32), dict(sd_ref.tiny_vae_config(), image_hw=256), "cuda"),
        "sd_text": _m("nerf.sd_text").TextEncoder("cuda", cfg=sd_text_ref.tiny_config()),
        "clip": _m("nerf.clip").ClipEngine(clip_ref.tiny_config(), "cuda"),
        "cx": _m("nerf.contextual_loss").CxEngine(1, 32, 32, "cuda"),
        "unet": _m("nerf.unet").UNetEngine(1, 16, 16, "cuda"),
        "dpt": _m("nerf.dpt").DPTDepthModel(),
        "blip2": _m("nerf.blip2").Blip2ForConditionalGeneration(cfg=_blip2_small_cfg()),
    }


# a registry entry of each engine, with its shape
KNOWN = {
    "sd": ("conv_in.weight", (64, 4, 3, 3)),
    "sd_text": ("text_model.embeddings.position_embedding.weight", (77, 128)),
    "clip": ("visual.conv1.weight", (128, 3, 16, 16)),
    "cx": ("vgg_model.slice1.0.weight#dgrad", (4, 64, 3, 3)),
    "unet": ("start.block.norm.num_batches_tracked", ()),
    "dpt": ("scratch.output_conv.4.bias", (1,)),
    "blip2": ("vision_model.embeddings.patch_embedding.weight", (704, 3, 14, 14)),
}


@pytest.mark.parametrize("kind", list(KNOWN))
def test_generic_accessors_reach_every_engine(engines, kind):
    L = _m("_lib")
    lib, e = L.lib(), engines[kind]
    n = lib.mi3d_engine_num_params(e.h)
    assert n > 0 and n == len(e.names) == len(e.shapes) and len(set(e.names)) == n
    name, shape = KNOWN[kind]
    assert e.shapes[e.names.index(name)] == shape
    shp = (C.c_int * 4)()
    for i in (0, n - 1):
        assert lib.mi3d_engine_param_name(e.h, i).decode() == e.names[i]
        r = lib.mi3d_engine_param_shape(e.h, i, shp)
        assert r == len(e.shapes[i]) and tuple(shp[k] for k in range(r)) == e.shapes[i]
    assert all(math.prod(s) > 0 for s in e.shapes)
    # a fresh engine has replayed nothing; replay can be switched off and on again
    assert e.graph_replays() == 0
    L.check(lib.mi3d_engine_set_graph_replay(e.h, 0), "set_graph_replay")
    L.check(lib.mi3d_engine_set_graph_replay(e.h, 0 if kind == "dpt" else 1), "set_graph_replay")
    with pytest.raises(L.Mi3dError):
        e.debug_tensor("no such tensor")


@pytest.mark.parametrize("kind", list(KNOWN))
def test_index_out_of_range_is_refused(engines, kind):
    L = _m("_lib")
    lib, e = L.lib(), engines[kind]
    n = len(e.names)
    shp = (C.c_int * 4)()
    src = torch.zeros(16, device="cuda")
    for i in (-1, n, n + 1000):
        assert lib.mi3d_engine_param_name(e.h, i) is None
        assert lib.mi3d_engine_param_shape(e.h, i, shp) == -1
        with pytest.raises(L.Mi3dError):
            L.check(lib.mi3d_engine_load_param(e.h, i, L.ptr(src), None, L.stream()), "load_param")
    assert lib.mi3d_engine_param_shape(e.h, 0, None) == -1


def test_null_handle_is_refused():
    L = _m("_lib")
    lib = L.lib()
    assert lib.mi3d_engine_num_params(None) == 0 and lib.mi3d_engine_param_name(None, 0) is None
    assert lib.mi3d_engine_param_shape(None, 0, (C.c_int * 4)()) == -1 and lib.mi3d_engine_graph_replays(None) == -1
    assert lib.mi3d_engine_set_graph_replay(None, 1) != 0
    lib.mi3d_engine_destroy(None)


def test_unet_weights_are_not_loaded(engines):
    """the refine U-Net reads its parameters on every call: loading one is refused"""
    L = _m("_lib")
    src = torch.zeros(16 * 19 * 9, device="cuda")
    with pytest.raises(L.Mi3dError):
        L.check(L.lib().mi3d_engine_load_param(engines["unet"].h, 0, L.ptr(src), None, L.stream()), "load_param")


def _calls(lib, p, s):
    """every engine-specific entry point with plausible arguments: p is a device buffer, s the stream"""
    i, f = C.c_int, C.c_float
    return {
        "sd": [lambda h: lib.mi3d_sd_encode(h, p, i(64), i(64), p, p, s),
               lambda h: lib.mi3d_sd_encode_backward(h, p, p, i(64), i(64), p, s),
               lambda h: lib.mi3d_sd_unet_sds(h, p, p, p, p, p, f(7.5), p, p, s),
               lambda h: lib.mi3d_sd_decode(h, p, p, s),
               lambda h: lib.mi3d_sd_profile(h, i(1), None, None)],
        "sd_text": [lambda h: lib.mi3d_sd_text_encode(h, p, i(1), p, s)],
        "clip": [lambda h: lib.mi3d_clip_encode_image(h, p, i(1), i(64), i(64), i(0), i(1), p, s),
                 lambda h: lib.mi3d_clip_encode_image_backward(h, p, i(1), p, s),
                 lambda h: lib.mi3d_clip_encode_text(h, p, i(1), p, s)],
        "cx": [lambda h: lib.mi3d_cx_forward(h, p, p, f(0.5), i(1), p, s),
               lambda h: lib.mi3d_cx_backward(h, p, p, s)],
        "unet": [lambda h: lib.mi3d_unet_forward(h, p, p, p, p, i(1), i(1), p, s),
                 lambda h: lib.mi3d_unet_backward(h, p, p, p, p, p, s)],
        "dpt": [lambda h: lib.mi3d_dpt_forward(h, p, p, s),
                lambda h: lib.mi3d_dpt_tap(h, i(0), p, s)],
        "blip2": [lambda h: lib.mi3d_blip2_encode(h, p, p, s),
                  lambda h: lib.mi3d_blip2_generate(h, p, i(4), C.c_longlong(-1), None, p, p, None, s),
                  lambda h: lib.mi3d_blip2_tap(h, b"image_embeds", p, s)],
    }


def test_another_engines_handle_is_refused(engines):
    L = _m("_lib")
    buf = torch.zeros(1 << 24, device="cuda")
    calls = _calls(L.lib(), L.ptr(buf), L.stream())
    kinds = list(engines)
    for k, fns in calls.items():
        for other in kinds:
            if other == k:
                continue
            for fn in fns:
                with pytest.raises(L.Mi3dError, match="MI3D_ERR_ARG"):
                    L.check(fn(engines[other].h), f"{k} entry point with a {other} handle")
        for fn in fns:
            with pytest.raises(L.Mi3dError, match="MI3D_ERR_ARG"):
                L.check(fn(None), f"{k} entry point with a NULL handle")
    torch.cuda.synchronize()
    assert not buf.any()          # nothing wrote to the buffer
