"""CPU: oracle/sd_text_ref.py (the fp32 restatement of the SD-2 text encoder the GPU tests compare against) pinned against transformers'
independently written CLIPTextModel at the SD-2 configuration, and the ctypes mirror of mi3d_sd_text_cfg against the header."""
import ctypes
import importlib
import os
import subprocess

import pytest
import torch

from oracle import sd_text_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_matches_transformers_clip_text_model_at_the_sd2_config():
    transformers = pytest.importorskip("transformers")
    c = sd_text_ref.sd2_text_config()
    torch.manual_seed(0)
    model = sd_text_ref.default_init(sd_text_ref.TextEncoderRef(c), seed=1).eval()
    hf_cfg = transformers.CLIPTextConfig(vocab_size=c["vocab"], hidden_size=c["width"], intermediate_size=4 * c["width"],
                                         num_hidden_layers=c["layers"], num_attention_heads=c["heads"], max_position_embeddings=c["context_len"],
                                         hidden_act="gelu", layer_norm_eps=1e-5)
    hf = transformers.CLIPTextModel(hf_cfg).eval()
    sd = model.state_dict()
    hf_names = {k for k in hf.state_dict() if not k.endswith("position_ids")}
    assert hf_names == set(sd) and len(sd) == 372
    assert sum(p.numel() for p in hf.parameters()) == sum(p.numel() for p in model.parameters()) == sd_text_ref.num_params(c) == 340_387_840
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    lengths = (2, 11, 40, 77, 90)                       # EOS at 1 (an empty prompt), 10, 39, 76, and a prompt truncated to 77
    ids = torch.cat([sd_text_ref.make_ids(lengths, pad=0, seed=2), sd_text_ref.make_ids((5, 30), pad=c["vocab"] - 1, seed=3)])
    with torch.no_grad():
        got = model(ids)[0]
        want = hf(input_ids=ids).last_hidden_state
    assert got.shape == (7, 77, c["width"])
    for i in range(ids.shape[0]):
        e = float((got[i] - want[i]).norm() / want[i].norm())
        print(f"prompt {i}: oracle vs transformers last_hidden_state rel {e:.2e}")
        assert e <= 1e-5, (i, e)


def test_make_ids_places_bos_eos_and_padding():
    ids = sd_text_ref.make_ids((2, 5, 100), pad=0)
    assert ids.shape == (3, 77) and ids.dtype == torch.long
    assert ids[0, :3].tolist() == [49406, 49407, 0] and (ids[0, 2:] == 0).all()
    assert ids[1, 4] == 49407 and (ids[1, 5:] == 0).all() and ((ids[1, 1:4] > 0) & (ids[1, 1:4] < 49406)).all()
    assert ids[2, 76] == 49407 and (ids[2, 1:76] < 49406).all()


def test_gemm_flops_counts_the_products_of_one_call():
    c = sd_text_ref.sd2_text_config()
    C, T = c["width"], c["context_len"]
    per_layer_linear = 2 * T * (12 * C * C)             # q, k, v, out (4 C^2) + fc1, fc2 (8 C^2) multiply-adds per token
    per_layer_attn = 2 * 2 * T * T * C                  # S = Q K^T and O = P V over all heads
    assert sd_text_ref.gemm_flops(c, 2) == 2 * c["layers"] * (per_layer_linear + per_layer_attn)


def test_sd_text_cfg_ctypes_mirror_matches_the_header(tmp_path):
    cls = importlib.import_module("make-it-3d_b200.nerf.sd_text").SdTextCfg
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(mi3d_sd_text_cfg));']
    src += [f'  printf("{f} %zu\\n", offsetof(mi3d_sd_text_cfg, {f}));' for f, *_ in cls._fields_]
    src += ['  return 0;', '}']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, *_ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


def test_text_encoder_refuses_cpu_only_use():
    m = importlib.import_module("make-it-3d_b200.nerf.sd_text")
    L = importlib.import_module("make-it-3d_b200._lib")
    with pytest.raises(L.Mi3dError):
        m.TextEncoder("cpu", cfg=sd_text_ref.tiny_config())


def test_workspace_query_is_pure_host_and_rejects_bad_configurations(mi3d):
    m = importlib.import_module("make-it-3d_b200.nerf.sd_text")
    lib = mi3d.lib()
    lib.mi3d_sd_text_workspace_bytes.restype = ctypes.c_size_t

    def ws(**kw):
        cfg = dict(sd_text_ref.sd2_text_config(), max_batch=2)
        cfg.update(kw)
        s = m.SdTextCfg(*(cfg[f] for f, _ in m.SdTextCfg._fields_))
        return lib.mi3d_sd_text_workspace_bytes(ctypes.byref(s))
    full = ws()
    # fp16 linears (12 C^2 per layer), fp32 embeddings / biases / LayerNorms, and one set of activation buffers
    weights = 23 * 12 * 1024 * 1024 * 2 + (49408 + 77) * 1024 * 4
    assert weights < full < weights + 64 * 2 ** 20, full
    assert ws(max_batch=8) > full
    for bad in (dict(max_batch=0), dict(max_batch=9), dict(heads=8), dict(width=1000), dict(layers=0), dict(vocab=0), dict(context_len=0)):
        assert ws(**bad) == 0, bad
