"""Time the SD-2 text encoder (nerf/sd_text.py) at the shape get_text_embeds runs: B = 2 ([uncond, cond]), 77 tokens, the full SD-2
configuration, seeded weights.  A/B arms on the same card: the fp32 oracle (oracle/sd_text_ref.py) in eager PyTorch, and transformers'
CLIPTextModel when it is importable.  Prints one JSON line (card name and power limit read in the same run).

  python tests/measure_sd_text.py [--calls 50] [--warmup 5]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import sd_text_ref  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else torch.cuda.get_device_name()


def time_calls(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_sd_text.py needs a GPU")
    st = importlib.import_module("make-it-3d_b200.nerf.sd_text")
    cfg = sd_text_ref.sd2_text_config()
    torch.manual_seed(0)
    ref = sd_text_ref.default_init(sd_text_ref.TextEncoderRef(cfg), seed=5).eval()
    sd = ref.state_dict()
    ids = sd_text_ref.make_ids((2, 11), pad=0, seed=7).cuda()
    free0 = torch.cuda.memory_allocated()
    enc = st.TextEncoder("cuda", cfg=cfg, state_dict=sd)
    footprint = torch.cuda.memory_allocated() - free0
    flops = sd_text_ref.gemm_flops(cfg, 2)
    res = dict(metric="SD-2 text encoder, get_text_embeds shape (B = 2, 77 tokens)", card=card(), calls=args.calls,
               engine_workspace_mib=round(enc.workspace.numel() / 2 ** 20, 1), engine_footprint_mib=round(footprint / 2 ** 20, 1),
               gemm_gflop_per_call=round(flops / 1e9, 2))
    ms = time_calls(lambda: enc(ids), args.calls, args.warmup)
    res.update(engine_ms=round(ms, 4), engine_gemm_tflops=round(flops / ms / 1e9, 1), engine_graph_replays=enc.graph_replays())
    plain = st.TextEncoder("cuda", cfg=cfg, state_dict=sd, graph_replay=False)
    res["engine_plain_launches_ms"] = round(time_calls(lambda: plain(ids), args.calls, args.warmup), 4)
    del plain
    torch.backends.cuda.matmul.allow_tf32 = False
    ref_cu = ref.cuda()
    with torch.no_grad():
        ms32 = time_calls(lambda: ref_cu(ids), args.calls, args.warmup)
        res["oracle_fp32_eager_ms"] = round(ms32, 4)
        want = ref_cu(ids)[0]
    got = enc(ids)[0]
    res["engine_vs_fp32_rel_l2"] = float((got.double() - want.double()).norm() / want.double().norm())
    del ref_cu
    try:
        transformers = importlib.import_module("transformers")
    except ImportError:
        transformers = None
    if transformers is not None:
        hf = transformers.CLIPTextModel(transformers.CLIPTextConfig(
            vocab_size=cfg["vocab"], hidden_size=cfg["width"], intermediate_size=4 * cfg["width"], num_hidden_layers=cfg["layers"],
            num_attention_heads=cfg["heads"], max_position_embeddings=cfg["context_len"], hidden_act="gelu", layer_norm_eps=1e-5))
        hf.load_state_dict(sd, strict=False)
        hf = hf.cuda().eval()
        with torch.no_grad():
            res["transformers_fp32_ms"] = round(time_calls(lambda: hf(input_ids=ids), args.calls, args.warmup), 4)
    else:
        res["transformers_fp32_ms"] = "not importable"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
