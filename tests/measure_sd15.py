"""Time SD-1.5 guidance against SD-2.0 on the same card, in one run:

* `unet_sds` (add_noise -> U-Net on [uncond, cond] -> CFG -> SDS gradient) at 64x64 latents, batch 2, for SD-2.0 and SD-1.5 engines
  built from seeded state dicts, in alternating windows of >= --window seconds each (CUDA events; graph replay on, as in training);
* the fused attention per launch, from the engine's profile (mi3d_sd_profile_dump), grouped by shape, with the useful rate
  4 T Tk_valid d heads B / time (the two products over the valid keys only);
* SD-1.5's text encoder at get_text_embeds' shape (B = 2, 77 tokens) against transformers' CLIPTextModel (quick-GELU) in fp32.

Prints the card name and power limit, then one JSON line.

  python tests/measure_sd15.py [--rounds 5] [--window 1.0] [--text-calls 50]
"""
import argparse
import collections
import ctypes as C
import importlib
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sd15_ref  # noqa: E402
from oracle import sd_ref, sd_text_ref  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else torch.cuda.get_device_name()


def seeded_state(make_unet, seed):
    """the U-Net's diffusers state_dict with PyTorch's default initialisers (names and shapes from the oracle make_unet() builds)"""
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    with torch.device("meta"):
        names = {k: tuple(v.shape) for k, v in make_unet().state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    return {k: sdm._default_init(k, s, g) for k, s in names.items()}


class Sds:
    def __init__(self, name, guide, cross):
        self.name, self.g = name, guide
        gen = torch.Generator().manual_seed(1)
        self.lat = (torch.randn(1, 4, 64, 64, generator=gen) * 0.8).cuda()
        self.noise = torch.randn(1, 4, 64, 64, generator=gen).cuda()
        self.ctx = torch.randn(2, 77, cross, generator=gen).cuda()
        self.t = torch.tensor([437], dtype=torch.long, device="cuda")

    def __call__(self):
        return self.g.unet_sds(self.lat, self.noise, self.t, self.ctx, 10.0)

    def window(self, seconds, per_call_ms):
        n = max(3, math.ceil(seconds * 1e3 / per_call_ms))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            self()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n, n

    def attention_profile(self, L, calls=3):
        """per-launch attention times from the engine's event bracket: {(T, Tk_valid, d, B*heads): [ms, ...]}"""
        L.check(L.lib().mi3d_sd_profile(self.g.engine.h, C.c_int(1), None, None), "sd_profile")
        for _ in range(calls):
            self()
        torch.cuda.synchronize()
        ms, n = C.c_float(0), C.c_int(0)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "launches.txt")
            L.check(L.lib().mi3d_sd_profile_dump(self.g.engine.h, C.c_int(0), C.byref(ms), C.byref(n), path.encode()), "sd_profile_dump")
            lines = open(path).read().split("\n")
        out = collections.defaultdict(list)
        for line in lines:
            f = line.split()
            if len(f) == 9 and f[5] == "2":                       # conv = 2: the fused attention (M = T, N = Tk_valid, K = d)
                out[(int(f[0]), int(f[1]), int(f[2]), int(f[6]))].append(float(f[8]))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--text-calls", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_sd15.py needs a GPU")
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    st = importlib.import_module("make-it-3d_b200.nerf.sd_text")
    L = importlib.import_module("make-it-3d_b200._lib")
    res = dict(metric="SD-1.5 vs SD-2.0 guidance: unet_sds (64x64 latents, batch 2), fused attention per launch, SD-1.5 text encoder",
               card=card())
    print(f"card: {res['card']}", flush=True)
    torch.manual_seed(0)
    vae = sd_ref.AutoencoderKLEncoder(sd_ref.sd_vae_config()).state_dict()
    models = [Sds("sd20", sdm.StableDiffusion("cuda", sd_version="2.0", unet_state=seeded_state(lambda: sd_ref.UNet2DConditionModel(sd_ref.sd20_unet_config()), 2), vae_state=vae), 1024),
              Sds("sd15", sdm.StableDiffusion("cuda", sd_version="1.5", unet_state=seeded_state(sd15_ref.sd15_unet, 2), vae_state=vae), 768)]
    per_call = {}
    for m in models:                                               # warm-up: first calls, graph capture, then a rough per-call time
        for _ in range(5):
            m()
        torch.cuda.synchronize()
        per_call[m.name] = m.window(0.2, 50.0)[0]
    samples = {m.name: [] for m in models}
    for _ in range(args.rounds):
        for m in models:
            ms, n = m.window(args.window, per_call[m.name])
            samples[m.name].append(ms)
    for m in models:
        s = samples[m.name]
        res[f"{m.name}_unet_sds_ms"] = dict(median=round(statistics.median(s), 3), min=round(min(s), 3), max=round(max(s), 3), windows=len(s))
        res[f"{m.name}_graph_replays"] = m.g.engine.graph_replays()
    res["sd15_over_sd20"] = round(res["sd15_unet_sds_ms"]["median"] / res["sd20_unet_sds_ms"]["median"], 4)
    for m in models:
        prof = m.attention_profile(L)
        rows, total = [], 0.0
        for (T, Tk, d, bh), ts in sorted(prof.items(), key=lambda kv: (-kv[0][0], kv[0][1])):
            ms = statistics.median(ts)
            flop = 4.0 * T * Tk * d * bh
            rows.append(dict(T=T, Tk_valid=Tk, d=d, B_heads=bh, launches_per_call=len(ts) // 3, median_ms=round(ms, 4),
                             useful_tflops=round(flop / ms / 1e9, 1)))
            total += sum(ts) / 3
        res[f"{m.name}_attention"] = rows
        res[f"{m.name}_attention_ms_per_call"] = round(total, 3)
    del models
    torch.cuda.empty_cache()

    # SD-1.5 text encoder against transformers' CLIPTextModel (fp32, same card)
    cfg = sd15_ref.sd15_text_config()
    ref = sd_text_ref.default_init(sd15_ref.sd15_text_encoder(cfg), seed=5).eval()
    sd = ref.state_dict()
    ids = sd_text_ref.make_ids((2, 11), pad=49407, seed=7).cuda()
    enc = st.TextEncoder("cuda", cfg=st.sd15_text_cfg(), state_dict=sd)

    def time_calls(fn, calls, warmup=5):
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
    flops = sd_text_ref.gemm_flops(cfg, 2)
    ms = time_calls(lambda: enc(ids), args.text_calls)
    res.update(text_engine_ms=round(ms, 4), text_engine_gemm_tflops=round(flops / ms / 1e9, 1))
    transformers = importlib.import_module("transformers")
    torch.backends.cuda.matmul.allow_tf32 = False
    hf = transformers.CLIPTextModel(transformers.CLIPTextConfig(
        vocab_size=cfg["vocab"], hidden_size=cfg["width"], intermediate_size=4 * cfg["width"], num_hidden_layers=cfg["layers"],
        num_attention_heads=cfg["heads"], max_position_embeddings=cfg["context_len"], hidden_act="quick_gelu", layer_norm_eps=1e-5))
    hf.load_state_dict(sd, strict=False)
    hf = hf.cuda().eval()
    with torch.no_grad():
        res["text_transformers_fp32_ms"] = round(time_calls(lambda: hf(input_ids=ids), args.text_calls), 4)
        want = hf(input_ids=ids).last_hidden_state
    got = enc(ids)[0]
    res["text_engine_vs_transformers_fp32_rel_l2"] = float((got.double() - want.double()).norm() / want.double().norm())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
