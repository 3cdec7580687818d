"""H100 timing of the BLIP-2 captioner (csrc/blip2_engine.cu) at the blip2-opt-2.7b configuration with seeded weights:
generate end to end (20 tokens), encode alone, one decode step, and the weight-streaming GEMM's GB/s beside the 3.35 TB/s of the H100
SXM data sheet; A/B arms on the same card: transformers' Blip2ForConditionalGeneration in fp16 (as main.py runs it) and the fp32 oracle.
Prints one JSON line.  Run: python tests/measure_blip2.py"""
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import blip2_ref  # noqa: E402

PEAK = 3.35e12


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    b2 = importlib.import_module("make-it-3d_b200.nerf.blip2")
    L = importlib.import_module("make-it-3d_b200._lib")
    lib = L.lib()
    lib.mi3d_stream_gemm_workspace_bytes.restype = C.c_size_t
    res = {"gpu": gpu}
    # the streaming GEMM alone
    for M, N, K in ((64, 10240, 2560), (64, 2560, 10240), (64, 7680, 2560), (1, 50272, 2560)):
        x = torch.randn(M, K, device="cuda").half(); w = torch.randn(N, K, device="cuda").half(); y = torch.empty(M, N, device="cuda").half()
        ws = torch.empty(lib.mi3d_stream_gemm_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
        f = lambda: lib.mi3d_stream_gemm_f16(L.ptr(x), L.ptr(w), None, None, 0, L.ptr(y), M, N, K, L.ptr(ws), C.c_size_t(ws.numel()), L.stream())
        ms = timed(f, reps=50, warm=10)
        gbs = N * K * 2 / (ms * 1e-3) / 1e9
        res[f"stream_gemm_{M}x{N}x{K}"] = {"ms": round(ms, 4), "GB/s": round(gbs, 1), "frac_of_3.35TB/s": round(gbs * 1e9 / PEAK, 3)}
    cfg = blip2_ref.blip2_opt_27b_cfg()
    p = blip2_ref.default_init(cfg, seed=0, device="cuda")
    model = b2.Blip2ForConditionalGeneration(cfg=cfg, state_dict=p)
    res["workspace_MiB"] = round(model.workspace_bytes / 2 ** 20)
    px = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
    res["engine_generate_20_ms"] = round(timed(lambda: model.generate(pixel_values=px, max_new_tokens=20, eos_token_id=-1)), 2)
    res["engine_generate_1_ms"] = round(timed(lambda: model.generate(pixel_values=px, max_new_tokens=1, eos_token_id=-1)), 2)
    res["engine_encode_ms"] = round(timed(lambda: model.encode(px)), 2)
    res["engine_decode_step_ms"] = round((res["engine_generate_20_ms"] - res["engine_generate_1_ms"]) / 19, 3)
    res["engine_decode_step_GB/s"] = round(2 * (blip2_ref_opt_params(cfg)) / (res["engine_decode_step_ms"] * 1e-3) / 1e9, 1)
    eng = model.generate(pixel_values=px, max_new_tokens=20, eos_token_id=-1)[0, 33:].tolist()
    with torch.no_grad():
        ref = blip2_ref.generate(p, cfg, px, 20, eos_token_id=-1)
        res["oracle_fp32_generate_20_ms"] = round(timed(lambda: blip2_ref.generate(p, cfg, px, 20, eos_token_id=-1), reps=1, warm=0), 1)
    orc = ref["ids"][33:]
    del model
    torch.cuda.empty_cache()
    try:
        import test_blip2_oracle_cpu as cpu_test  # noqa: PLC0415
        from transformers import Blip2ForConditionalGeneration
        with torch.device("meta"):
            hf = Blip2ForConditionalGeneration(cpu_test._hf_config(cfg))
        sd = {k: v.half() for k, v in p.items()}
        sd["language_model.lm_head.weight"] = sd["language_model.model.decoder.embed_tokens.weight"]
        hf.load_state_dict(sd, assign=True, strict=True)
        hf = hf.cuda().eval()
        hf.generation_config.eos_token_id = None
        hf.generation_config.max_new_tokens = 20
        run = lambda: hf.generate(pixel_values=px.half(), max_new_tokens=20, min_new_tokens=20)
        with torch.no_grad():
            res["transformers_fp16_generate_20_ms"] = round(timed(run, reps=3, warm=1), 1)
            hfi = run()[0, 33:].tolist()
        res["transformers_fp16_agrees_with_engine"] = sum(a == b for a, b in zip(hfi, eng))
        res["transformers_fp16_agrees_with_oracle"] = sum(a == b for a, b in zip(hfi, orc))
    except Exception as e:  # noqa: BLE001
        res["transformers_fp16"] = f"not run: {type(e).__name__}: {e}"[:300]
    res["engine_agrees_with_oracle"] = sum(a == b for a, b in zip(eng, orc))
    print(json.dumps(res))


def blip2_ref_opt_params(cfg):
    C_, F_, L_ = cfg["opt_width"], cfg["opt_ffn"], cfg["opt_layers"]
    return L_ * (4 * C_ * C_ + 2 * C_ * F_) + cfg["vocab"] * C_


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    main()
