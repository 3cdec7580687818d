"""Times the per-step CLIP losses on the GPU (python tests/measure_clip.py [--out FILE]).

Legs, all at the Trainer's shapes (two 512x512 images, one 77-token prompt, ViT-B/16 with seeded weights), after warm-up, graph replay on:
  losses_fwd_bwd   CLIP.losses(pred_rgb, gt_rgb, tokens) + backward into pred_rgb  (nerf/utils.py:561-563)
  losses_no_grad   the same under torch.no_grad()                                  (the SD denoise branch, nerf/sd.py:157-158)
  reference_fp16   the A/B arm: oracle/clip_ref.py converted to fp16 on the GPU in eager PyTorch, called the way the reference
                   calls openai CLIP (aug in torch, encode_image twice, encode_text once, fp16 model as clip.load makes it)
Reported per leg: ms per call (CUDA events over the timed calls), kernels per call (torch.profiler, one separate call), algorithmic
FLOPs per call from the shapes and the achieved TFLOP/s; plus the card name and power limit read in the same run.  Lives under tests/
because it imports the oracle."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import clip_ref  # noqa: E402


def tower_flops(T, C, layers, backward=False):
    """2*M*N*K of the GEMMs and attention products of `layers` blocks on T tokens; backward = input-gradient products only"""
    lin = 2 * T * C * (3 * C + C + 4 * C + 4 * C)
    att = 2 * 2 * T * T * C
    return layers * (lin + (2 * att if backward else att))


def flops(cfg, n_img_fwd, n_img_bwd, n_txt):
    c = cfg
    np_ = (c["image_res"] // c["patch"]) ** 2
    T, C, P = np_ + 1, c["width"], 3 * c["patch"] ** 2
    img_f = 2 * np_ * P * C + tower_flops(T, C, c["layers"]) + 2 * C * c["embed_dim"]
    img_b = 2 * np_ * P * C + tower_flops(T, C, c["layers"], True) + 2 * C * c["embed_dim"]
    txt = tower_flops(c["context_len"], c["text_width"], c["text_layers"]) + 2 * c["text_width"] * c["embed_dim"]
    return n_img_fwd * img_f + n_img_bwd * img_b + n_txt * txt


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernels_per_call(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
               and "memset" not in e.name.lower())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "measure_clip.py needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    card = q.strip().splitlines()[0] if q.strip() else "unknown"
    clipm = importlib.import_module("make-it-3d_b200.nerf.clip")
    cfg = clip_ref.vit_b16_config()
    torch.manual_seed(0)
    ref = clip_ref.default_init(clip_ref.CLIPRef(cfg), seed=0).eval()
    model = clipm.CLIP("cuda", cfg=cfg, state_dict=ref.state_dict())
    g = torch.Generator().manual_seed(0)
    pred = torch.rand(1, 3, 512, 512, generator=g).cuda().requires_grad_()
    gt = torch.rand(1, 3, 512, 512, generator=g).cuda()
    tok = clip_ref.make_tokens([12], seed=0).cuda()

    def native():
        a, b = model.losses(pred, gt, tok)
        (a + b).backward()

    def native_no_grad():
        with torch.no_grad():
            model.losses(pred, gt, tok)

    half = ref.half().cuda()
    for p in half.parameters():
        p.requires_grad_(False)
    enc = lambda x: half.encode_image(x.half()).float()

    class _Ref:
        encode_image = staticmethod(enc)
        encode_text = staticmethod(lambda t: half.encode_text(t).float())

    def reference():
        loss = clip_ref.img_clip_loss(_Ref, pred, gt) + clip_ref.img_text_clip_loss(_Ref, pred, tok)
        loss.backward()

    rows = []
    for name, fn, fl in (("losses_fwd_bwd", native, flops(cfg, 2, 1, 1)), ("losses_no_grad", native_no_grad, flops(cfg, 2, 0, 1)),
                         ("reference_fp16", reference, flops(cfg, 3, 2, 1))):
        ms = timed(fn, args.warmup, args.iters)
        k = kernels_per_call(fn)
        rows.append(dict(leg=name, ms_per_call=round(ms, 3), kernels_per_call=k, gflop_per_call=round(fl / 1e9, 1),
                         achieved_tflops=round(fl / (ms * 1e-3) / 1e12, 1)))
    out = dict(card=card, model="ViT-B/16 (seeded weights)", shapes="2 x 512^2 images, 1 x 77 tokens", warmup=args.warmup, iters=args.iters,
               graph_replay=True, legs=rows, speedup_fwd_bwd_vs_reference=round(rows[2]["ms_per_call"] / rows[0]["ms_per_call"], 2))
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
