"""Per-role cycle breakdown of the field backward chain kernel (k_field_bwd_tc) on bench.py's scene (128x128, k = 13).

Builds field.cu with -DMI3D_FIELD_BWD_CLOCKS into a separate libmi3d.so under --out (the other objects come from the in-tree
build), loads it through MI3D_LIB_PATH and runs bench.py's step.  The SDS backward inside guidance.train_step is the image pass
(1 evaluation per sample); loss.backward() is the full pass (13).  For each it prints, per warp of each role and per evaluation:
  owners  : cycles in total and waiting on stg_full (the MMA warpgroup's next staged accumulator)
  MMA     : cycles in total and waiting on a1..a4_full (encodings / owner epilogues)
  encoders: cycles in total, waiting on d4_full (the chain's dEnc) and scattering dEnc into the table gradient
The instrumented kernel spills more than the shipped one, so its cycle counts are a breakdown, not a timing.
Usage (GPU): python tools/prof_field_bwd.py [--steps 4] [--out build/prof_field_bwd]"""
import argparse
import ctypes
import glob
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "make-it-3d_b200", "csrc")
SLOTS = ["owner_total", "owner_wait_stg", "mma_total", "mma_wait_a", "enc_total", "enc_wait_d4", "enc_scatter", "evals"]
WARPS = {"owner": 4, "mma": 4, "enc": 8}


def build(out):
    os.makedirs(out, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    obj = os.path.join(out, "field_clocks.o")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-lineinfo", *arch, "-Xcompiler", "-fPIC", "-DMI3D_FIELD_BWD_CLOCKS", "-c",
                    os.path.join(CSRC, "field.cu"), "-o", obj], check=True)
    others = [o for o in sorted(glob.glob(os.path.join(CSRC, "*.o"))) if os.path.basename(o) != "field.o"]
    if not others:
        raise SystemExit("no objects under make-it-3d_b200/csrc: build the library first")
    so = os.path.join(out, "libmi3d.so")
    subprocess.run([nvcc, *arch, "-shared", "-o", so, obj, *others, "-lcudart_static"], check=True)
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4, help="bench steps after one warm-up step")
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "prof_field_bwd"))
    args = ap.parse_args()
    so = build(args.out)
    os.environ["MI3D_LIB_PATH"] = so
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench

    lib = ctypes.CDLL(so)
    lib.mi3d_field_bwd_clocks.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
    buf = (ctypes.c_ulonglong * 8)()

    def read():
        rc = lib.mi3d_field_bwd_clocks(buf)
        if rc != 0:
            raise RuntimeError(f"mi3d_field_bwd_clocks: {rc}")
        return dict(zip(SLOTS, list(buf)))

    device = torch.device("cuda", 0)
    model, guidance = bench.build_models(device, seed=0)
    opt = model.opt
    HW = bench.HW
    text_z = torch.randn(2, 77, 1024, generator=torch.Generator().manual_seed(0)).to(device)
    rng = np.random.default_rng(0)
    gen = torch.Generator(device=device).manual_seed(4242)
    t_cycle = (250, 450, 600)
    sums = {"image": dict.fromkeys(SLOTS, 0), "full": dict.fromkeys(SLOTS, 0)}
    for s in range(args.steps + 1):
        pose, fov = bench.synth_pose(s, rng)
        focal = HW / (2 * math.tan(math.radians(fov) / 2))
        cams = torch.from_numpy(np.concatenate([pose[:3].reshape(-1), np.array([focal, focal, HW / 2, HW / 2], np.float32)])
                                .astype(np.float32)[None]).to(device)
        model.zero_grad(set_to_none=True)
        bg = torch.rand(3, device=device, generator=gen)
        kw = dict(bg_color=bg, staged=False, perturb=True, ambient_ratio=1.0, shading='albedo', force_all_rays=True, **vars(opt))
        out = model.render(None, None, cam_table=cams, cam_hw=(HW, HW), **kw)
        read()
        pred = out['image'].reshape(1, HW, HW, 3).permute(0, 3, 1, 2).contiguous()
        loss, _ = guidance.train_step(text_z, pred, islarge=True, guidance_scale=10, t=t_cycle[s % 3])
        img = read()
        (loss + bench.regulariser_loss(out, opt)).backward()
        full = read()
        if s > 0:
            for k in SLOTS:
                sums["image"][k] += img[k]; sums["full"][k] += full[k]
    props = torch.cuda.get_device_properties(0)
    report = {"gpu": props.name, "sms": props.multi_processor_count, "steps": args.steps, "passes": {}}
    for name, c in sums.items():
        ev = max(c["evals"], 1)
        per = lambda slot, role: round(c[slot] / WARPS[role] / ev)
        report["passes"][name] = {
            "evaluations_per_step": c["evals"] // max(args.steps, 1),
            "cycles_per_eval": {
                "owner": {"total": per("owner_total", "owner"), "wait_stg_full": per("owner_wait_stg", "owner")},
                "mma": {"total": per("mma_total", "mma"), "wait_a_full": per("mma_wait_a", "mma")},
                "encoder": {"total": per("enc_total", "enc"), "wait_d4_full": per("enc_wait_d4", "enc"),
                            "scatter": per("enc_scatter", "enc")},
            }}
    line = json.dumps(report)
    print(line)
    with open(os.path.join(args.out, "prof_field_bwd.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
