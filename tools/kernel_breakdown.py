"""Per-kernel GPU time of the bench step IN PIPELINE CONTEXT (CUPTI activity records through torch.profiler: real timeline, kernels
of graph replays included, no serialisation / cache flush like ncu) -- the nsys substitute of this image.
    python tools/kernel_breakdown.py [--steps 4] [--defer-backward]        (1 GPU)
Prints per kernel name: launches / step, total us / step, mean us, share of the summed kernel time; then the GPU busy time per step
(union of kernel intervals) and the wall time per step, i.e. how much of the step the GPU sits idle between launches."""
import argparse
import collections
import importlib
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--defer-backward", action="store_true")
    a = ap.parse_args()
    device = torch.device("cuda", 0)
    model, guidance = bench.build_models(device, seed=0, defer_backward=a.defer_backward)
    utils = importlib.import_module("make-it-3d_b200.nerf.utils")
    opt = model.opt
    HW = bench.HW
    text_z = torch.randn(2, 77, 1024, generator=torch.Generator().manual_seed(0)).to(device)
    pose = torch.from_numpy(bench.orbit_pose(1.0, 90.0, 180.0))[None]
    import math
    focal = HW / (2 * math.tan(math.radians(20.0) / 2))
    cams = utils.camera_table(pose, (focal, focal, HW / 2, HW / 2), device)

    def step(s):
        model.zero_grad(set_to_none=True)
        out = model.render(None, None, cam_table=cams, cam_hw=(HW, HW), bg_color=torch.rand(3, device=device), staged=False, perturb=True,
                           ambient_ratio=1.0, shading='albedo', force_all_rays=True, **vars(opt))
        pred = out['image'].reshape(1, HW, HW, 3).permute(0, 3, 1, 2).contiguous()
        loss, _ = guidance.train_step(text_z, pred, islarge=True, guidance_scale=10, t=(250, 450, 600)[s % 3])
        loss = loss + bench.regulariser_loss(out, opt)
        loss.backward()
    for s in range(5):
        step(s)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        for s in range(a.steps):
            step(s)
        e1.record()
        torch.cuda.synchronize()
    wall = e0.elapsed_time(e1) / a.steps
    agg = collections.OrderedDict()
    ivals = []
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.replace("(anonymous namespace)::", "").replace("<unnamed>::", "").replace("void ", "")
        name = re.sub(r"\(.*$", "", name)
        d = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        r = agg.setdefault(name[:70], [0, 0.0])
        r[0] += 1; r[1] += d
        tr = ev.time_range
        ivals.append((tr.start, tr.end, name[:48]))
    ivals.sort()
    # idle gaps between consecutive kernels (where the host, not the GPU, paces the step)
    gaps, last_e, last_n = [], None, None
    for s_, e_, n_ in ivals:
        if last_e is not None and s_ > last_e:
            gaps.append((s_ - last_e, last_n, n_))
        if last_e is None or e_ > last_e:
            last_e, last_n = e_, n_
    ivals = [(s_, e_) for s_, e_, _ in ivals]
    busy, cur_s, cur_e = 0.0, None, None
    for s_, e_ in ivals:
        if cur_e is None or s_ > cur_e:
            if cur_e is not None:
                busy += cur_e - cur_s
            cur_s, cur_e = s_, e_
        else:
            cur_e = max(cur_e, e_)
    if cur_e is not None:
        busy += cur_e - cur_s
    tot = sum(v[1] for v in agg.values())
    print(f"# bench step (front view, M ~ 635 k samples), {a.steps} steps profiled with torch.profiler (CUPTI); sds backward: "
          f"{'deferred (one render backward)' if a.defer_backward else 'immediate (two render backwards)'}; SD lists: "
          f"{'graph replay' if guidance.engine.graph_replays() else 'plain launches'}")
    print(f"# wall {wall:.3f} ms/step | GPU busy (union of kernel intervals) {busy / a.steps / 1e3:.3f} ms/step | summed kernel time {tot / a.steps / 1e3:.3f} ms/step")
    print(f"{'kernel':70s} {'n/step':>7s} {'us/step':>9s} {'mean us':>8s} {'share':>6s}")
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:70s} {n / a.steps:7.1f} {us / a.steps:9.1f} {us / n:8.1f} {100 * us / tot:5.1f}%")
    gagg = collections.OrderedDict()
    for g_, a_, b_ in gaps:
        r = gagg.setdefault((a_, b_), [0, 0.0]); r[0] += 1; r[1] += g_
    print(f"# idle gaps: {sum(g for g, _, _ in gaps) / a.steps / 1e3:.3f} ms/step in {len(gaps) / a.steps:.0f} gaps/step; largest (after kernel -> before kernel):")
    for (a_, b_), (n, us) in sorted(gagg.items(), key=lambda kv: -kv[1][1])[:14]:
        print(f"#   {us / a.steps:8.1f} us/step  n/step {n / a.steps:5.1f}  {a_}  ->  {b_}")


if __name__ == "__main__":
    main()
