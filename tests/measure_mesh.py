"""H100 timing of the mesh export (csrc/mesh.cu, nerf/mesh.py) at resolution 256 on a seeded field shaped like an object (the
reference's density blob widened to radius 0.5, hash-grid noise on top): device-event times of the volume query, the marching-cubes
count and emit passes, the atlas texel pass, the albedo query and the file write; the marching-cubes kernels' algorithmic bytes over
their time beside the 3.35 TB/s of the H100 SXM data sheet; the card's name and power limit.  Prints one JSON line.
Run: python tests/measure_mesh.py [--resolution 256]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import make_table  # noqa: E402

PEAK = 3.35e12


def events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    out = None
    for _ in range(reps):
        torch.cuda.synchronize()
        a.record(); out = fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    mesh = importlib.import_module("make-it-3d_b200.nerf.mesh")
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    opt = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.5, lambda_smooth=1,
                             max_depth=10.0)
    torch.manual_seed(0)
    net = nt.NeRFNetwork(opt)
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(make_table(net.encoder.params.numel(), 3, 0.1)))
    net = net.cuda().eval()
    net.mean_density = torch.full((1,), 40.0, device="cuda")          # threshold min(40, 10) = 10, read on the device
    res, reps = args.resolution, args.reps
    out = {"gpu": gpu, "resolution": res}
    iso, iso_dev = mesh.density_threshold(net)
    for _ in range(2):                                                   # warm-up of every shape
        vol = mesh.density_volume(net, res)
        v, f = mesh.extract_mesh(net, res)
        mesh.bake_texture(net, v, f)
    t_vol, vol = events(lambda: mesh.density_volume(net, res), reps)
    t_count, (ws, counts) = events(lambda: mesh.mc_count(vol, iso, iso_dev), reps)
    V, F = counts.cpu().tolist()
    t_emit, (v, f) = events(lambda: mesh.mc_emit(vol, iso, ws, V, F, iso_dev, 2.0 / (res - 1.0), -1.0), reps)
    T, c, n = mesh.atlas_layout(F)
    t_bake, baked = events(lambda: mesh.bake_texture(net, v, f), reps)
    # the atlas texel kernel alone
    import ctypes as C
    L = importlib.import_module("make-it-3d_b200._lib")
    pts = torch.empty(T * T, 3, device="cuda"); own = torch.empty(T * T, dtype=torch.int32, device="cuda")
    vt = torch.empty(3 * F, 2, device="cuda")
    t_atlas, _ = events(lambda: L.check(L.lib().mi3d_mesh_atlas_texels(L.ptr(v), L.ptr(f), C.c_uint32(F), C.c_uint32(T), C.c_uint32(c),
                                                                      C.c_uint32(n), C.c_float(1.0), L.ptr(pts), L.ptr(own), L.ptr(vt),
                                                                      L.stream()), "atlas"), reps)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        mesh.write_files(d, v, f, *baked[:3])
        t_write = (time.perf_counter() - t0) * 1e3
        sizes = {k: os.path.getsize(os.path.join(d, k)) for k in os.listdir(d)}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        net.export_mesh(d, resolution=res)
        torch.cuda.synchronize()
        t_total = (time.perf_counter() - t0) * 1e3
    N = res ** 3
    count_bytes = 4 * N + 10 * N                     # volume read; vertex offset, face offset, code written
    emit_bytes = 10 * N + 8 * V + 12 * V + 12 * F    # offsets and codes read, two samples per vertex, vertices and faces written
    out.update({"V": V, "F": F, "atlas_T": T, "atlas_cell": c,
                "volume_query_ms": round(t_vol, 3), "mc_count_ms": round(t_count, 3), "mc_emit_ms": round(t_emit, 3),
                "mc_count_TB/s": round(count_bytes / (t_count * 1e-3) / 1e12, 3), "mc_emit_TB/s": round(emit_bytes / (t_emit * 1e-3) / 1e12, 3),
                "mc_count_frac_of_3.35TB/s": round(count_bytes / (t_count * 1e-3) / PEAK, 3),
                "mc_emit_frac_of_3.35TB/s": round(emit_bytes / (t_emit * 1e-3) / PEAK, 3),
                "atlas_texels_ms": round(t_atlas, 3), "atlas_and_albedo_ms": round(t_bake, 3), "file_write_ms": round(t_write, 1),
                "file_bytes": sizes, "export_mesh_total_ms": round(t_total, 1)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
