"""The reference's OWN ray-march / composite kernels (raymarching/src/raymarching.cu compiled for sm_90a into oracle/_ref/, driven
exactly like raymarching/raymarching.py:173-303 drives them: 268 MB zero-fill, .item() host sync, zeros_like for the gradients)
timed beside the mi3d kernels on the bench's rays (128x128, sphere r = 0.2, front view: M ~ 635 k samples).  CUDA events, median
of 20, legacy default stream for the reference (its launches use <<<g,b>>> with no stream).  TEST/MEASUREMENT TOOL, not product.
It needs oracle/_ref/, which build() only makes when MI3D_REFERENCE_DIR names a checkout of Make-It-3D:
    MI3D_REFERENCE_DIR=<checkout> python -c "import __graft_entry__ as g; g.build()"
    python tests/measure_ref_kernels.py       (GPU machine)"""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def med_ms(fn, n=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def main():
    from oracle import build_ref
    import bench
    ref = build_ref.load_ref()
    if ref is None:
        print("oracle/_ref/_raymarching_ref.so missing"); return 1
    L = importlib.import_module("make-it-3d_b200._lib")
    U = importlib.import_module("make-it-3d_b200.nerf.utils")
    lib = L.lib()
    HW, max_steps = 128, 512
    N, M = HW * HW, HW * HW * max_steps
    pose = torch.from_numpy(bench.orbit_pose(1.0, 90.0, 180.0))[None].cuda()
    focal = HW / (2 * np.tan(np.radians(20.0) / 2))
    r = U.get_rays(pose, (focal, focal, HW / 2, HW / 2), HW, HW, -1)
    rays_o, rays_d = r["rays_o"][0].contiguous(), r["rays_d"][0].contiguous()
    bits = torch.from_numpy(bench.sphere_bitfield_numpy(0.2)).cuda()
    aabb = torch.tensor([-1, -1, -1, 1, 1, 1], dtype=torch.float32, device="cuda")
    noises = torch.rand(N, device="cuda")
    # ---------------- reference, as its wrapper drives it (raymarching.py:31-61, 173-303) ----------------
    st = {}

    def ref_near_far():
        st["nears"], st["fars"] = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
        ref.near_far_from_aabb(rays_o, rays_d, aabb, N, 0.2, st["nears"], st["fars"])

    def ref_march():
        xyzs = torch.zeros(M, 3, device="cuda"); dirs = torch.zeros(M, 3, device="cuda"); deltas = torch.zeros(M, 2, device="cuda")   # :217-219
        rays = torch.empty(N, 3, dtype=torch.int32, device="cuda")
        counter = torch.zeros(2, dtype=torch.int32, device="cuda")
        ref.march_rays_train(rays_o, rays_d, bits, 1.0, 0.0, max_steps, N, 1, 128, M, st["nears"], st["fars"], xyzs, dirs, deltas, rays, counter, noises)
        m = int(counter[0].item())                                                                                                     # :236 host sync
        m += 128 - m % 128
        st.update(xyzs=xyzs[:m], dirs=dirs[:m], deltas=deltas[:m], rays=rays, m=m)
    ref_near_far(); ref_march()
    m = st["m"]
    sig = torch.rand(m, device="cuda") * 20
    rgb = torch.rand(m, 3, device="cuda")

    def ref_comp_fwd():
        st["ws"], st["dep"], st["img"] = torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, 3, device="cuda")
        ref.composite_rays_train_forward(sig, rgb, st["deltas"], st["rays"], m, N, 1e-4, st["ws"], st["dep"], st["img"])
    ref_comp_fwd()
    gw, gi = torch.randn(N, device="cuda"), torch.randn(N, 3, device="cuda")

    def ref_comp_bwd():
        gs, gr = torch.zeros_like(sig), torch.zeros_like(rgb)                                                                        # :295-296
        ref.composite_rays_train_backward(gw, gi, sig, rgb, st["deltas"], st["rays"], st["ws"], st["img"], m, N, 1e-4, gs, gr)
    t_ref = dict(near_far=med_ms(ref_near_far), march=med_ms(ref_march), comp_fwd=med_ms(ref_comp_fwd), comp_bwd=med_ms(ref_comp_bwd))
    # ---------------- mi3d kernels (capacity-sized buffers allocated once, device-side count, fused near/far) ----------------
    cap = M + 128
    xyzs, dirs, deltas = torch.empty(cap, 3, device="cuda"), torch.empty(cap, 3, device="cuda"), torch.empty(cap, 2, device="cuda")
    rays = torch.empty(N, 3, dtype=torch.int32, device="cuda"); counter = torch.zeros(2, dtype=torch.int32, device="cuda")
    nears, fars = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
    ws_b = torch.empty(lib.mi3d_march_rays_train_workspace_bytes(C.c_uint32(N)), dtype=torch.uint8, device="cuda")

    def our_march():
        counter.zero_()
        L.check(lib.mi3d_march_rays_train(L.ptr(rays_o), L.ptr(rays_d), L.ptr(bits), C.c_float(1.0), C.c_float(0.0), C.c_uint32(max_steps), C.c_uint32(N),
                                          C.c_uint32(1), C.c_uint32(128), C.c_uint32(M), C.c_void_p(0), C.c_void_p(0), L.ptr(aabb), C.c_float(0.2), L.ptr(nears),
                                          L.ptr(fars), L.ptr(noises), C.c_uint64(0), L.ptr(xyzs), L.ptr(dirs), L.ptr(deltas), L.ptr(rays), L.ptr(counter),
                                          L.ptr(ws_b), L.stream()), "march")
    our_march()
    torch.cuda.synchronize()
    m2 = int(counter[0])
    sig2, rgb2 = torch.rand(cap, device="cuda") * 20, torch.rand(cap, 3, device="cuda")
    ws_o, dep_o, img_o = torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, 3, device="cuda")
    gs2, gr2 = torch.empty(cap, device="cuda"), torch.empty(cap, 3, device="cuda")

    def our_comp_fwd():
        L.check(lib.mi3d_composite_rays_train_forward(L.ptr(sig2), L.ptr(rgb2), L.ptr(deltas), L.ptr(rays), C.c_uint32(M), C.c_uint32(N), C.c_float(1e-4),
                                                      L.ptr(ws_o), L.ptr(dep_o), L.ptr(img_o), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), L.stream()), "cf")

    def our_comp_bwd():
        L.check(lib.mi3d_composite_rays_train_backward(L.ptr(gw), L.ptr(gi), C.c_void_p(0), L.ptr(sig2), L.ptr(rgb2), L.ptr(deltas), L.ptr(rays), L.ptr(ws_o),
                                                       L.ptr(img_o), C.c_uint32(M), C.c_uint32(N), C.c_float(1e-4), C.c_void_p(0), L.ptr(gs2), L.ptr(gr2), C.c_int(1),
                                                       L.stream()), "cb")
    our_comp_fwd()
    t_our = dict(march=med_ms(our_march), comp_fwd=med_ms(our_comp_fwd), comp_bwd=med_ms(our_comp_bwd))
    print(f"# 128x128 rays, sphere r=0.2 occupancy, front view; samples: reference {m} (padded), mi3d {m2}; CUDA events, median of 20, us")
    print(f"{'stage':44s} {'reference (raymarching.cu via its wrapper)':>44s} {'mi3d':>10s} {'ratio':>7s}")
    rows = [("near/far + march_rays_train (+zero-fill, .item())", (t_ref["near_far"] + t_ref["march"]) * 1e3, t_our["march"] * 1e3),
            ("composite_rays_train forward", t_ref["comp_fwd"] * 1e3, t_our["comp_fwd"] * 1e3),
            ("composite_rays_train backward (+zeros_like x2)", t_ref["comp_bwd"] * 1e3, t_our["comp_bwd"] * 1e3)]
    for name, a, b in rows:
        print(f"{name:44s} {a:44.1f} {b:10.1f} {a / b:7.2f}x")
    print(f"(reference near_far alone {t_ref['near_far'] * 1e3:.1f} us, march alone incl. 268 MB zero-fill + host sync {t_ref['march'] * 1e3:.1f} us)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
