"""GPU: our CUDA operators and the CPU oracle against the UNMODIFIED reference kernels
(raymarching/src/raymarching.cu of junshutang/Make-It-3D, compiled by oracle/build_ref.py), whose outputs on these exact inputs
are stored in tests/golden/ref_kernels.npz by tests/golden/make_golden_ref_kernels.py.
This is what pins the oracle for rows R1-R4, R6 of SURVEY.md 8a: the reference itself, run on the GPU."""
import importlib

import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import camera_rays, max_abs, orm, sphere_bitfield

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    return load_golden("ref_kernels.npz")


@pytest.fixture(scope="module")
def rm():
    return importlib.import_module("make-it-3d_b200.raymarching")


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_near_far_morton_packbits_vs_reference_kernels(ref, rm):
    ro, rd, _ = camera_rays(64)
    aabb = np.array([-1, -1, -1, 1, 1, 1], np.float32)
    n_r, f_r = ref["nf64_near"], ref["nf64_far"]
    n, f = rm.near_far_from_aabb(_cu(ro), _cu(rd), _cu(aabb), 0.2)
    torch.cuda.synchronize()
    # the reference binary contracts a*b+c into FMA; ours is built with -fmad=false: allow 2 ulp
    assert max_abs(n.cpu(), n_r) < 1e-6 and max_abs(f.cpu(), f_r) < 1e-6
    n_o, f_o = orm.near_far_from_aabb(ro, rd, aabb, 0.2)
    assert max_abs(n_o, n_r) < 1e-6 and max_abs(f_o, f_r) < 1e-6
    rng = np.random.default_rng(0)
    coords = rng.integers(0, 128, size=(100000, 3), dtype=np.int32)
    sel = ref["morton_sel"]
    np.testing.assert_array_equal(orm.morton3D(coords)[sel], ref["morton_idx"])
    np.testing.assert_array_equal(rm.morton3D(_cu(coords)).cpu().numpy(), orm.morton3D(coords))
    grid = rng.random((1, 128 ** 3), dtype=np.float32)
    sel = ref["pack_sel"]
    bits_o = orm.packbits(grid.reshape(-1), 0.4)
    np.testing.assert_array_equal(bits_o[sel], ref["pack_bits"])
    np.testing.assert_array_equal(rm.packbits(_cu(grid), 0.4).cpu().numpy(), bits_o)


def test_march_train_vs_reference_kernel(ref, rm):
    """Per-ray comparison (the reference's sample ORDER is atomic-arrival, ours is ray-id): counts and positions."""
    ro, rd, _ = camera_rays(96)
    bits = sphere_bitfield(0.25)
    aabb = np.array([-1, -1, -1, 1, 1, 1], np.float32)
    nears, fars = orm.near_far_from_aabb(ro, rd, aabb, 0.2)
    N = ro.shape[0]
    noises = np.random.default_rng(4).random(N, dtype=np.float32)
    cnt_r = ref["march_counter"]
    x_o, _, dl_o, rays_o_, tot = orm.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, noises, 0.0, 512, align=-1)
    assert cnt_r[1] == N
    count_r = ref["march_count"]
    # FMA contraction in the reference binary can move a sample across a voxel face for a handful of rays
    same = int((count_r == rays_o_[:, 2]).sum())
    assert same >= 0.999 * N, same
    assert abs(int(cnt_r[0]) - tot) <= 0.001 * tot
    # positions of the stored rays' samples
    worst, pos = 0.0, 0
    for n in ref["march_rays_sel"]:
        c_r = int(count_r[n])
        off_o, c_o = int(rays_o_[n, 1]), int(rays_o_[n, 2])
        if c_r == c_o and c_r:
            worst = max(worst, float(np.abs(ref["march_xyz"][pos:pos + c_r] - x_o[off_o:off_o + c_o]).max()))
            assert np.array_equal(ref["march_delta0"][pos:pos + c_r], dl_o[off_o:off_o + c_o, 0])
        pos += c_r
    assert worst < 1e-5


def test_composite_vs_reference_kernel(ref, rm):
    ro, rd, _ = camera_rays(64)
    bits = sphere_bitfield(0.3)
    aabb = np.array([-1, -1, -1, 1, 1, 1], np.float32)
    nears, fars = orm.near_far_from_aabb(ro, rd, aabb, 0.2)
    N = ro.shape[0]
    rng = np.random.default_rng(8)
    x, d, dl, rays, tot = orm.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, rng.random(N, dtype=np.float32), 0.0, 512, align=128)
    m = x.shape[0]
    sig = (rng.random(m, dtype=np.float32) * 20).astype(np.float32); rgb = rng.random((m, 3), dtype=np.float32)
    ws_r, dep_r, img_r = ref["comp_ws"], ref["comp_depth"], ref["comp_image"]
    s_t, c_t = _cu(sig).requires_grad_(), _cu(rgb).requires_grad_()
    ws, dep, img = rm.composite_rays_train(s_t, c_t, _cu(dl), _cu(rays), 1e-4)
    torch.cuda.synchronize()
    assert max_abs(ws.detach().cpu(), ws_r) < 2e-6 and max_abs(img.detach().cpu(), img_r) < 2e-6
    assert max_abs(dep.detach().cpu(), dep_r) < 5e-6
    ws_o, dep_o, img_o = orm.composite_rays_train_forward(sig, rgb, dl, rays, 1e-4)
    assert max_abs(ws_o, ws_r) < 5e-6 and max_abs(img_o, img_r) < 5e-6       # pins the CPU oracle (expf vs __expf)
    gw, gi = rng.standard_normal(N).astype(np.float32), rng.standard_normal((N, 3)).astype(np.float32)
    ((ws * _cu(gw)).sum() + (img * _cu(gi)).sum()).backward()
    torch.cuda.synchronize()
    sel = ref["comp_grad_sel"]
    gs_r, gr_r = ref["comp_grad_sigma"], ref["comp_grad_rgb"]
    assert max_abs(c_t.grad.cpu().numpy()[sel], gr_r) < 2e-6
    assert max_abs(s_t.grad.cpu().numpy()[sel], gs_r) < 1e-5 * max(1.0, float(np.abs(gs_r).max()))
