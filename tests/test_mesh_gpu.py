"""GPU: mesh export (csrc/mesh.cu, nerf/mesh.py) against oracle/mesh_ref.py and oracle/field_ref.py."""
import argparse
import filecmp
import importlib
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import field_from_golden, make_table, max_abs, rel_err
from oracle import mesh_ref as M

pytestmark = pytest.mark.gpu

mesh = importlib.import_module("make-it-3d_b200.nerf.mesh")
Mi3dError = importlib.import_module("make-it-3d_b200").Mi3dError

REF_MTL = ("newmtl mat0 \nKa 1.000000 1.000000 1.000000 \nKd 1.000000 1.000000 1.000000 \nKs 0.000000 0.000000 0.000000 \n"
           "Tr 1.000000 \nillum 1 \nNs 0.000000 \nmap_Kd albedo.png \n")


def _sphere(shape, r=0.5):
    axes = [np.linspace(-1, 1, n).astype(np.float32) for n in shape]
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    return (r - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32)


def _random(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


def _net():
    g = load_golden("render_albedo.npz")
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    opt = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1,
                             lambda_smooth=1, max_depth=10.0)
    net = nt.NeRFNetwork(opt)
    table = make_table(net.encoder.params.numel(), int(g["table_seed"]), float(g["table_scale"]))
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(table))
        for l, (w, b) in enumerate((("w1", "b1"), ("w2", "b2"), ("w3", "b3"))):
            net.sigma_net.net[l].weight.copy_(torch.from_numpy(g[w]))
            net.sigma_net.net[l].bias.copy_(torch.from_numpy(g[b]))
    field, _ = field_from_golden(g)
    return net.cuda().eval(), field


def _net_with_surface(resolution=40):
    """the golden field, with a device mean_density at the volume's median so the surface cuts through it"""
    net, field = _net()
    vol = mesh.density_volume(net, resolution, 128)
    net.mean_density = vol.flatten().median().reshape(1).clone()
    return net, field


def _check_against_oracle(vol_np, iso):
    v, f = mesh.marching_cubes(vol_np, iso)
    vr, fr_ = M.marching_cubes(vol_np, iso)
    assert v.dtype == np.float64 and f.dtype == np.int64
    assert len(fr_) > 0 and np.array_equal(f, fr_)
    assert np.array_equal(v.astype(np.float32), vr) and np.array_equal(v, vr.astype(np.float64))
    vt, ft = mesh.marching_cubes(torch.from_numpy(vol_np).cuda(), iso)
    assert vt.dtype == torch.float32 and ft.dtype == torch.int32 and vt.is_cuda
    assert np.array_equal(vt.cpu().numpy(), vr) and np.array_equal(ft.cpu().numpy(), fr_)
    return vr, fr_


@pytest.mark.parametrize("shape", [(64, 64, 64), (41, 53, 29)])
def test_marching_cubes_sphere_matches_oracle(shape):
    v, f = _check_against_oracle(_sphere(shape), 0.0)
    assert M.is_closed_oriented(f) and M.euler_characteristic(v, f) == 2 and M.signed_volume(v, f) > 0


@pytest.mark.parametrize("shape,seed", [((48, 48, 48), 0), ((37, 23, 51), 1), ((2, 2, 2), 2), ((300, 17, 9), 3)])
def test_marching_cubes_random_matches_oracle(shape, seed):
    vol = _random(shape, seed)
    if shape == (2, 2, 2):
        vol = np.array([[[1, -1], [-1, -1]], [[-1, -1], [-1, 1]]], np.float32)
    _check_against_oracle(vol, 0.1)


def test_marching_cubes_field_volume_matches_oracle():
    net, _ = _net()
    vol = mesh.density_volume(net, 56, 32)
    iso = float(vol.flatten().median())
    _check_against_oracle(vol.cpu().numpy(), iso)


def test_device_threshold_equals_float_and_adds_no_sync():
    vol = torch.from_numpy(_random((40, 33, 45), 7)).cuda()
    v0, f0 = mesh.marching_cubes(vol, 0.3)
    for iso, dev in ((10.0, 0.3), (0.3, 5.0)):          # min(iso, *iso_dev) = 0.3 either way
        iso_dev = torch.tensor([dev], dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ws, counts = mesh.mc_count(vol, iso, iso_dev)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        V, F = counts.cpu().tolist()
        torch.cuda.set_sync_debug_mode("error")
        try:
            v, f = mesh.mc_emit(vol, iso, ws, V, F, iso_dev)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.equal(v, v0) and torch.equal(f, f0)


def test_volume_equals_reference_density_loop():
    """renderer.py:167-180 run literally over model.density(): identical bits; and within the field tolerance of the oracle"""
    net, field = _net()
    res, S = 45, 16
    vol = mesh.density_volume(net, res, S)
    X = torch.linspace(-1, 1, res).split(S)
    ref = np.zeros([res] * 3, np.float32)
    for xi, xs in enumerate(X):
        for yi, ys in enumerate(X):
            for zi, zs in enumerate(X):
                xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
                pts = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
                val = net.density(pts.to(net.aabb_train.device))
                ref[xi * S: xi * S + len(xs), yi * S: yi * S + len(ys), zi * S: zi * S + len(zs)] = \
                    val['sigma'].reshape(len(xs), len(ys), len(zs)).detach().cpu().numpy()
    assert np.array_equal(vol.cpu().numpy(), ref)
    lin = torch.linspace(-1, 1, res)
    idx = np.random.default_rng(0).integers(0, res, (4000, 3))
    pts = torch.stack([lin[idx[:, 0]], lin[idx[:, 1]], lin[idx[:, 2]]], -1)
    with torch.no_grad():
        sr = field.density(pts)["sigma"].numpy()
    assert rel_err(ref[idx[:, 0], idx[:, 1], idx[:, 2]], sr, floor=1e-3) < 2e-5


def test_extract_mesh_scaling_and_threshold():
    net, _ = _net_with_surface(40)
    v, f = mesh.extract_mesh(net, 40, 128)
    vol = mesh.density_volume(net, 40, 128).cpu().numpy()
    iso = float(net.mean_density.cpu())
    vr, fr_ = M.marching_cubes(vol, iso, scale=np.float32(2.0 / 39.0), offset=-1.0)
    assert np.array_equal(f.cpu().numpy(), fr_) and np.array_equal(v.cpu().numpy(), vr)
    assert float(v.abs().max()) <= 1.0


def test_bake_texture_matches_oracle():
    net, field = _net_with_surface(32)
    v, f = mesh.extract_mesh(net, 32, 128)
    F = f.shape[0]
    vt, ft, albedo, owner = mesh.bake_texture(net, v, f)
    T, c, n = mesh.atlas_layout(F)
    assert (T, c, n) == M.atlas_layout(F) and albedo.shape == (T, T, 3) and owner.shape == (T, T)
    pts_r, own_r, vt_r = M.atlas_texels(v.cpu().numpy(), f.cpu().numpy(), T, c, n, 1.0)
    assert np.array_equal(owner.cpu().numpy(), own_r)
    assert np.array_equal(vt.cpu().numpy(), vt_r)
    assert np.array_equal(ft.cpu().numpy(), np.arange(3 * F).reshape(F, 3))
    alb = albedo.cpu().numpy()
    assert (alb[own_r < 0] == 0).all()
    r, x = np.nonzero(own_r >= 0)
    sub = np.random.default_rng(1).choice(len(r), 20000, replace=False)
    with torch.no_grad():
        ref = field.density(torch.from_numpy(pts_r[r[sub], x[sub]]))["albedo"].numpy()
    assert max_abs(alb[r[sub], x[sub]], ref) < 2e-5


def _parse_obj(p):
    v, vt, f, ft = [], [], [], []
    with open(p) as fp:
        lines = fp.read().splitlines()
    assert lines[0] == "mtllib mesh.mtl "
    for ln in lines[1:]:
        tok = ln.split()
        if tok[0] == "v":
            v.append([np.float32(t) for t in tok[1:4]])
        elif tok[0] == "vt":
            vt.append([np.float32(t) for t in tok[1:3]])
        elif tok[0] == "f":
            pairs = [t.split("/") for t in tok[1:4]]
            f.append([int(a) - 1 for a, _ in pairs])
            ft.append([int(b) - 1 for _, b in pairs])
        else:
            assert ln == "usemtl mat0 "
    return (np.array(v, np.float32), np.array(vt, np.float32), np.array(f, np.int64), np.array(ft, np.int64))


def test_export_mesh_writes_reference_files(tmp_path):
    import cv2
    net, _ = _net_with_surface(36)
    assert net.export_mesh(str(tmp_path), resolution=36) is None
    assert sorted(os.listdir(tmp_path)) == ["albedo.png", "mesh.mtl", "mesh.obj"]
    with open(tmp_path / "mesh.mtl") as fp:
        assert fp.read() == REF_MTL
    v, f = mesh.extract_mesh(net, 36, 128)
    vt, ft, albedo, _ = mesh.bake_texture(net, v, f)
    pv, pvt, pf, pft = _parse_obj(tmp_path / "mesh.obj")
    assert np.array_equal(pv, v.cpu().numpy())
    vt_np = vt.cpu().numpy()
    assert np.array_equal(pvt[:, 0], vt_np[:, 0]) and np.array_equal(pvt[:, 1], np.float32(1) - vt_np[:, 1])
    assert np.array_equal(pf, f.cpu().numpy()) and np.array_equal(pft, ft.cpu().numpy())
    img = cv2.imread(str(tmp_path / "albedo.png"), cv2.IMREAD_UNCHANGED)
    expect = cv2.cvtColor((albedo.cpu().numpy() * 255).astype(np.uint8), cv2.COLOR_RGB2BGR)
    assert img.dtype == np.uint8 and np.array_equal(img, expect)


def test_export_mesh_is_deterministic(tmp_path):
    net, _ = _net_with_surface(36)
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    net.export_mesh(str(a), resolution=36)
    net.export_mesh(str(b), resolution=36)
    for name in ("mesh.obj", "mesh.mtl", "albedo.png"):
        assert filecmp.cmp(a / name, b / name, shallow=False), name


def test_export_mesh_default_resolution_is_grid_size(tmp_path):
    net, _ = _net_with_surface(24)
    net.grid_size = 24
    net.export_mesh(str(tmp_path))
    pv, _, pf, _ = _parse_obj(tmp_path / "mesh.obj")
    v, f = mesh.extract_mesh(net, net.grid_size, 128)
    assert np.array_equal(pv, v.cpu().numpy()) and np.array_equal(pf, f.cpu().numpy())


def test_errors(tmp_path):
    net, _ = _net()
    net.mean_density = 0                                # threshold min(0, 10) = 0 < every sigma: no surface
    with pytest.raises(Mi3dError):
        net.export_mesh(str(tmp_path), resolution=24)
    assert os.listdir(tmp_path) == []
    vol = torch.from_numpy(_random((8, 9, 10), 0))
    with pytest.raises(Mi3dError):
        mesh.marching_cubes(vol, 0.0)                   # CPU tensor
    with pytest.raises(Mi3dError):
        mesh.marching_cubes(vol.cuda().double(), 0.0)
    with pytest.raises(Mi3dError):
        mesh.marching_cubes(vol.cuda().transpose(0, 2), 0.0)
    with pytest.raises(Mi3dError):
        mesh.marching_cubes(torch.zeros(1, 5, 5, device="cuda"), 0.0)
    with pytest.raises(Mi3dError):
        mesh.marching_cubes(torch.zeros(5, 5, device="cuda"), 0.0)
    with pytest.raises(Mi3dError):
        mesh.bake_texture(net, torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32))
    with pytest.raises(Mi3dError):
        mesh.atlas_layout(2 * 2049 ** 2)
