"""GPU parity (through the C ABI): hash grid, the field forward's tf32 split tiles, fused field forward/backward, fused render
step vs the oracle and vs the golden vectors recorded from the reference's Python.  Tolerances (fp32 path): 1e-3 relative is
BASELINE.json's bar; these tests hold the fp32 kernels to much tighter bounds and say so per assertion."""
import argparse
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import field_from_golden, fr, make_table, max_abs, orm, rel_err, sphere_bitfield

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    return importlib.import_module("make-it-3d_b200._lib")


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _opt(**kw):
    o = argparse.Namespace(bound=1, min_near=0.1, density_thresh=10, bg_radius=-1, blob_density=5, blob_radius=0.1,
                           lambda_smooth=1, max_depth=10.0)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _net_from_golden(g, **optkw):
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    net = nt.NeRFNetwork(_opt(**optkw))
    table = make_table(net.encoder.params.numel(), int(g["table_seed"]), float(g["table_scale"]))
    with torch.no_grad():
        net.encoder.params.copy_(torch.from_numpy(table))
        for l, (w, b) in enumerate((("w1", "b1"), ("w2", "b2"), ("w3", "b3"))):
            net.sigma_net.net[l].weight.copy_(torch.from_numpy(g[w]))
            net.sigma_net.net[l].bias.copy_(torch.from_numpy(g[b]))
    return net.cuda()


def test_hashgrid_forward_backward_vs_oracle():
    nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
    enc = nt.HashGridEncoding().cuda()
    table = make_table(enc.params.numel(), 5, 1.0)
    with torch.no_grad():
        enc.params.copy_(torch.from_numpy(table))
    rng = np.random.default_rng(1)
    x = rng.random((20000, 3), dtype=np.float32)
    x[:6] = np.array([[0, 0, 0], [1, 1, 1], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0.5, 0.5]], np.float32)   # x == 1 wraps dense levels
    out = enc(_cu(x))
    ref = orm.hashgrid_forward(x, table, orm.hashgrid_levels())
    assert max_abs(out.detach().cpu(), ref) < 2e-6            # fp32 interpolation, different summation order only
    # backward: scatter-add == autograd of the torch restatement
    g = rng.standard_normal(ref.shape).astype(np.float32)
    (out * _cu(g)).sum().backward()
    enc_ref = fr.HashGridRef()
    with torch.no_grad():
        enc_ref.params.copy_(torch.from_numpy(table))
    (enc_ref(torch.from_numpy(x)) * torch.from_numpy(g)).sum().backward()
    gt, gr = enc.params.grad.cpu().numpy(), enc_ref.params.grad.numpy()
    assert np.array_equal(gt != 0, gr != 0)
    assert max_abs(gt, gr) < 1e-4 * max(1.0, np.abs(gr).max())


@pytest.mark.parametrize("shading,ratio", [("albedo", 1.0), ("lambertian", 0.1), ("textureless", 0.1), ("normal", 0.1)])
def test_field_forward_backward_vs_torch_oracle(shading, ratio):
    """NeRFNetwork.forward on random points (incl. points on the box faces) vs oracle.FieldRef + autograd."""
    g = load_golden("render_albedo.npz")
    net = _net_from_golden(g)
    field, _ = field_from_golden(g)
    rng = np.random.default_rng(11)
    m = 3000
    x = (rng.random((m, 3), dtype=np.float32) * 2 - 1) * 0.6
    x[:4] = np.array([[1, 1, 1], [-1, -1, -1], [0.995, 0, 0], [0, 0, 0]], np.float32)
    d = rng.standard_normal((m, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=1, keepdims=True)
    l = np.array([0.3, 0.5, 0.81], np.float32); l /= np.linalg.norm(l)
    sig, col, nrm = net(_cu(x), _cu(d), _cu(l), ratio=ratio, shading=shading)
    sig_r, col_r, nrm_r = field(torch.from_numpy(x), torch.from_numpy(d), torch.from_numpy(l), ratio=ratio, shading=shading)
    assert rel_err(sig.detach().cpu(), sig_r.detach(), floor=1e-3) < 2e-5
    # lit colours inherit the normal's fp32 cancellation error (<= 5e-4 on a unit vector)
    assert max_abs(col.detach().cpu(), col_r.detach()) < (2e-5 if shading == 'albedo' else 5e-4)
    # normals difference two densities 0.02 apart: allow 5e-4 absolute on unit vectors (fp32 cancellation)
    assert max_abs(nrm.detach().cpu(), nrm_r.detach()) < 5e-4
    gs, gc, gn = rng.standard_normal(m).astype(np.float32), rng.standard_normal((m, 3)).astype(np.float32), rng.standard_normal((m, 3)).astype(np.float32) * 0.1
    ((sig * _cu(gs)).sum() + (col * _cu(gc)).sum() + (nrm * _cu(gn)).sum()).backward()
    ((sig_r * torch.from_numpy(gs)).sum() + (col_r * torch.from_numpy(gc)).sum() + (nrm_r * torch.from_numpy(gn)).sum()).backward()
    for lyr in range(3):
        for p, q in ((net.sigma_net.net[lyr].weight, field.sigma_net.net[lyr].weight), (net.sigma_net.net[lyr].bias, field.sigma_net.net[lyr].bias)):
            scale = max(1e-3, float(q.grad.abs().max()))
            assert max_abs(p.grad.cpu(), q.grad) / scale < 2e-3, (lyr, tuple(q.shape))
    gt, gr = net.encoder.params.grad.cpu().numpy(), field.encoder.params.grad.numpy()
    assert max_abs(gt, gr) / max(1e-6, np.abs(gr).max()) < 2e-3


@pytest.mark.parametrize("N,K", [(64, 32), (64, 64), (32, 64), (16, 64), (64, 128), (32, 128)])
def test_tf32_split_tiles(L, N, K):
    """Hand-written wgmma tf32 tiles of the field FORWARD kernel (K-major operands): the 3-term split must be fp32-class.
    (tf32 wgmma reads K-major operands only, which is why the backward uses bf16 tiles.)"""
    g = torch.Generator(device="cuda").manual_seed(N + K)
    a = torch.randn(128, K, device="cuda", generator=g); b = torch.randn(N, K, device="cuda", generator=g); ref = a.double() @ b.double().t()
    d = torch.empty(128, N, device="cuda")
    L.check(L.lib().mi3d_tf32_tile_test(L.ptr(a), L.ptr(b), L.ptr(d), C.c_int(N), C.c_int(K), C.c_int(0), L.stream()), "tf32_tile_test")
    torch.cuda.synchronize()
    err = (d.double() - ref).abs().max().item()
    assert err < 2e-5 * max(1.0, ref.abs().max().item()), (N, K, err)     # plain tf32 would be ~1e-2


def test_density_matches_oracle_and_k1_backward():
    g = load_golden("render_albedo.npz")
    net = _net_from_golden(g)
    field, _ = field_from_golden(g)
    rng = np.random.default_rng(12)
    x = (rng.random((1000, 3), dtype=np.float32) * 2 - 1)
    out = net.density(_cu(x))
    ref = field.density(torch.from_numpy(x))
    assert rel_err(out["sigma"].detach().cpu(), ref["sigma"].detach(), floor=1e-3) < 2e-5
    assert max_abs(out["albedo"].detach().cpu(), ref["albedo"].detach()) < 2e-5
    (out["sigma"].sum() + out["albedo"].sum()).backward()
    (ref["sigma"].sum() + ref["albedo"].sum()).backward()
    q = field.sigma_net.net[1].weight.grad
    assert max_abs(net.sigma_net.net[1].weight.grad.cpu(), q) / float(q.abs().max()) < 1e-3


@pytest.mark.parametrize("case", ["albedo", "lambertian", "textureless"])
def test_fused_render_step_matches_reference_golden(case):
    """The drop-in call Trainer.train_step makes (model.render(...), nerf/utils.py:496) on the fused CUDA path vs the
    golden vectors recorded from the reference's Python: image / depth / weights_sum / losses and parameter gradients."""
    g = load_golden(f"render_{case}.npz")
    net = _net_from_golden(g)
    net.train()
    net.density_bitfield = _cu(sphere_bitfield(float(g["radius"])))
    out = net.render(_cu(g["rays_o"])[None], _cu(g["rays_d"])[None], depth_scale=_cu(g["depth_scale"])[None], bg_color=_cu(g["bg_color"]),
                     staged=False, perturb=True, light_d=_cu(g["light_d"]), ambient_ratio=float(g["ratio"]), shading=str(g["shading"]),
                     force_all_rays=True, max_steps=512, dt_gamma=0, T_thresh=1e-4, noises=_cu(g["noises"]),
                     smooth_noise=_cu(g["smooth_noise"]))
    ws = list(net._workspaces.values())[0]
    assert int(ws.counter[0]) == int(g["total"])
    tol = 1e-3   # BASELINE.json north_star: "outputs within 1e-3 rel of reference"
    assert max_abs(out["image"][0].detach().cpu(), g["image"]) < 2e-5
    assert max_abs(out["weights_sum"][0].detach().cpu(), g["weights_sum"]) < 2e-5
    assert rel_err(out["depth"][0, :, 0].detach().cpu(), g["depth"], floor=1e-2) < 1e-4
    assert np.array_equal(out["mask"][0].cpu().numpy(), g["mask"])
    assert abs(out["loss_orient"].item() / float(g["loss_orient"]) - 1) < tol
    assert abs(out["loss_smooth"].item() / float(g["loss_smooth"]) - 1) < tol
    loss = (out["image"][0] * _cu(g["A"])).sum() + (out["weights_sum"][0] * _cu(g["B"])).sum() + (out["depth"][0, :, 0] * _cu(g["Cd"])).sum() \
        + 30.0 * out["loss_orient"] + 50.0 * out["loss_smooth"]
    loss.backward()
    for l, (w, b) in enumerate((("g_w1", "g_b1"), ("g_w2", "g_b2"), ("g_w3", "g_b3"))):
        for p, ref in ((net.sigma_net.net[l].weight.grad, g[w]), (net.sigma_net.net[l].bias.grad, g[b])):
            assert max_abs(p.cpu(), ref) / max(1e-3, np.abs(ref).max()) < 5e-3, (case, w)
    gt = net.encoder.params.grad.cpu().numpy()
    ref = g["g_table_val"]
    assert max_abs(gt[g["g_table_idx"]], ref) / np.abs(ref).max() < 5e-3
    assert abs(np.sqrt((gt.astype(np.float64) ** 2).sum()) / float(g["g_table_l2"]) - 1) < 5e-3
    assert abs(np.count_nonzero(gt) / int(g["g_table_nnz"]) - 1) < 1e-3
    # second backward through the retained tape (sd.py:171 then utils.py:983): gradients ACCUMULATE
    net.zero_grad()
    out2 = net.render(_cu(g["rays_o"])[None], _cu(g["rays_d"])[None], depth_scale=_cu(g["depth_scale"])[None], bg_color=_cu(g["bg_color"]),
                      perturb=True, light_d=_cu(g["light_d"]), ambient_ratio=float(g["ratio"]), shading=str(g["shading"]),
                      force_all_rays=True, max_steps=512, noises=_cu(g["noises"]), smooth_noise=_cu(g["smooth_noise"]))
    (out2["image"][0] * _cu(g["A"])).sum().backward(retain_graph=True)
    g1 = net.sigma_net.net[2].weight.grad.clone()
    (out2["image"][0] * _cu(g["A"])).sum().backward()
    assert max_abs(net.sigma_net.net[2].weight.grad.cpu(), 2 * g1.cpu()) < 1e-4 * float(g1.abs().max())


def test_full_size_properties_128():
    """BASELINE size (128x128, sphere r=0.2, radius 1.25): size-independent properties of the fused path."""
    from helpers import camera_rays
    g = load_golden("render_albedo.npz")
    net = _net_from_golden(g)
    net.train()
    net.density_bitfield = _cu(sphere_bitfield(0.2))
    ro, rd, sc = camera_rays(128)
    noises = np.random.default_rng(3).random(128 * 128, dtype=np.float32)
    kw = dict(depth_scale=_cu(sc)[None], bg_color=_cu(np.array([0.2, 0.5, 0.7], np.float32)), perturb=True, light_d=_cu(g["light_d"]),
              shading="albedo", force_all_rays=True, max_steps=512, noises=_cu(noises))
    torch.manual_seed(0)
    a = net.render(_cu(ro)[None], _cu(rd)[None], **kw)
    ws = list(net._workspaces.values())[0]
    total = int(ws.counter[0])
    aabb = np.array([-1, -1, -1, 1, 1, 1], np.float32)
    n_o, f_o = orm.near_far_from_aabb(ro, rd, aabb, 0.2)
    *_, rays_o_, tot_o = orm.march_rays_train(ro, rd, 1.0, sphere_bitfield(0.2), 1, 128, n_o, f_o, noises, 0.0, 512, align=128)
    assert total == tot_o and 400000 < total < 450000                 # oracle count (SURVEY 8d: M ~ 0.42 M for this camera)
    assert np.array_equal(ws.rays.cpu().numpy(), rays_o_)
    img, wsum = a["image"][0], a["weights_sum"][0]
    assert torch.isfinite(img).all() and (wsum >= 0).all() and (wsum <= 1 + 1e-5).all()
    # rays that miss every occupied cell return exactly the background and the far depth
    rays = ws.rays.cpu().numpy()
    empty = torch.from_numpy(rays[:, 2] == 0).cuda()
    assert torch.equal(img[empty], _cu(np.array([0.2, 0.5, 0.7], np.float32)).expand(int(empty.sum()), 3))
    assert torch.allclose(a["depth"][0, :, 0][empty], 10.0 * _cu(sc)[empty])
    # linearity of compositing in the colour channel: image - (1-ws)*bg is independent of bg
    kw2 = dict(kw, bg_color=_cu(np.array([0.9, 0.1, 0.3], np.float32)))
    b = net.render(_cu(ro)[None], _cu(rd)[None], **kw2)
    fa = img - (1 - wsum)[:, None] * kw["bg_color"]
    fb = b["image"][0] - (1 - b["weights_sum"][0])[:, None] * kw2["bg_color"]
    assert torch.equal(wsum, b["weights_sum"][0]) and (fa - fb).abs().max() < 1e-6
    # determinism: same inputs, same bits (ray-ordered compaction, fixed-order loss reduction)
    c = net.render(_cu(ro)[None], _cu(rd)[None], **kw)
    assert torch.equal(c["image"], a["image"]) and torch.equal(c["loss_orient"], a["loss_orient"])


def test_update_extra_state_matches_oracle():
    """renderer.py:587-637 on the device (one C-ABI call) vs the oracle restatement with the same jitter."""
    g = load_golden("render_albedo.npz")
    net = _net_from_golden(g)
    field, _ = field_from_golden(g)
    H = 128
    rng = np.random.default_rng(21)
    jitter = rng.random((1, H ** 3, 3), dtype=np.float32)
    grid0 = (rng.random((1, H ** 3), dtype=np.float32) * 2).astype(np.float32)
    net.density_grid.copy_(_cu(grid0))
    net.update_extra_state(decay=0.95, jitter=_cu(jitter))
    # oracle: cell m (Morton order) -> coords -> xyz in [-1,1] * (bound - hgs) + (2u-1) * hgs
    coords = orm.morton3D_invert(np.arange(H ** 3, dtype=np.int32)).astype(np.float32)
    xyz = 2 * coords / (H - 1) - 1
    hgs = np.float32(1.0 / H)
    pts = xyz * (np.float32(1.0) - hgs) + (jitter[0] * 2 - 1) * hgs
    sub = rng.choice(H ** 3, 20000, replace=False)
    with torch.no_grad():
        sig = field.density(torch.from_numpy(pts[sub]))["sigma"].numpy()
    want = np.maximum(grid0[0, sub] * np.float32(0.95), sig)
    got = net.density_grid[0].cpu().numpy()
    assert rel_err(got[sub], want, floor=1e-3) < 5e-5
    mean = float(got.astype(np.float64).mean())
    assert abs(float(net.mean_density) / mean - 1) < 1e-5
    np.testing.assert_array_equal(net.density_bitfield.cpu().numpy(), orm.packbits(got, min(mean, 10.0)))


def test_march_overflow_exposes_only_written_rows():
    """opt.max_samples caps the per-sample buffers below N*max_steps (ADVICE r1): rays that do not fit write nothing
    (raymarching.cu:416) and counter[0] must then be the emitted prefix, so that the field kernels never touch unwritten rows
    (nothing is zero-filled here, unlike raymarching.py:217-219).  Dropped rays composite to the background."""
    from helpers import camera_rays
    g = load_golden("render_albedo.npz")
    cap = 20000
    net = _net_from_golden(g, max_samples=cap)
    net.train()
    net.density_bitfield = _cu(sphere_bitfield(0.3))
    HW = 64
    ro, rd, sc = camera_rays(HW)
    noises = np.random.default_rng(5).random(HW * HW, dtype=np.float32)
    bg = np.array([0.2, 0.5, 0.7], np.float32)
    kw = dict(depth_scale=_cu(sc)[None], bg_color=_cu(bg), perturb=True, light_d=_cu(g["light_d"]), shading="lambertian", ambient_ratio=0.1,
              force_all_rays=True, max_steps=512, noises=_cu(noises))
    out = net.render(_cu(ro)[None], _cu(rd)[None], **kw)
    ws = list(net._workspaces.values())[0]
    ws.xyzs.fill_(float("nan")); ws.tape.fill_(float("nan"))          # poison: a second render must not read stale / unwritten rows
    out = net.render(_cu(ro)[None], _cu(rd)[None], **kw)
    rays = ws.rays.cpu().numpy()
    total_uncapped = int(rays[:, 2].sum())
    assert total_uncapped > cap, "test must overflow"
    fits = (rays[:, 1] + rays[:, 2]) <= cap
    emitted = int(rays[fits, 2].sum())
    assert int(ws.counter[0]) == emitted and emitted <= cap
    assert np.all(np.diff(fits.astype(np.int8)) <= 0)                  # dropped rays are a suffix (ray-ordered compaction)
    assert torch.isfinite(out["image"]).all() and torch.isfinite(out["loss_orient"]) and torch.isfinite(out["loss_smooth"])
    dropped = torch.from_numpy(~fits & (rays[:, 2] > 0)).cuda()
    assert torch.equal(out["image"][0][dropped], _cu(bg).expand(int(dropped.sum()), 3))
    (out["image"].sum() + out["loss_orient"] + out["loss_smooth"]).backward()
    assert torch.isfinite(net.encoder.params.grad).all() and all(torch.isfinite(p.grad).all() for p in net.sigma_net.parameters())
    # same result as a render given only the rays that fit (the cap changes nothing for them)
    n_fit = int(fits.sum())
    net2 = _net_from_golden(g)
    net2.train(); net2.density_bitfield = net.density_bitfield
    kw2 = dict(kw, depth_scale=_cu(sc[:n_fit])[None], noises=_cu(noises[:n_fit]))
    ref = net2.render(_cu(ro[:n_fit])[None], _cu(rd[:n_fit])[None], **kw2)
    assert torch.equal(ref["image"][0], out["image"][0][:n_fit])


def test_benchmark_size_render_matches_oracle_golden_128():
    """BASELINE size (128x128 rays, max_steps 512, k = 13, lambertian): image / depth / weights_sum / per-ray sample counts and the
    orientation mean against tests/golden/render_128.npz, computed once by the CPU oracle (tests/golden/make_golden_128.py; the
    oracle itself is pinned to the reference's Python by the 24x24 fixtures above)."""
    from helpers import camera_rays
    g = load_golden("render_albedo.npz")
    z = load_golden("render_128.npz")
    net = _net_from_golden(g)
    net.train()
    net.density_bitfield = _cu(sphere_bitfield(float(z["radius"])))
    ro, rd, sc = camera_rays(128)
    out = net.render(_cu(ro)[None], _cu(rd)[None], depth_scale=_cu(sc)[None], bg_color=_cu(z["bg_color"]), perturb=True, light_d=_cu(z["light_d"]),
                     ambient_ratio=float(z["ratio"]), shading="lambertian", force_all_rays=True, max_steps=512, noises=_cu(z["noises"]))
    ws = list(net._workspaces.values())[0]
    assert int(ws.counter[0]) == int(z["total"]) == 424346
    np.testing.assert_array_equal(ws.rays.cpu().numpy()[:, 2], z["counts"])
    assert max_abs(out["image"][0].detach().cpu(), z["image"]) < 5e-5
    assert max_abs(out["weights_sum"][0].detach().cpu(), z["weights_sum"]) < 2e-5
    assert rel_err(out["depth"][0, :, 0].detach().cpu(), z["depth"], floor=1e-2) < 1e-4
    # loss_orient = sum / padded rows (raymarching.py:237-241 padding applies to the whole image's sample list)
    m_pad = int(z["total"]) + 128 - int(z["total"]) % 128
    assert abs(out["loss_orient"].item() / (float(z["sum_orient"]) / m_pad) - 1) < 1e-3


def test_update_extra_state_matches_reference_golden():
    """Row R6 against the REFERENCE's own NeRFRenderer.update_extra_state (renderer.py:587-637) run through the import shims
    (tests/golden/make_golden_r6.py -> density_r6.npz): EMA-max grid, cells < 0 left alone, mean density, packed bitfield.  The
    reference's cell jitter (torch.rand_like after manual_seed) is regenerated here and re-ordered from its meshgrid order to the
    Morton order mi3d_density_grid_update indexes jitter by."""
    g = load_golden("render_albedo.npz")
    z = load_golden("density_r6.npz")
    net = _net_from_golden(g)
    H = 128
    grid0 = (np.random.default_rng(int(z["grid0_seed"])).random((1, H ** 3), dtype=np.float32) * 2).astype(np.float32)
    grid0[0, ::97] = -1.0
    net.density_grid.copy_(_cu(grid0))
    torch.manual_seed(int(z["seed"]))
    j_ref = torch.rand(H ** 3, 3).numpy()                                     # row i = (x, y, z) in meshgrid('ij') order
    idx = np.arange(H, dtype=np.int32)
    xx, yy, zz = np.meshgrid(idx, idx, idx, indexing="ij")
    morton = orm.morton3D(np.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], 1))
    jitter = np.empty_like(j_ref)
    jitter[morton] = j_ref
    net.update_extra_state(decay=0.95, jitter=_cu(jitter[None]))
    got = net.density_grid[0].cpu().numpy()
    sub = z["sub"]
    assert rel_err(got[sub], z["sub_vals"], floor=1e-3) < 5e-5
    assert np.all(got[::97] == -1.0)
    assert abs(float(net.mean_density) / float(z["mean_density"]) - 1) < 1e-5
    bits = net.density_bitfield.cpu().numpy()
    diff = np.unpackbits(bits ^ z["bitfield"]).sum()
    assert diff <= 2, diff            # a cell sitting on the threshold (mean density, 4.7358) may flip with the last bit of sigma


def test_update_extra_state_with_shared_seed_is_replica_identical():
    """Multi-GPU invariant (parallel.py): every rank refreshes its own copy of the density grid with `seed=shared_seed(...)` and no
    broadcast follows, so two replicas holding the same parameters must end with BIT-identical grids and bitfields -- and a different
    seed must move the jittered cell positions (ADVICE r1: the jitter used to come from the process-global CPU generator)."""
    par = importlib.import_module("make-it-3d_b200.parallel")
    g = load_golden("render_albedo.npz")
    nets = [_net_from_golden(g) for _ in range(3)]
    for i, (net, seed) in enumerate(zip(nets, (par.shared_seed(3, 16), par.shared_seed(3, 16), par.shared_seed(3, 32)))):
        torch.manual_seed(100 + i)                      # the global generators differ between replicas, like between ranks
        net.update_extra_state(decay=0.95, seed=seed)
        net.update_extra_state(decay=0.95, seed=seed + 1)
    a, b, c = nets
    assert torch.equal(a.density_grid, b.density_grid) and torch.equal(a.density_bitfield, b.density_bitfield)
    assert float(a.mean_density) == float(b.mean_density)
    assert not torch.equal(a.density_grid, c.density_grid)
