"""GPU checks of the refine stage's point renderer and z-buffer (csrc/points.cu behind nerf/refine_utils.py):
- against the CPU oracle (oracle/points_ref.py) at the same fp32 op order: identical slot indices, bit-equal zbuf / dist2, image within
  1e-6, feature gradient within 1e-5 of the oracle's autograd;
- against the reference's own render_point glue and z_buffer (tests/golden/points_ref.npz);
- run-to-run determinism, argument handling, and one refine-shaped step (three scales + the mask at 800^2, loss, backward, Adam)."""
import importlib

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import points_ref as pr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ru():
    return importlib.import_module("make-it-3d_b200.nerf.refine_utils")


def _scene(kind, S, P, C, seed):
    rng = np.random.default_rng(seed)
    if kind == "dense":
        cloud = pr.surface_cloud(33, max(32, int(np.sqrt(P / 33 / 0.3))), seed=seed)
        pts = cloud[rng.permutation(cloud.shape[0])[:P]]
    else:
        pts = (rng.standard_normal((P, 3)) * 0.4).astype(np.float32)
        pts[: P // 20] *= 4.0                                   # some behind the camera, some off the image
    feats = rng.random((pts.shape[0], C), dtype=np.float32)
    c2w = pr.lookat_c2w(1.2, 70.0 + seed, 30.0 * seed)
    return pts, feats, pr.intrinsics(S), np.linalg.inv(c2w)


# (S, cloud, points, channels, radius in NDC): 0.005 is the refine stage's 2 px at 800^2 (0.5 px at 200^2)
CASES = [(64, "dense", 20000, 3, 4 / 64), (64, "random", 5000, 19, 4 / 64), (200, "dense", 100000, 19, 0.005),
         (200, "random", 50000, 3, 2 / 200 * 2), (800, "dense", 200000, 3, 0.005), (800, "random", 200000, 19, 0.005)]


@pytest.mark.parametrize("S,kind,P,C,radius", CASES)
def test_matches_oracle(ru, S, kind, P, C, radius):
    pts, feats, K, w2c = _scene(kind, S, P, C, seed=S + C)
    ref_f = torch.from_numpy(feats).requires_grad_()
    img_r, idx_r, zb_r, d2_r, _ = pr.render_point_ref(torch.from_numpy(pts), ref_f, S, S, torch.from_numpy(K), torch.from_numpy(w2c),
                                                      [S, S], radius, 8)
    G = torch.randn(img_r.shape, generator=torch.Generator().manual_seed(1))
    (img_r * G).sum().backward()

    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    Kc, w2cc = cu(K).float(), cu(w2c).float()
    f = cu(feats).requires_grad_()
    img = ru.render_point(cu(pts), f, S, S, Kc, w2cc, [S, S], radius, 8)
    (img * G.cuda()).sum().backward()
    idx, zb, d2 = ru.rasterize_points(cu(pts), S, S, Kc, w2cc, [S, S], radius, 8)
    torch.cuda.synchronize()
    covered = float((idx_r[..., 0] >= 0).float().mean())
    print(f"S={S} {kind} P={P} C={C}: covered {covered:.3f}, full {float((idx_r[..., -1] >= 0).float().mean()):.3f}")
    assert covered > 0.05
    assert torch.equal(idx[0].cpu().long(), idx_r)
    assert torch.equal(zb[0].cpu(), zb_r) and torch.equal(d2[0].cpu(), d2_r)
    assert float((img.detach().cpu() - img_r.detach()).abs().max()) <= 1e-6
    gr, g = ref_f.grad, f.grad.cpu()
    assert float((g - gr).abs().max() / gr.abs().max()) <= 1e-5


@pytest.mark.parametrize("case", ["a", "b"])
def test_matches_reference_glue(ru, case):
    g = pr.golden_case(load_golden("points_ref.npz"), case + "_")
    S, radius = int(g["S"]), float(g["radius"])
    ndc = torch.from_numpy(g["ndc"])
    idx_g, _, _ = pr.rasterize_ndc(ndc[:, 0], ndc[:, 1], ndc[:, 2], S, radius, 8)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    args = (S, S, cu(g["K"]).float(), cu(g["w2c"]).float(), [S, S], radius, 8)
    img = ru.render_point(cu(g["points"]), cu(g["feats"]), *args)
    idx = ru.rasterize_points(cu(g["points"]), *args)[0][0].cpu().long()
    same = (idx == idx_g).all(-1)
    err = (img[0].cpu() - torch.from_numpy(g["image"])[0]).abs().amax(0)[same]
    print(f"case {case}: same slot lists {float(same.float().mean()):.5f}, max |d image| there {float(err.max()):.2e}")
    assert same.float().mean() >= 0.999 and float(err.max()) <= 1e-5


@pytest.mark.parametrize("case", ["depth", "rand0", "rand1"])
def test_zbuffer_matches_reference(ru, case):
    g = pr.golden_case(load_golden("points_ref.npz"), f"zb_{case}_")
    S = int(g["S"])
    mask = ru.z_buffer(g["v"], g["w2c"], S, S, g["K"])
    assert mask.dtype == bool and np.array_equal(mask, g["mask"])


def test_zbuffer_large_matches_oracle(ru):
    S = 800
    c2w = pr.lookat_c2w(1.2, 75.0, 40.0)
    v = np.concatenate([pr.surface_cloud(33, 96, seed=4).astype(np.float64), np.random.default_rng(4).standard_normal((100000, 3)) * 0.5])
    mask = ru.z_buffer(v, np.linalg.inv(c2w), S, S, pr.intrinsics(S))
    assert np.array_equal(mask, pr.z_buffer_ref(v, np.linalg.inv(c2w), S, S, pr.intrinsics(S)))


def test_bit_identical_across_runs(ru):
    S, C = 200, 19
    pts, feats, K, w2c = _scene("dense", S, 150000, C, seed=2)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    G = torch.randn(1, C, S, S, device="cuda")
    outs = []
    for _ in range(2):
        f = cu(feats).requires_grad_()
        img = ru.render_point(cu(pts), f, S, S, cu(K).float(), cu(w2c).float(), [S, S], 0.01, 8)
        saved = [t.clone() for t in img.grad_fn.saved_tensors[3:]]        # idx, w
        (img * G).sum().backward()
        outs.append([img.detach().clone(), f.grad.clone()] + saved)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_float64_cameras_and_channel_counts(ru):
    S = 64
    pts, feats, K, w2c = _scene("dense", S, 8000, 19, seed=3)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for C in (3, 19):
        a = ru.render_point(cu(pts), cu(feats[:, :C]), S, S, cu(K), cu(w2c), [S, S], 0.05, 8)         # float64 K / world2cam
        b = ru.render_point(cu(pts), cu(feats[:, :C]), S, S, cu(K).float(), cu(w2c).float(), [S, S], 0.05, 8)
        assert a.shape == (1, C, S, S) and torch.equal(a, b) and float(a.abs().sum()) > 0


def test_argument_errors(ru):
    from importlib import import_module
    Mi3dError = import_module("make-it-3d_b200._lib").Mi3dError
    pts, feats = torch.rand(100, 3, device="cuda"), torch.rand(100, 3, device="cuda")
    K, w2c = torch.from_numpy(pr.intrinsics(32)).cuda(), torch.eye(4, device="cuda")
    with pytest.raises(Mi3dError):
        ru.render_point(pts.cpu(), feats.cpu(), 32, 32, K.cpu(), w2c.cpu(), [32, 32], 0.1, 8)
    with pytest.raises(Mi3dError):
        ru.render_point(pts, feats, 32, 32, K, w2c, [32, 32], 0.1, 8, acc="normweightedsum")
    with pytest.raises(Mi3dError):
        ru.render_point(pts, feats, 32, 32, K, w2c, [32, 48], 0.1, 8)
    with pytest.raises(Mi3dError):
        ru.render_point(pts.clone().requires_grad_(), feats, 32, 32, K, w2c, [32, 32], 0.1, 8)
    with pytest.raises(Mi3dError):      # more than 16 points per pixel
        ru.render_point(pts, feats, 32, 32, K, w2c, [32, 32], 0.1, 17)
    with pytest.raises(Mi3dError):      # more than 32 channels
        ru.render_point(pts, torch.rand(100, 33, device="cuda"), 32, 32, K, w2c, [32, 32], 0.1, 8)


def test_refine_shaped_step(ru):
    """nerf/utils.py:846-868: three colour renders (3 + 16 channels) at 800 / 400 / 200 and the 800^2 mask, loss, backward, Adam"""
    H = 800
    radius, ppp = 2.0 / H * 2.0, 8
    v = torch.from_numpy(pr.surface_cloud(33, 128, seed=5)).cuda()
    P = v.shape[0]
    color = torch.nn.Parameter(torch.rand(P, 3, device="cuda"))
    feat = torch.nn.Parameter(torch.randn(P, 16, device="cuda"))
    opt = torch.optim.Adam([color, feat], lr=1e-3, betas=(0.9, 0.99), eps=1e-15)
    w2c = torch.linalg.inv(torch.from_numpy(pr.lookat_c2w(1.2, 60.0, 20.0)).float().cuda())
    c0, f0 = color.detach().clone(), feat.detach().clone()
    all_c = torch.cat((color, feat), dim=-1)
    preds = []
    for scale in (1, 2, 4):
        h = H // scale
        preds.append(ru.render_point(v, all_c, h, h, torch.from_numpy(pr.intrinsics(h)).float().cuda(), w2c, (h, h), radius, ppp))
    mask = ru.render_point(v, torch.ones_like(v), H, H, torch.from_numpy(pr.intrinsics(H)).float().cuda(), w2c, (H, H), radius, ppp)
    loss = sum(((p[:, :3] - 0.5) ** 2).mean() + p[:, 3:].abs().mean() for p in preds) + (1 - mask).mean()
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert [tuple(p.shape) for p in preds] == [(1, 19, 800, 800), (1, 19, 400, 400), (1, 19, 200, 200)]
    assert 0.1 < float(mask.mean()) < 1.0
    for p, p0 in ((color, c0), (feat, f0)):
        assert torch.isfinite(p.grad).all() and float(p.grad.abs().sum()) > 0
        assert (p.detach() != p0).any(dim=1).float().mean() > 0.2
