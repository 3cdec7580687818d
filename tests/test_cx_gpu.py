"""The contextual-loss engine (csrc/cx_engine.cu, nerf/contextual_loss.py) against the fp32 oracle (oracle/cx_ref.py) on the GPU.

Tolerance: max(2.5 x the oracle's own fp16-storage error, 1e-3), the floor measured by running the oracle with every VGG layer output
rounded to fp16, as the engine stores them.  The oracle runs with TF32 off."""
import importlib
import math

import pytest
import torch

from oracle import cx_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return importlib.import_module("make-it-3d_b200.nerf.contextual_loss"), importlib.import_module("make-it-3d_b200._lib")


def _module(cl, seed=0, **kw):
    params = cx_ref.seeded_params(seed, "cuda")
    return cl.ContextualLoss(device="cuda", state_dict=params, **kw), params


def _images(N, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(N, 3, H, W, device="cuda", generator=g)
    y = 0.3 * x + 0.7 * torch.rand(N, 3, H, W, device="cuda", generator=g)
    return x, y


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _oracle(params, x, y, round_fp16):
    xr = x.detach().clone().requires_grad_(True)
    loss = cx_ref.contextual_loss(xr, y, params, 0.5, round_fp16)
    loss.backward()
    with torch.no_grad():
        feats = cx_ref.vgg_features(cx_ref.normalize_images(torch.cat([x, y])), params, round_fp16)
    return float(loss.detach()), xr.grad, feats


@pytest.mark.parametrize("N,H,W", [(1, 64, 64), (1, 200, 200), (1, 96, 160), (2, 64, 96), (1, 800, 800)])
def test_engine_matches_oracle(mods, N, H, W):
    cl, _ = mods
    m, params = _module(cl)
    x, y = _images(N, H, W, seed=H + W + N)
    xg = x.clone().requires_grad_(True)
    loss = m(xg, y)
    loss.backward()
    feats = m.engine(N, H, W).debug_tensor("relu5_4").view(2 * N, H // 16, W // 16, 512).permute(0, 3, 1, 2).float()
    l32, g32, f32 = _oracle(params, x, y, False)
    l16, g16, f16 = _oracle(params, x, y, True)
    # the loss is relative to max(|loss|, 1e-3): small images (few relu5_4 positions) give losses near -1e-5, where relative error is noise
    lscale = max(abs(l32), 1e-3)
    floor_f, floor_l, floor_g = _rel(f16, f32), abs(l16 - l32) / lscale, _rel(g16, g32)
    err_f, err_l, err_g = _rel(feats, f32), abs(float(loss.detach()) - l32) / lscale, _rel(xg.grad, g32)
    print(f"{N}x{H}x{W}: loss {float(loss):.6f} vs {l32:.6f}; feats {err_f:.2e} (floor {floor_f:.2e}) loss {err_l:.2e} "
          f"(floor {floor_l:.2e}) dx {err_g:.2e} (floor {floor_g:.2e})")
    assert err_f <= max(2.5 * floor_f, 1e-3)
    assert err_l <= max(2.5 * floor_l, 1e-3)
    assert err_g <= max(2.5 * floor_g, 1e-3)


def test_identical_images_give_finite_loss(mods):
    cl, _ = mods
    m, _ = _module(cl)
    x, _ = _images(1, 800, 800, seed=7)
    xg = x.clone().requires_grad_(True)
    loss = m(xg, x.clone())
    loss.backward()
    assert math.isfinite(float(loss)) and abs(float(loss) - (-math.log(1 + 1e-5))) < 1e-6, float(loss)
    assert torch.isfinite(xg.grad).all()


def test_repeat_and_graph_replay_bit_identical(mods):
    cl, _ = mods
    x, y = _images(1, 200, 200, seed=3)
    outs = []
    for replay in (False, True):
        m, _ = _module(cl, graph_replay=replay)
        for _ in range(4):
            xg = x.clone().requires_grad_(True)
            loss = m(xg, y)
            loss.backward()
            outs.append((loss.detach().clone(), xg.grad.clone()))
        if replay:
            assert m.engine(1, 200, 200).graph_replays() == 2
    for l, g in outs[1:]:
        assert torch.equal(l, outs[0][0]) and torch.equal(g, outs[0][1])


def test_no_grad_runs_forward_only(mods):
    cl, _ = mods
    m, _ = _module(cl)
    x, y = _images(1, 64, 64, seed=5)
    with torch.no_grad():
        a = m(x, y)
    b = m(x.clone().requires_grad_(True), y)
    assert torch.equal(a, b.detach()) and a.grad_fn is None


def test_argument_errors(mods):
    cl, L = mods
    m, _ = _module(cl)
    x, y = _images(1, 64, 64, seed=1)
    with pytest.raises(L.Mi3dError):
        m(x.cpu(), y.cpu())
    with pytest.raises(L.Mi3dError):
        m(x[:, :2], y[:, :2])
    with pytest.raises(L.Mi3dError):
        m(x, y[:, :, :32])
    with pytest.raises(L.Mi3dError):
        m(x[:, :, :15], y[:, :, :15])
    with pytest.raises(L.Mi3dError):
        m(x, y.clone().requires_grad_(True))
    for kw in (dict(loss_type="l1"), dict(loss_type="l2"), dict(use_vgg=False), dict(vgg_layer="relu3_4"), dict(vgg_layer="relu4_4")):
        with pytest.raises(L.Mi3dError):
            cl.ContextualLoss(device="cuda", **kw)


def test_refine_shaped_step(mods):
    """render_point at 800^2 -> a small torch head -> ContextualLoss -> backward: the gradient reaches the point colours and features"""
    from oracle import points_ref as pr
    cl, _ = mods
    ru = importlib.import_module("make-it-3d_b200.nerf.refine_utils")
    m, _ = _module(cl)
    H = 800
    v = torch.from_numpy(pr.surface_cloud(33, 128, seed=5)).cuda()
    P = v.shape[0]
    color = torch.nn.Parameter(torch.rand(P, 3, device="cuda"))
    feat = torch.nn.Parameter(torch.randn(P, 16, device="cuda"))
    w2c = torch.linalg.inv(torch.from_numpy(pr.lookat_c2w(1.2, 60.0, 20.0)).float().cuda())
    img = ru.render_point(v, torch.cat((color, feat), dim=-1), H, H, torch.from_numpy(pr.intrinsics(H)).float().cuda(), w2c, (H, H),
                          2.0 / H * 2.0, 8)
    head = torch.nn.Conv2d(19, 3, 1).cuda()
    rgb = torch.sigmoid(head(img))
    gt = torch.rand(1, 3, H, H, device="cuda")
    loss = m(rgb, gt)
    loss.backward()
    assert math.isfinite(float(loss))
    for t in (color, feat):
        assert t.grad is not None and torch.isfinite(t.grad).all() and float(t.grad.abs().sum()) > 0
