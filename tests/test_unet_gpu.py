"""The gated U-Net engine (csrc/unet_engine.cu, nerf/unet.py) against the functional oracle (oracle/unet_ref.py) on the GPU.

The engine stores and accumulates in fp32, so it is held to an fp32-level bound: the reference is the oracle in float64, and each
tensor's max-abs error relative to its largest reference value must stay within max(20 x the fp32 oracle's own error, 2e-5) (TF32
off).  That is far inside the issue's fp16-storage bound and catches formula slips of 1e-4 (e.g. a biased running variance)."""
import importlib
import math

import pytest
import torch

from oracle import unet_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def um():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return importlib.import_module("make-it-3d_b200.nerf.unet")


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _inputs(N, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand(N, 19, H >> i, W >> i, device="cuda", generator=g) for i in range(3)]


def _module(um, seed=0):
    torch.manual_seed(seed)
    net = um.UNet(num_input_channels=3 + 16).cuda()
    with torch.no_grad():                  # non-trivial BatchNorm affine parameters and running statistics
        g = torch.Generator().manual_seed(seed + 1)
        for n, b in list(net.named_parameters()) + list(net.named_buffers()):
            if ".norm." in n and b.is_floating_point():
                b.add_((0.25 * (2 * torch.rand(b.shape, generator=g) - 1)).cuda())
    return net


def _oracle_params(net, double=False):
    out = {}
    for k, v in net.state_dict().items():
        t = v.detach().clone()
        if double and t.is_floating_point():
            t = t.double()
        out[k] = t.requires_grad_(True) if k in unet_ref.param_names() else t
    return out


def _oracle(net, xs, w, train=True, double=False, p=None):
    """-> output, input gradients, parameter gradients, buffers after the call; float64 when double"""
    p = _oracle_params(net, double) if p is None else p
    cast = (lambda t: t.double()) if double else (lambda t: t)
    xr = [cast(x.detach().clone()).requires_grad_(True) for x in xs]
    out = unet_ref.unet(xr, p, train=train)
    (out * cast(w)).sum().backward()
    grads = {n: p[n].grad for n in unet_ref.param_names()}
    bufs = {n: p[n] for n in p if n not in grads}
    return out.detach(), [x.grad for x in xr], grads, bufs


def _refs(net, xs, w, train=True):
    return _oracle(net, xs, w, train, double=True), _oracle(net, xs, w, train)


def _check(res, ref, floor_res, tag):
    tol = max(20 * _rel(floor_res, ref), 2e-5)
    err = _rel(res, ref)
    assert err <= tol, (tag, err, tol)
    return err


def _check_grads(xgrads, params, ref, flo, tag=""):
    for i in range(3):
        _check(xgrads[i], ref[1][i], flo[1][i], f"{tag}dx{i}")
    for n, p in params:
        _check(p.grad, ref[2][n], flo[2][n], tag + n)


def _check_buffers(buffers, ref, flo, count):
    for n, b in buffers:
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(ref[3][n]) == count, n
        else:
            _check(b, ref[3][n], flo[3][n], n)


def _compare(um, N, H, W, train=True):
    net = _module(um)
    if not train:
        net.eval()
    xs = _inputs(N, H, W, 1)
    w = torch.randn(N, 3, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    ref, flo = _refs(net, xs, w, train)
    xe = [x.clone().requires_grad_(True) for x in xs]
    out = net(xe)
    (out * w).sum().backward()
    torch.cuda.synchronize()
    _check(out, ref[0], flo[0], "out")
    _check_grads([x.grad for x in xe], net.named_parameters(), ref, flo)
    _check_buffers(net.named_buffers(), ref, flo, 1 if train else 0)


@pytest.mark.parametrize("N,H,W", [(1, 64, 64), (1, 200, 200), (2, 96, 160), (1, 800, 800)])
def test_engine_matches_oracle(um, N, H, W):
    _compare(um, N, H, W, train=True)


def test_eval_mode_matches_oracle(um):
    _compare(um, 1, 200, 200, train=False)


def test_running_statistics_small_batch(um):
    """N = 1 at 8 x 8: the coarsest BatchNorm averages 2 x 2 values, so a biased running variance would be off by a third of its update"""
    _compare(um, 1, 8, 8, train=True)
    L = importlib.import_module("make-it-3d_b200._lib")
    net = _module(um)
    xs = _inputs(1, 4, 4, 0)
    with pytest.raises(L.Mi3dError):           # one value per channel at H/4 x W/4, as torch's BatchNorm refuses in train mode
        net(xs)
    net.eval()
    assert torch.isfinite(net(xs)).all()


def test_two_backwards(um):
    net = _module(um)
    xs = _inputs(1, 64, 96, 3)
    g = torch.Generator(device="cuda").manual_seed(4)
    w1, w2 = torch.randn(1, 3, 64, 96, device="cuda", generator=g), torch.randn(1, 3, 64, 96, device="cuda", generator=g)
    ref, flo = _refs(net, xs, w1 + w2)
    xe = [x.clone().requires_grad_(True) for x in xs]
    out = net(xe)
    (out * w1).sum().backward(retain_graph=True)
    (out * w2).sum().backward()
    _check_grads([x.grad for x in xe], net.named_parameters(), ref, flo)


@pytest.mark.parametrize("train", [True, False])
def test_superseded_tape(um, train):
    """a later forward on the same engine replaces the tape: the earlier graph still gets its own forward's input and parameter
    gradients, and its rebuild neither updates the running statistics again (train) nor reads the updated ones (eval)"""
    net = _module(um)
    xs = _inputs(1, 64, 96, 3)
    w = torch.randn(1, 3, 64, 96, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    if not train:
        net.eval()
    ref, flo = _refs(net, xs, w, train)
    xa, xb = [x.clone().requires_grad_(True) for x in xs], [x.clone().requires_grad_(True) for x in _inputs(1, 64, 96, 9)]
    oa = net(xa)
    if not train:
        net.train()                            # the later forward updates the running statistics the eval tape read
    ob = net(xb)
    bufs = {n: b.clone() for n, b in net.named_buffers()}
    (oa * w).sum().backward()
    _check_grads([x.grad for x in xa], net.named_parameters(), ref, flo, "superseded ")
    for n, b in net.named_buffers():
        assert torch.equal(b, bufs[n]), n
        if n.endswith("num_batches_tracked"):
            assert int(b) == (2 if train else 1)
    del ob


@pytest.mark.parametrize("scale", [1e-8, 1e4])
def test_gradient_range(um, scale):
    net = _module(um)
    xs = _inputs(1, 64, 64, 5)
    w = scale * torch.randn(1, 3, 64, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    ref, flo = _refs(net, xs, w)
    xe = [x.clone().requires_grad_(True) for x in xs]
    (net(xe) * w).sum().backward()
    assert all(torch.isfinite(x.grad).all() for x in xe)
    _check_grads([x.grad for x in xe], net.named_parameters(), ref, flo)


def test_adam_steps_track_oracle(um):
    net = _module(um)
    pd, pf = _oracle_params(net, double=True), _oracle_params(net)
    opts = [torch.optim.Adam(net.parameters(), lr=1e-3)] + [torch.optim.Adam([q[n] for n in unet_ref.param_names()], lr=1e-3)
                                                             for q in (pd, pf)]
    for step in range(5):
        xs = _inputs(1, 64, 64, 10 + step)
        tgt = torch.rand(1, 3, 64, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(20 + step))
        for opt, fn in zip(opts, (lambda: net(xs), lambda: unet_ref.unet([x.double() for x in xs], pd),
                                  lambda: unet_ref.unet(xs, pf))):
            opt.zero_grad()
            ((fn() - tgt) ** 2).mean().backward()
            opt.step()
    for n, q in net.named_parameters():
        _check(q.detach(), pd[n].detach(), pf[n].detach(), n)


def test_bit_identical_and_graph_replay(um):
    xs = _inputs(1, 96, 128, 7)
    w = torch.randn(1, 3, 96, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    results = []
    for graph in (False, True):
        torch.manual_seed(0)
        net = um.UNet(num_input_channels=19, graph_replay=graph).cuda()
        for _ in range(4):
            for p in net.parameters():
                p.grad = None
            xe = [x.clone().requires_grad_(True) for x in xs]
            out = net(xe)
            (out * w).sum().backward()
            torch.cuda.synchronize()
            results.append([out.clone()] + [x.grad.clone() for x in xe] + [p.grad.clone() for p in net.parameters()])
        if graph:
            assert net.engines[(1, 96, 128, xs[0].device)].graph_replays() >= 2
    for r in results[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, results[0]))


def test_argument_errors(um):
    L = importlib.import_module("make-it-3d_b200._lib")
    net = _module(um)
    with pytest.raises(L.Mi3dError):
        net(_inputs(1, 66, 64, 0))
    xs = _inputs(1, 64, 64, 0)
    with pytest.raises(L.Mi3dError):
        net([xs[0], xs[1], xs[1]])
    with pytest.raises(L.Mi3dError):
        net([xs[0].cpu(), xs[1].cpu(), xs[2].cpu()])


def test_refine_shaped_step(um):
    """render_point x3 -> UNet -> ContextualLoss + an image loss -> backward: the gradient reaches the point colours and features and
    the U-Net's parameters"""
    from oracle import cx_ref
    from oracle import points_ref as pr
    ru = importlib.import_module("make-it-3d_b200.nerf.refine_utils")
    cl = importlib.import_module("make-it-3d_b200.nerf.contextual_loss")
    net = _module(um)
    cx = cl.ContextualLoss(device="cuda", state_dict=cx_ref.seeded_params(0, "cuda"))
    H = 800
    v = torch.from_numpy(pr.surface_cloud(33, 128, seed=5)).cuda()
    P = v.shape[0]
    color = torch.nn.Parameter(torch.rand(P, 3, device="cuda"))
    feat = torch.nn.Parameter(torch.randn(P, 16, device="cuda"))
    w2c = torch.linalg.inv(torch.from_numpy(pr.lookat_c2w(1.2, 60.0, 20.0)).float().cuda())
    imgs = [ru.render_point(v, torch.cat((color, feat), dim=-1), h, h, torch.from_numpy(pr.intrinsics(h)).float().cuda(), w2c, (h, h),
                            2.0 / h * 2.0, 8) for h in (H, H // 2, H // 4)]
    rgb = net(imgs)
    gt = torch.rand(1, 3, H, H, device="cuda")
    loss = cx(rgb, gt) + ((rgb - gt) ** 2).mean()
    loss.backward()
    assert math.isfinite(float(loss))
    for t in [color, feat] + list(net.parameters()):
        assert t.grad is not None and torch.isfinite(t.grad).all() and float(t.grad.abs().sum()) > 0
