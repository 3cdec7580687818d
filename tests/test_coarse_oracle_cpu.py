"""CPU checks of the coarse loop's losses: oracle/coarse_ref.py against torch CPU autograd of the reference expressions
(nerf/utils.py:491-493, :519-533, :551-556, torchmetrics' PearsonCorrCoef formula), including non-finite depth, weights at the
clamp bounds, a non-square render and an empty mask; and the host-side checks of nerf/coarse.py."""
import argparse
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import coarse_ref as cr  # noqa: E402

coarse = importlib.import_module("make-it-3d_b200.nerf.coarse")
_lib = importlib.import_module("make-it-3d_b200._lib")


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def torch_pearson(x, y):
    """torchmetrics' PearsonCorrCoef for one batch (update + compute), in fp64"""
    n = x.shape[0]
    mx, my = x.mean(), y.mean()
    var_x, var_y = x.var() * (n - 1), y.var() * (n - 1)
    corr = ((x - mx) * (y - my)).sum()
    var_x, var_y, corr = var_x / (n - 1), var_y / (n - 1), corr / (n - 1)
    return torch.clamp(corr / (var_x * var_y).sqrt(), -1.0, 1.0)


def reference_terms(image, depth, ws, h, w, ref, bg, prior, depth_mask, front):
    """the reference's expressions on torch CPU: fp32 render outputs, fp64 prior, Pearson in fp64 as the [mask] compaction gives it"""
    pred_rgb = image.reshape(1, h, w, 3).permute(0, 3, 1, 2).contiguous()
    pred_depth = depth.reshape(1, h, w, 1).permute(0, 3, 1, 2).contiguous()
    pred_ws = ws.reshape(1, 1, h, w)
    bg_img = bg.expand(1, 512, 512, 3).permute(0, 3, 1, 2).contiguous()
    gt_rgb = ref[:, :3, :, :] * ref[:, 3:, :, :] + bg_img * (1 - ref[:, 3:, :, :])
    loss_opacity = (pred_ws ** 2).mean()
    alphas = pred_ws.clamp(1e-5, 1 - 1e-5)
    loss_entropy = (- alphas * torch.log2(alphas) - (1 - alphas) * torch.log2(1 - alphas)).mean()
    pred_rgb = F.interpolate(pred_rgb, (512, 512), mode='bilinear', align_corners=True)
    pred_depth = F.interpolate(pred_depth, (512, 512), mode='bilinear', align_corners=True)
    out = [loss_opacity, loss_entropy]
    if front:
        out.append(torch.nn.L1Loss()(pred_rgb, gt_rgb))
        x = torch.nan_to_num(pred_depth.squeeze()).reshape(-1)
        m = (~depth_mask).reshape(-1) == 1
        out.append(torch_pearson(x[m].double(), prior.reshape(-1)[m]))
    return out, pred_rgb, gt_rgb


def _case(h, w, seed, nonfinite=False, at_bounds=False, mask_kind="blob"):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(h * w, 3, generator=g)
    depth = 1 + torch.rand(h * w, generator=g) * 2
    ws = torch.rand(h * w, generator=g)
    if at_bounds:
        ws[::7] = 1e-5
        ws[3::7] = 1 - 1e-5
        ws[5::11] = 0.0
        ws[6::11] = 1.0
    if nonfinite:
        # NaN inside the object (nan_to_num makes it 0 there); +-inf in the background, outside the depth term's mask
        depth[(h // 2) * w + w // 2] = float("nan")
        depth[w - 1] = float("inf")
        depth[2 * w + 1] = -float("inf")
    ref = torch.rand(1, 4, 512, 512, generator=g)
    bg = torch.rand(3, generator=g)
    yy, xx = torch.meshgrid(torch.arange(512), torch.arange(512), indexing="ij")
    if mask_kind == "blob":
        obj = ((yy - 250) ** 2 + (xx - 270) ** 2) < 150 ** 2
    elif mask_kind == "empty":
        obj = torch.zeros(512, 512, dtype=torch.bool)
    else:                                                   # one pixel
        obj = (yy == 100) & (xx == 200)
    depth_mask = ~obj
    prior = torch.rand(512, 512, generator=g, dtype=torch.float64) * obj + (yy.double() / 512) * obj
    return image, depth, ws, ref, bg, prior, depth_mask


CASES = [dict(h=32, w=32, seed=0), dict(h=24, w=40, seed=1), dict(h=17, w=9, seed=2, nonfinite=True),
         dict(h=32, w=32, seed=3, at_bounds=True), dict(h=16, w=20, seed=4, mask_kind="empty"),
         dict(h=16, w=16, seed=5, mask_kind="one")]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_oracle_matches_torch_autograd_of_the_reference(case):
    h, w = case["h"], case["w"]
    image, depth, ws, ref, bg, prior, depth_mask = _case(**case)
    mask_u8 = (~depth_mask).to(torch.uint8).numpy()
    gen = torch.Generator().manual_seed(9)
    g_terms = torch.tensor([0.7, -1.3, 2.1, -0.9], dtype=torch.float64)
    g_pred = torch.randn(1, 3, 512, 512, generator=gen, dtype=torch.float64) * 1e-3
    for front in (True, False):
        ti, td, tw = (t.clone().requires_grad_() for t in (image, depth, ws))
        terms, pred512, gt512 = reference_terms(ti, td, tw, h, w, ref, bg, prior, depth_mask, front)
        args = (image.numpy(), depth.numpy(), ws.numpy(), h, w, ref.numpy(), bg.numpy(), prior.numpy(), mask_u8, front)
        o_terms, o_pred, o_gt = cr.forward(*args)
        assert float(np.abs(o_pred - pred512.detach().double().numpy()).max()) <= 1e-6
        assert np.array_equal(o_gt, gt512.double().numpy())
        for k, t in enumerate(terms):
            want = t.item()
            if np.isnan(want):
                assert np.isnan(o_terms[k]), k
            else:
                # the coefficient lies in [-1, 1]: held absolutely (the fp32 upsample's rounding moves it by ~1e-9)
                assert abs(o_terms[k] - want) <= 1e-6 * (1.0 if k == 3 else abs(want)), (k, o_terms[k], want)
        if not front:
            assert o_terms[2] == 0.0 and o_terms[3] == 0.0
        total = sum(g * t.double() for g, t in zip(g_terms, terms) if not torch.isnan(t))
        total = total + (g_pred * pred512.double()).sum()
        gi_t, gd_t, gw_t = torch.autograd.grad(total, (ti, td, tw), allow_unused=True)
        gi, gd, gw = cr.backward(*args, g_terms.numpy(), g_pred.numpy())
        assert _rel(gi, gi_t) <= 1e-5
        assert _rel(gw, gw_t) <= 1e-5
        if front and gd_t is not None and float(gd_t.abs().max()) > 0:
            assert _rel(gd, gd_t) <= 1e-5
        else:
            assert float(np.abs(gd).max()) == 0.0
        if front and case.get("nonfinite"):
            assert np.isfinite(gd).all()


def test_pearson_with_fewer_than_two_pixels_is_nan_and_passes_no_gradient():
    x, y = np.arange(10.0), np.arange(10.0) ** 2
    for m in (np.zeros(10, bool), np.eye(1, 10, 4, dtype=bool)[0]):
        r, g = cr.pearson(x, y, m)
        assert np.isnan(r) and not g.any()
    r, g = cr.pearson(x, 3 * x + 1, np.ones(10, bool))
    assert abs(r - 1.0) <= 1e-15


def test_upsample_adjoint_is_the_transpose():
    g = np.random.default_rng(0)
    for h, w in ((2, 2), (7, 13), (128, 128), (600, 520)):
        x, y = g.standard_normal((h, w)), g.standard_normal((512, 512))
        lhs = float((cr.upsample(x.astype(np.float32)) * y).sum())
        rhs = float((x.astype(np.float32).astype(np.float64) * cr.upsample_adjoint(y, h, w)).sum())
        assert abs(lhs - rhs) <= 1e-9 * max(abs(lhs), 1.0)


def test_coarse_step_refuses_fp16_cpu_tensors_and_other_sizes():
    opt = argparse.Namespace(fp16=True)
    with pytest.raises(_lib.Mi3dError):
        coarse.CoarseStep(None, None, None, None, opt, torch.zeros(1, 4, 512, 512), torch.zeros(512, 512, dtype=torch.float64),
                          torch.zeros(512, 512, dtype=torch.bool), [None, None], torch.zeros(2, 77, dtype=torch.long))
    opt.fp16 = False
    with pytest.raises(_lib.Mi3dError, match="CUDA"):
        coarse.CoarseStep(None, None, None, None, opt, torch.zeros(1, 4, 512, 512), torch.zeros(512, 512, dtype=torch.float64),
                          torch.zeros(512, 512, dtype=torch.bool), [None, None], torch.zeros(2, 77, dtype=torch.long))
    with pytest.raises(_lib.Mi3dError):
        coarse.coarse_losses(torch.zeros(16, 3), torch.zeros(16), torch.zeros(16), 4, 4, torch.zeros(1, 4, 512, 512), torch.zeros(3),
                             torch.zeros(512, 512, dtype=torch.float64), torch.zeros(512, 512, dtype=torch.uint8), True)


def test_shading_schedule():
    assert coarse.pick_shading(5, False, 1000) == ("albedo", 1.0)
    assert coarse.pick_shading(5000, True, 1000) == ("albedo", 1.0)
    seen = {coarse.pick_shading(5000, False, 1000)[0] for _ in range(200)}
    assert seen == {"albedo", "textureless", "lambertian"}


def test_workspace_query_is_pure_host(mi3d):
    import ctypes
    lib = mi3d.lib()
    n = lib.mi3d_coarse_losses_workspace_bytes(ctypes.c_uint32(128), ctypes.c_uint32(128))
    assert n >= 512 * 512 * 4
    assert lib.mi3d_coarse_losses_workspace_bytes(ctypes.c_uint32(1), ctypes.c_uint32(128)) == 0
