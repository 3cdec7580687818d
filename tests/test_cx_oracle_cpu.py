"""CPU: oracle/cx_ref.py (the restatement of the contextual_loss package the GPU tests compare against) pinned against torchvision's
VGG19, an independent loop-form restatement of the loss, autograd's gradcheck, hand cases for the tie rules, and the ctypes mirror of
mi3d_cx_cfg against the header."""
import ctypes
import importlib
import math
import os
import subprocess

import torch
import torch.nn.functional as F

from oracle import cx_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torchvision_features():
    torchvision = importlib.import_module("torchvision")
    torch.manual_seed(0)
    return torchvision.models.vgg19(weights=None).features[:36].eval()


def test_vgg_matches_torchvision():
    feats = _torchvision_features()
    sd = feats.state_dict()
    assert sum(v.numel() for v in sd.values()) == 20_024_384
    names = cx_ref.package_to_torchvision()
    params = {pkg: sd[tv.replace("features.", "")] for pkg, tv in names.items()}
    x = torch.randn(2, 3, 37, 53)
    with torch.no_grad():
        a, b = cx_ref.vgg_features(x, params), feats(x)
    assert a.shape == b.shape == (2, 512, 2, 3)
    assert float((a - b).abs().max()) <= 1e-6 * max(1.0, float(b.abs().max()))


def test_name_maps_cover_every_tensor():
    cl = importlib.import_module("make-it-3d_b200.nerf.contextual_loss")
    sd = _torchvision_features().state_dict()
    names = cx_ref.package_to_torchvision()
    assert sorted(v.replace("features.", "") for v in names.values()) == sorted(sd.keys())
    m = cl.ContextualLoss(device="cpu")
    own = {k for k, _ in m.named_parameters()}
    assert own == set(names)
    assert sum(p.numel() for p in m.parameters()) == 20_024_384
    assert set(m.state_dict()) == set(names) | {"vgg_mean", "vgg_std"}
    for pkg, tv in names.items():
        assert cl.torchvision_name(pkg) == tv and cl.package_name(tv) == pkg


def test_loop_form_agrees_with_vectorised():
    g = torch.Generator().manual_seed(0)
    xf = torch.relu(torch.randn(2, 8, 3, 4, generator=g, dtype=torch.float64))
    yf = torch.relu(torch.randn(2, 8, 3, 4, generator=g, dtype=torch.float64))
    for bw in (0.5, 0.2):
        a = float(cx_ref.cx_from_features(xf, yf, bw))
        b = cx_ref.cx_from_features_loop(xf, yf, bw)
        assert abs(a - b) <= 1e-12 * max(1.0, abs(b)), (a, b)


def test_gradcheck():
    g = torch.Generator().manual_seed(1)
    xf = torch.randn(2, 6, 2, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    yf = torch.randn(2, 6, 2, 3, generator=g, dtype=torch.float64)
    assert torch.autograd.gradcheck(lambda t: cx_ref.cx_from_features(t, yf, 0.5), (xf,), eps=1e-6, atol=1e-7)


def test_identical_features():
    g = torch.Generator().manual_seed(2)
    f = torch.relu(torch.randn(1, 16, 4, 5, generator=g))
    assert abs(float(cx_ref.cx_from_features(f, f.clone())) - (-math.log(1 + 1e-5))) <= 1e-7


def test_tie_rules():
    # two identical y columns: the row min and the cx row are shared, min's gradient goes to the lower index only
    y = torch.tensor([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0]], dtype=torch.float64).T.reshape(1, 2, 1, 3)    # y_0 == y_2
    x = torch.tensor([[1.0, 0.1], [0.2, 1.0], [0.9, 0.3]], dtype=torch.float64).T.reshape(1, 2, 1, 3).requires_grad_(True)
    d = torch.tensor([[1.0, 2.0, 1.0]])
    assert int(torch.min(d, dim=1)[1]) == 0 and int(torch.max(-d, dim=1)[1]) == 0
    loss = cx_ref.cx_from_features(x, y)
    loss.backward()
    assert torch.isfinite(x.grad).all()
    # duplicated x columns: the column max over i goes to the lower i, so only that x position receives the max/mean gradient
    xd = torch.cat([x.detach()[..., :1], x.detach()[..., :1], x.detach()[..., 1:2]], -1).requires_grad_(True)
    yd = torch.cat([x.detach()[..., :1] * 3, y[..., 1:]], -1)
    cx_ref.cx_from_features(xd, yd).backward()
    assert float(xd.grad[..., 1].abs().max()) < float(xd.grad[..., 0].abs().max())


def test_maxpool_ties_to_first_element():
    x = torch.tensor([[[[2.0, 2.0], [2.0, 2.0]]]], requires_grad=True)
    F.max_pool2d(x, 2, 2).sum().backward()
    assert x.grad.flatten().tolist() == [1.0, 0.0, 0.0, 0.0]
    # odd sizes are floored: the last row / column get no gradient
    z = torch.arange(25.0).reshape(1, 1, 5, 5).requires_grad_(True)
    F.max_pool2d(z, 2, 2).sum().backward()
    assert float(z.grad[..., 4, :].abs().sum()) == 0 and float(z.grad[..., :, 4].abs().sum()) == 0


def test_cfg_layout_matches_header(tmp_path):
    cl = importlib.import_module("make-it-3d_b200.nerf.contextual_loss")
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(mi3d_cx_cfg));']
    for f, _ in cl.CxCfg._fields_:
        src.append(f'  printf("{f} %zu\\n", offsetof(mi3d_cx_cfg, {f}));')
    src += ['  return 0;', '}']
    c = tmp_path / "cx_layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "cx_layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cl.CxCfg)
    for f, _ in cl.CxCfg._fields_:
        assert int(out[f]) == getattr(cl.CxCfg, f).offset
