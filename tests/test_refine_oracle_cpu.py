"""CPU checks of the refine loop's pieces: oracle/refine_ref.py against torch's own CPU modules in fp64, the host pose sampler of
nerf/refine.py against the reference's fix_poses rules, and the ctypes mirror of mi3d_adam_segment against the header."""
import ctypes
import importlib
import math
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refine_ref as rr  # noqa: E402

refine = importlib.import_module("make-it-3d_b200.nerf.refine")


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1.0, float(np.abs(b).max()))
    assert float(np.abs(a - b).max()) <= tol * scale, float(np.abs(a - b).max())


def test_image_terms_match_torch_modules():
    g = torch.Generator().manual_seed(0)
    S, ppp = 24, 8
    w = torch.rand(S, S, ppp, generator=g, dtype=torch.float64) * (torch.rand(S, S, 1, generator=g, dtype=torch.float64) > 0.5)
    _close(rr.coverage(w.numpy()), w.sum(-1).numpy())
    dil = rr.dilate(w.sum(-1).numpy())
    ref = torch.nn.MaxPool2d(5, 1, 2)(w.sum(-1)[None, None].expand(1, 3, S, S))
    assert np.array_equal(dil, ref[0, 0].numpy()) and np.array_equal(dil, ref[0, 2].numpy())
    pred = torch.rand(1, 3, S, S, generator=g, dtype=torch.float64, requires_grad=True)
    gt = torch.rand(1, 3, S, S, generator=g, dtype=torch.float64)
    m = (torch.rand(1, 1, S, S, generator=g, dtype=torch.float64) > 0.3).double()
    bg = 1e-3 * (1 - pred * (1 - ref)).sum()
    l1 = 1000 * torch.nn.L1Loss()(pred * m, gt * m)
    (gb,) = torch.autograd.grad(bg, pred)
    (gl,) = torch.autograd.grad(l1, pred)
    v, d = rr.bg_loss(pred.detach().numpy(), dil)
    _close(v, bg.item())
    _close(d, gb.numpy())
    v, d = rr.masked_l1(pred.detach().numpy(), gt.numpy(), m.numpy())
    _close(v, l1.item())
    _close(d, gl.numpy())


def test_regulariser_and_adam_match_torch_optim_over_six_groups():
    """three Adam steps over the reference's six groups (bg_feat without a gradient) with the regulariser in the loss"""
    g = torch.Generator().manual_seed(1)
    pc, pn = 7, 5
    leaves = [torch.rand(pn, 3, generator=g, dtype=torch.float64), torch.rand(pc, 3, generator=g, dtype=torch.float64),
              torch.randn(pn, 16, generator=g, dtype=torch.float64), torch.randn(pc, 16, generator=g, dtype=torch.float64),
              torch.ones(1, 19, 1, 1, dtype=torch.float64), torch.randn(4, 6, generator=g, dtype=torch.float64)]
    leaves = [torch.nn.Parameter(t.clone()) for t in leaves]
    o_n, o_c = leaves[0].detach().clone() + 0.01, leaves[1].detach().clone() - 0.02
    opt = torch.optim.Adam([{"params": [p], "lr": 1e-3} for p in leaves], betas=(0.9, 0.99), eps=1e-15)
    mine = [p.detach().numpy().copy() for p in leaves]
    ms = [np.zeros_like(a) for a in mine]
    vs = [np.zeros_like(a) for a in mine]
    for step in range(1, 4):
        ext = [torch.randn(p.shape, generator=g, dtype=torch.float64) for p in leaves]
        opt.zero_grad()
        reg = torch.nn.MSELoss()(leaves[0], o_n) * 1e3 + torch.nn.MSELoss()(leaves[1], o_c) * 1e5
        loss = reg + sum((p * e).sum() for i, (p, e) in enumerate(zip(leaves, ext)) if i != 4)
        loss.backward()
        val, gc, gn = rr.regulariser(mine[1], o_c.numpy(), mine[0], o_n.numpy())
        _close(val, reg.item())
        opt.step()
        for i in range(6):
            if i == 4:
                continue
            gi = ext[i].numpy() + (gn if i == 0 else gc if i == 1 else 0.0)
            mine[i], ms[i], vs[i] = rr.adam_step(mine[i], gi, ms[i], vs[i], step)
        for i, p in enumerate(leaves):
            _close(mine[i], p.detach().numpy())
        assert leaves[4] not in opt.state and torch.equal(leaves[4].detach(), torch.ones(1, 19, 1, 1, dtype=torch.float64))


def test_pose_sampler_front_rule_and_phi_buckets():
    gen, rnd = torch.Generator().manual_seed(0), random.Random(0)
    front, _, _ = refine.fix_poses(0, gen, rnd)
    buckets = {0: 0, 1: 0, 2: 0, 3: 0, 4: 0}
    edges = [(315, 360), (0, 45), (240, 315), (45, 120), (120, 240)]      # rand > .85, > .7, > .5, > .3, else
    for i in range(400):
        state = rnd.getstate()
        pose, is_front, is_large = refine.fix_poses(i, gen, rnd)
        if i % 4 == 0:
            assert is_front and torch.equal(pose, front)
            continue
        assert not is_front
        r = random.Random()
        r.setstate(state)
        u = r.random()
        k = 0 if u > 0.85 else 1 if u > 0.7 else 2 if u > 0.5 else 3 if u > 0.3 else 4
        buckets[k] += 1
        # recover phi from the camera centre: x = r sin(theta) sin(phi), z = r sin(theta) cos(phi)
        c = pose[:3, 3].double()
        phi = math.degrees(math.atan2(c[0], c[2])) % 360.0
        lo, hi = edges[k]
        assert lo - 1e-3 <= phi <= hi + 1e-3 or (k == 0 and phi < 1e-3), (k, phi)
        assert is_large == (phi <= 45 + 1e-4 or phi >= 315 - 1e-4)
        rad = float(c.norm())
        assert 1 - 1e-5 <= rad <= 1.5 + 1e-5
        # a look-at pose: orthonormal rotation, forward axis toward the origin
        R = pose[:3, :3].double()
        assert torch.allclose(R.T @ R, torch.eye(3, dtype=torch.float64), atol=1e-5)
        assert torch.allclose(R[:, 2], -c / rad, atol=1e-5)
    assert all(n > 0 for n in buckets.values()), buckets
    # the front pose: radius 1, theta = phi = the middle of their ranges (50 and 180 degrees)
    c = front[:3, 3].double()
    assert abs(float(c.norm()) - 1) < 1e-6 and abs(math.degrees(math.acos(float(c[1]))) - 50) < 1e-4
    assert abs(math.degrees(math.atan2(c[0], c[2])) % 360 - 180) < 1e-4


def test_level_intrinsics_are_the_reference_ones():
    focal = 1 / (2 * np.tan(np.deg2rad(20) / 2))
    K = np.array([[focal * 800, 0, 0.5 * 800], [0, focal * 800, 0.5 * 800], [0, 0, 1]])
    for j, w in enumerate((800, 400, 200)):
        want = torch.tensor(np.array([[focal * w, 0, 0.5 * w], [0, focal * w, 0.5 * w], [0, 0, 1]])).float()
        assert torch.equal(refine.level_K(K, j), want)


def test_adam_segment_mirror_matches_the_header(tmp_path):
    L = importlib.import_module("make-it-3d_b200._lib")
    cls = L.AdamSegment
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(mi3d_adam_segment));']
    src += [f'  printf("{f} %zu\\n", offsetof(mi3d_adam_segment, {f}));' for f, _ in cls._fields_]
    src += ['  return 0;', '}']
    c = tmp_path / "seg.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "seg"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f
