"""`optimizer.Adam` (csrc/adam.cu) on the GPU against `torch.nn.utils.clip_grad_norm_(params, 10)` + `torch.optim.Adam(..., betas=(0.9,
0.99), eps=1e-15)` (foreach path), at the shapes of a real `NeRFNetwork(opt).get_params(1e-3)` with about 1 % non-zero table
gradients: 1 fp32 ulp with the clip inactive or off, rel-L2 1e-6 with it active (the norm is summed in another order), skipped
parameters, checkpoint interchange both ways under a LambdaLR, no host synchronisation, and the coarse loop (`CoarseStep`,
`train_one_epoch`) with Adam against the reference iteration."""
import argparse
import importlib
import io
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_coarse_gpu import BRANCHES, _rel, build_scene, eager_train_step, make_model, make_opt, view  # noqa: E402

pytestmark = pytest.mark.gpu

co = importlib.import_module("make-it-3d_b200.nerf.coarse")
nt = importlib.import_module("make-it-3d_b200.nerf.network_tcnn")
Adam = importlib.import_module("make-it-3d_b200.optimizer").Adam

BETAS, EPS, CLIP = (0.9, 0.99), 1e-15, 10.0


def _shapes():
    torch.manual_seed(0)
    m = nt.NeRFNetwork(make_opt())
    return [[p.detach().clone() for p in g['params']] for g in m.get_params(1e-3)]


SHAPES = None


def _tensors():
    global SHAPES
    if SHAPES is None:
        SHAPES = _shapes()
    return SHAPES


def make_arms(clip):
    """(mine, torch) parameter lists (two groups: encoder at 10 lr, MLP at lr) and their optimisers"""
    groups = _tensors()
    pa = [[torch.nn.Parameter(t.clone().cuda()) for t in g] for g in groups]
    pb = [[torch.nn.Parameter(t.clone().cuda()) for t in g] for g in groups]
    mine = Adam([{'params': pa[0], 'lr': 1e-2}, {'params': pa[1], 'lr': 1e-3}], betas=BETAS, eps=EPS, clip_grad_norm=clip)
    ref = torch.optim.Adam([{'params': pb[0], 'lr': 1e-2}, {'params': pb[1], 'lr': 1e-3}], betas=BETAS, eps=EPS)
    return sum(pa, []), mine, sum(pb, []), ref


def grads(params, seed, scale):
    """table gradients with about 1 % non-zero entries, dense MLP gradients"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for p in params:
        if p.numel() > 1 << 20:
            gr = torch.zeros(p.numel())
            idx = torch.randperm(p.numel(), generator=g)[:p.numel() // 100]      # distinct: the scatter is then deterministic
            gr[idx] = torch.randn(idx.numel(), generator=g) * scale
            out.append(gr.view_as(p).cuda())
        else:
            out.append((torch.randn(p.shape, generator=g) * scale * 0.1).cuda())
    return out


def set_grads(params, gs):
    for p, g in zip(params, gs):
        p.grad = g.clone()


def torch_step(params, opt, clip):
    if clip:
        torch.nn.utils.clip_grad_norm_(params, clip)
    opt.step()


def assert_ulp(a, b, what):
    b = b.detach()
    ulp = (torch.nextafter(b, torch.full_like(b, float("inf"))) - b).abs()
    assert bool(((a.detach() - b).abs() <= ulp).all()), (what, float(((a.detach() - b).abs() / ulp).max()))


def states(opt, params):
    return [(opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], opt.state[p]["step"]) for p in params]


@pytest.mark.parametrize("clip", [CLIP, 0.0])
def test_within_one_ulp_of_torch_with_the_clip_inactive_or_off(clip):
    pa, mine, pb, ref = make_arms(clip)
    for step in range(3):
        gs = grads(pa, 10 + step, 1e-3)
        set_grads(pa, gs)
        set_grads(pb, gs)
        mine.step()
        torch_step(pb, ref, clip)
        norm = torch.stack([g.norm() for g in gs]).norm()
        assert float(norm) < CLIP
        for k, (a, b) in enumerate(zip(pa, pb)):
            assert_ulp(a, b, f"param {k} step {step}")
            (ma, va, sa), (mb, vb, sb) = states(mine, [a])[0], states(ref, [b])[0]
            assert_ulp(ma, mb, f"exp_avg {k}")
            assert_ulp(va, vb, f"exp_avg_sq {k}")
            assert sa.device.type == "cpu" and sa.dtype == torch.float32 and float(sa) == float(sb) == step + 1
            assert torch.equal(a.grad, b.grad)


def test_active_clip_matches_torch_to_rel_l2_1e6():
    pa, mine, pb, ref = make_arms(CLIP)
    p0 = [p.detach().clone() for p in pa]
    for step in range(3):
        gs = grads(pa, 20 + step, 1.0)
        assert float(torch.stack([g.norm() for g in gs]).norm()) > 10 * CLIP
        set_grads(pa, gs)
        set_grads(pb, gs)
        mine.step()
        torch_step(pb, ref, CLIP)
        for k, (a, b, z) in enumerate(zip(pa, pb, p0)):
            assert _rel(a.grad, b.grad) <= 1e-6, (k, _rel(a.grad, b.grad))
            assert _rel(a.detach() - z, b.detach() - z) <= 1e-6, (k, step)
            (ma, va, _), (mb, vb, _) = states(mine, [a])[0], states(ref, [b])[0]
            assert _rel(ma, mb) <= 1e-6 and _rel(va, vb) <= 1e-6, k


def test_a_parameter_without_grad_is_skipped():
    pa, mine, _, _ = make_arms(CLIP)
    never = pa[-1]
    for p, g in zip(pa[:-1], grads(pa[:-1], 30, 1e-3)):
        p.grad = g
    v0 = never.detach().clone()
    mine.step()
    assert len(mine.state[never]) == 0 and torch.equal(never.detach(), v0)
    later = pa[1]                                   # stepped once, then left without a gradient
    saved = (later.detach().clone(), mine.state[later]["exp_avg"].clone(), mine.state[later]["exp_avg_sq"].clone())
    for p, g in zip(pa, grads(pa, 31, 1e-3)):
        p.grad = g
    later.grad = None
    mine.step()
    assert torch.equal(later.detach(), saved[0])
    assert torch.equal(mine.state[later]["exp_avg"], saved[1]) and torch.equal(mine.state[later]["exp_avg_sq"], saved[2])
    assert float(mine.state[later]["step"]) == 1.0 and float(mine.state[pa[0]]["step"]) == 2.0
    assert float(mine.state[never]["step"]) == 1.0


def _with_sched(opt):
    return torch.optim.lr_scheduler.LambdaLR(opt, lambda it: 1.0 / (1.0 + it))


def _roundtrip(opt, sched):
    buf = io.BytesIO()
    torch.save({'optimizer': opt.state_dict(), 'lr_scheduler': sched.state_dict()}, buf)
    buf.seek(0)
    return torch.load(buf)


@pytest.mark.parametrize("first", ["torch", "mine"])
def test_checkpoints_interchange_with_torch_adam(first):
    k = 3
    pa, mine, pb, ref = make_arms(CLIP)
    pc = [torch.nn.Parameter(p.detach().clone()) for p in pb]
    full = torch.optim.Adam([{'params': pc[:1], 'lr': 1e-2}, {'params': pc[1:], 'lr': 1e-3}], betas=BETAS, eps=EPS)
    s_full = _with_sched(full)
    gs = [grads(pa, 40 + i, 1.0) for i in range(k + 1)]
    for i in range(k + 1):                              # the uninterrupted torch run
        set_grads(pc, gs[i])
        torch_step(pc, full, CLIP)
        s_full.step()
    if first == "torch":
        a_params, a_opt, b_params, b_cls = pb, ref, pa, "mine"
    else:
        a_params, a_opt, b_params, b_cls = pa, mine, pb, "torch"
    s_a = _with_sched(a_opt)
    for i in range(k):
        set_grads(a_params, gs[i])
        if a_opt is mine:
            mine.step()
        else:
            torch_step(a_params, a_opt, CLIP)
        s_a.step()
    ck = _roundtrip(a_opt, s_a)
    with torch.no_grad():
        for p, q in zip(b_params, a_params):
            p.copy_(q)
    groups = [{'params': b_params[:1], 'lr': 1e-2}, {'params': b_params[1:], 'lr': 1e-3}]
    b_opt = Adam(groups, betas=BETAS, eps=EPS, clip_grad_norm=CLIP) if b_cls == "mine" else torch.optim.Adam(groups, betas=BETAS, eps=EPS)
    s_b = _with_sched(b_opt)
    b_opt.load_state_dict(ck['optimizer'])
    s_b.load_state_dict(ck['lr_scheduler'])
    set_grads(b_params, gs[k])
    if b_cls == "mine":
        b_opt.step()
    else:
        torch_step(b_params, b_opt, CLIP)
    s_b.step()
    assert [g['lr'] for g in b_opt.param_groups] == [g['lr'] for g in full.param_groups]
    p0 = _tensors()
    for j, (a, b, z) in enumerate(zip(b_params, pc, sum(p0, []))):
        z = z.cuda()
        assert _rel(a.detach() - z, b.detach() - z) <= 1e-6, j
        (ma, va, sa), (mb, vb, sb) = states(b_opt, [a])[0], states(full, [b])[0]
        assert _rel(ma, mb) <= 1e-6 and _rel(va, vb) <= 1e-6, j
        assert sa.device.type == "cpu" and float(sa) == float(sb) == k + 1


def _run(n_steps, seed0):
    pa, mine, _, _ = make_arms(CLIP)
    for i in range(n_steps):
        set_grads(pa, grads(pa, seed0 + i, 1.0))
        mine.step()
    return pa, mine


def test_step_never_synchronises_and_repeats_bitwise():
    pa, mine = _run(1, 50)                              # warm-up: state and scratch allocation
    gs = [grads(pa, 51 + i, 1.0) for i in range(2)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for g in gs:
            for p, gi in zip(pa, g):
                p.grad.copy_(gi)
            mine.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    pb, other = _run(3, 50)
    for a, b in zip(pa, pb):
        assert torch.equal(a.detach(), b.detach()) and torch.equal(a.grad, b.grad)
        assert torch.equal(mine.state[a]["exp_avg"], other.state[b]["exp_avg"])
        assert torch.equal(mine.state[a]["exp_avg_sq"], other.state[b]["exp_avg_sq"])


# ---- the coarse loop with Adam ----

@pytest.fixture(scope="module")
def scene():
    return build_scene()


def make_adam(model):
    return Adam(model.get_params(1e-3), betas=BETAS, eps=EPS)          # main.py:133-134; CoarseStep sets the clip to 10


class ClipThenAdam:
    """the reference's `--optim adam` update: nn.utils.clip_grad_norm(model.parameters(), 10) (utils.py:984), then torch's Adam"""

    def __init__(self, model):
        self.model = model
        self.opt = torch.optim.Adam(model.get_params(1e-3), betas=BETAS, eps=EPS)

    def zero_grad(self):
        self.opt.zero_grad()

    def step(self):
        torch.nn.utils.clip_grad_norm_(self.model.parameters(), CLIP)
        self.opt.step()


@pytest.mark.parametrize("branch", ["front", "sds", "denoise"])
def test_one_coarse_iteration_with_adam_matches_the_reference_step(scene, branch):
    global_step, vkw, t, shading = BRANCHES[branch]
    opt = make_opt()
    model_a = make_model(opt)
    adam = make_adam(model_a)
    cs = co.CoarseStep(model_a, scene["guidance"], scene["clip"], adam, opt, scene["ref"], scene["prior"], scene["depth_mask"],
                       scene["text_z"], scene["tokens"])
    assert adam.clip_grad_norm == CLIP
    model_b = make_model(opt)
    data = view(**vkw)
    bg = torch.tensor([0.3, 0.6, 0.2], device="cuda")
    light = torch.tensor([0.0, 0.6, 0.8], device="cuda")
    g = torch.Generator().manual_seed(5)
    noise, eps = torch.randn(1, 4, 32, 32, generator=g).cuda(), torch.randn(1, 4, 32, 32, generator=g).cuda()
    torch.manual_seed(123)
    res = cs.step(data, global_step, shading=shading, bg_color=bg, t=t, noise=noise, eps_posterior=eps, light_d=light)
    grads_a = {n: p.grad.clone() for n, p in cs.model.named_parameters()}      # clipped in place by Adam's step
    torch.manual_seed(123)
    loss_b, grads_b = eager_train_step(model_b, ClipThenAdam(model_b), opt, scene, data, global_step, shading, bg, light, t=t,
                                       noise=noise, eps_posterior=eps)
    torch.cuda.synchronize()
    # the tolerances of test_coarse_gpu.py::test_one_iteration_matches_the_reference_step
    tol, tol_grad = (1e-5, 1e-4) if vkw.get("front") else (1e-4, 3e-3)
    assert abs(res["loss"].item() - loss_b.item()) <= tol * abs(loss_b.item()), (res["loss"].item(), loss_b.item())
    for n, gb in grads_b.items():
        if n == "encoder.params":
            continue
        assert _rel(grads_a[n], gb) <= tol_grad, (n, _rel(grads_a[n], gb))
    table_a, table_b = grads_a["encoder.params"], grads_b["encoder.params"]
    sample = torch.randint(0, table_b.numel(), (1 << 18,), generator=torch.Generator().manual_seed(0)).cuda()
    assert float(table_b[sample].abs().max()) > 0
    assert _rel(table_a[sample], table_b[sample]) <= max(5e-4, tol_grad), _rel(table_a[sample], table_b[sample])
    for (n, pa), (_, pb) in zip(cs.model.named_parameters(), model_b.named_parameters()):
        gb = grads_b[n]
        sel = gb.abs() > 1e-2 * gb.abs().max()
        assert float((pa.detach() - pb.detach())[sel].abs().max()) <= 1e-6, (n, float((pa.detach() - pb.detach())[sel].abs().max()))


def test_coarse_step_refuses_another_clip(scene):
    opt = make_opt()
    model = make_model(opt)
    adam = Adam(model.get_params(1e-3), betas=BETAS, eps=EPS, clip_grad_norm=5.0)
    with pytest.raises(co.L.Mi3dError, match="clip_grad_norm"):
        co.CoarseStep(model, scene["guidance"], scene["clip"], adam, opt, scene["ref"], scene["prior"], scene["depth_mask"],
                      scene["text_z"], scene["tokens"])


def test_train_one_epoch_with_adam_and_lambdalr(scene, tmp_path):
    opt = make_opt(diff_iters=4, albedo_iters=2, update_extra_interval=4)
    model = make_model(opt)
    adam = make_adam(model)
    sched = torch.optim.lr_scheduler.LambdaLR(adam, lambda it: 0.1 ** min(it / 8, 1))
    trainer = argparse.Namespace(model=model, guidance=scene["guidance"], clip_model=scene["clip"], optimizer=adam, opt=opt,
                                 ref_imgs=scene["ref"], depth_prediction=scene["prior"], depth_mask=scene["depth_mask"],
                                 text_z=scene["text_z"], clip_text_tokens=scene["tokens"], global_step=0, epoch=1, workspace=str(tmp_path),
                                 img_path=str(tmp_path / "images"), log=lambda *a: None, stats={"loss": []}, lr_scheduler=sched,
                                 scheduler_update_every_step=True, fp16=False, ema=None, world_size=1)
    loader = [view(0.0 if i % 4 == 0 else 45.0 * i, front=i % 4 == 0, large=i == 5) for i in range(8)]
    p0 = [p.detach().clone() for p in model.parameters()]
    co.train_one_epoch(trainer, loader)
    assert trainer.global_step == 8 and sched.last_epoch == 8
    assert len(trainer.stats["loss"]) == 1 and np.isfinite(trainer.stats["loss"][0])
    assert adam.clip_grad_norm == CLIP
    assert [g['lr'] for g in adam.param_groups] == pytest.approx([1e-3, 1e-4])
    assert all(bool(torch.isfinite(p).all()) and not torch.equal(p.detach(), q) for p, q in zip(model.parameters(), p0))
    # the finished state dict loads into torch.optim.Adam and steps there
    buf = io.BytesIO()
    torch.save(adam.state_dict(), buf)
    buf.seek(0)
    twin = make_model(opt)
    ref = torch.optim.Adam(twin.get_params(1e-3), betas=BETAS, eps=EPS)
    ref.load_state_dict(torch.load(buf))
    for p, q in zip(model.parameters(), twin.parameters()):
        st = ref.state[q]
        assert float(st["step"]) == 8.0 and st["step"].device.type == "cpu"
        assert torch.equal(st["exp_avg"], adam.state[p]["exp_avg"]) and torch.equal(st["exp_avg_sq"], adam.state[p]["exp_avg_sq"])
        q.grad = torch.zeros_like(q)
    ref.step()
