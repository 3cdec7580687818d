"""`Adan` with the reference's constructor (optimizer.py:22-96; main.py:132 builds it as
Adan(model.get_params(5 * lr), eps=1e-8, weight_decay=2e-5, max_grad_norm=5.0, foreach=False)) on libmi3d.so: SURVEY.md 8f-1.

One `step()` = Trainer's `nn.utils.clip_grad_norm(model.parameters(), max_norm)` (nerf/utils.py:984; pass clip_grad_norm=10 instead
of calling it separately) + the reference's Adan.step() (global-norm clip 5.0, _single_tensor_adan), as
    one deterministic sum-of-squares pass  ->  [all-reduce of that scalar]  ->  one fused elementwise kernel per tensor
with the norm, both clip factors and every state update on the device (the reference syncs the host with .item() twice).

Multi-GPU (`group=` / an initialised default process group with world_size > 1), fused with the gradient collective:
    big tensors (the 48.8 MB hash table): reduce-scatter(SUM) of the per-rank gradients -> each rank updates its 1/G shard of
        (param, exp_avg, exp_avg_sq, exp_avg_diff, neg_pre_grad) -> all-gather of the updated parameter shards.
        Optimizer state and update math are sharded G ways; the wire carries (G-1)/G * 48.8 MB twice, like the all-reduce it replaces.
    small tensors (the 6 MLP tensors, 26 KB): all-reduce(SUM), identical replicated update on every rank.
Call it INSTEAD of parallel.GradientAllReduce + a separate optimizer step.  The result equals the single-process reference update on
the summed gradients (tests/test_adan_gpu.py, tests/golden/adan.npz recorded from the reference's optimizer.py).

`Adam`: torch.optim.Adam for `--optim adam|adamw` (main.py:133-134), single-GPU, with the same clip folded in (csrc/adam.cu).
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import _lib as L

SHARD_MIN_NUMEL = 1 << 20


class Adan(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.98, 0.92, 0.99), eps=1e-8, weight_decay=0.0, max_grad_norm=0.0, no_prox=False,
                 foreach=False, clip_grad_norm=0.0, group=None):
        if not 0.0 <= max_grad_norm or not 0.0 <= lr or not 0.0 <= eps or not all(0.0 <= b < 1.0 for b in betas):
            raise ValueError("invalid Adan hyper-parameter")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, max_grad_norm=max_grad_norm, no_prox=no_prox, foreach=foreach)
        super().__init__(params, defaults)
        self.clip_grad_norm = float(clip_grad_norm)
        self.group = group
        self._scratch = {}

    # ---- helpers ---------------------------------------------------------------------------------------------------------------
    def _world(self):
        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size(self.group), dist.get_rank(self.group)
        return 1, 0

    def _dev_scratch(self, device):
        key = str(device)
        if key not in self._scratch:
            self._scratch[key] = dict(ws=torch.empty(L.lib().mi3d_sumsq_workspace_bytes(), dtype=torch.uint8, device=device),
                                      sumsq=torch.zeros(1, dtype=torch.float32, device=device))
        return self._scratch[key]

    def _state_for(self, p, numel):
        st = self.state[p]
        if len(st) == 0:
            z = lambda: torch.zeros(numel, dtype=torch.float32, device=p.device)
            st["exp_avg"], st["exp_avg_sq"], st["exp_avg_diff"], st["neg_pre_grad"] = z(), z(), z(), z()
            st["has_prev"] = False
        return st

    @torch.no_grad()
    def restart_opt(self):
        """optimizer.py:85-100: zero the moments, restart the step count"""
        for group in self.param_groups:
            group["step"] = 0
            for p in group["params"]:
                st = self.state.get(p)
                if st:
                    for k in ("exp_avg", "exp_avg_sq", "exp_avg_diff"):
                        st[k].zero_()

    # ---- the step ----------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = L.lib()
        world, rank = self._world()
        items = []          # (group, param, grad_flat (shard or whole), param_flat (shard or whole), sharded?, shard slice)
        device = None
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                L.require_cuda(p, p.grad)
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise L.Mi3dError("Adan: parameters must be contiguous fp32")
                device = p.device
                g = L.f32c(p.grad).view(-1)
                sharded = world > 1 and p.numel() >= SHARD_MIN_NUMEL and p.numel() % (4 * world) == 0
                if sharded:
                    n = p.numel() // world
                    gs = torch.empty(n, dtype=torch.float32, device=device)
                    dist.reduce_scatter_tensor(gs, g, op=dist.ReduceOp.SUM, group=self.group)
                    items.append((group, p, gs, p.data.view(-1)[rank * n:(rank + 1) * n], True))
                else:
                    if world > 1:
                        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
                    items.append((group, p, g, p.data.view(-1), False))
        if not items:
            return loss
        sc = self._dev_scratch(device)
        need_norm = self.defaults["max_grad_norm"] > 0 or self.clip_grad_norm > 0
        if need_norm:
            # ||g||^2 over ALL parameters: shards are summed over ranks, replicated tensors are counted once
            first = True
            for _, _, g, _, sharded in items:
                if sharded:
                    L.check(lib.mi3d_sumsq(L.ptr(g), C.c_uint64(g.numel()), L.ptr(sc["sumsq"]), C.c_int(0 if first else 1), L.ptr(sc["ws"]), L.stream()), "sumsq")
                    first = False
            if first:
                sc["sumsq"].zero_()
            if world > 1:
                dist.all_reduce(sc["sumsq"], op=dist.ReduceOp.SUM, group=self.group)
            for _, _, g, _, sharded in items:
                if not sharded:
                    L.check(lib.mi3d_sumsq(L.ptr(g), C.c_uint64(g.numel()), L.ptr(sc["sumsq"]), C.c_int(1), L.ptr(sc["ws"]), L.stream()), "sumsq")
        stepped = set()
        for group, p, g, pf, sharded in items:
            if id(group) not in stepped:
                group["step"] = group.get("step", 0) + 1              # optimizer.py:140-143
                stepped.add(id(group))
            st = self._state_for(p, g.numel())
            cfg = L.AdanCfg()
            cfg.lr = group["lr"]; cfg.beta1, cfg.beta2, cfg.beta3 = group["betas"]; cfg.eps = group["eps"]; cfg.weight_decay = group["weight_decay"]
            cfg.max_grad_norm = self.defaults["max_grad_norm"]; cfg.clip_grad_norm = self.clip_grad_norm; cfg.no_prox = 1 if group["no_prox"] else 0
            cfg.step = group["step"]; cfg.reset_prev = 0 if st["has_prev"] else 1
            L.check(lib.mi3d_adan_step(L.ptr(pf), L.ptr(g), L.ptr(st["exp_avg"]), L.ptr(st["exp_avg_sq"]), L.ptr(st["exp_avg_diff"]), L.ptr(st["neg_pre_grad"]),
                                       C.c_uint64(g.numel()), L.ptr(sc["sumsq"]) if need_norm else C.c_void_p(0), C.byref(cfg), L.stream()), "adan_step")
            st["has_prev"] = True
            if sharded:
                dist.all_gather_into_tensor(p.data.view(-1), pf.clone(), group=self.group)
            elif g.data_ptr() != p.grad.data_ptr():
                p.grad.copy_(g.view_as(p.grad))
        return loss


class Adam(torch.optim.Optimizer):
    """`torch.optim.Adam` for `--optim adam|adamw` (main.py:133-134: Adam(model.get_params(opt.lr), betas=(0.9, 0.99), eps=1e-15)) on
    libmi3d.so, with the Trainer's `nn.utils.clip_grad_norm(model.parameters(), max_norm)` (nerf/utils.py:984) folded in when
    clip_grad_norm > 0.

    One `step()` = one deterministic sum-of-squares pass per tensor into a device scalar (mi3d_sumsq, only when clipping), then one
    elementwise launch per tensor (mi3d_adam_step): clip, then torch's foreach Adam in its operation order.  The host never
    synchronises.  Parameter groups, `group['lr']` (read every step, so lr schedulers work) and the per-parameter state (`step` a
    CPU fp32 scalar tensor, `exp_avg`, `exp_avg_sq`) are torch's, so state dicts interchange with `torch.optim.Adam` both ways.
    Parameters whose `.grad` is None are skipped, as torch skips them.  Refused with Mi3dError: weight decay, amsgrad, maximize,
    capturable, differentiable, fused=True, parameters that are not contiguous fp32 CUDA tensors, and a process group of more than
    one rank."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None, maximize=False,
                 capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False, clip_grad_norm=0.0):
        if not 0.0 <= lr or not 0.0 <= eps or not all(0.0 <= b < 1.0 for b in betas) or not 0.0 <= weight_decay:
            raise ValueError("invalid Adam hyper-parameter")
        if not 0.0 <= clip_grad_norm:
            raise ValueError(f"invalid clip_grad_norm: {clip_grad_norm}")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize, foreach=foreach,
                        capturable=capturable, differentiable=differentiable, fused=fused, decoupled_weight_decay=decoupled_weight_decay)
        _adam_check_world()
        super().__init__(params, defaults)
        self.clip_grad_norm = float(clip_grad_norm)
        self._scratch = {}

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        _adam_check_group(group)
        for p in group["params"]:
            _adam_check_param(p)

    def _dev_scratch(self, device):
        key = str(device)
        if key not in self._scratch:
            self._scratch[key] = dict(ws=torch.empty(L.lib().mi3d_sumsq_workspace_bytes(), dtype=torch.uint8, device=device),
                                      sumsq=torch.zeros(1, dtype=torch.float32, device=device))
        return self._scratch[key]

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        _adam_check_world()
        items = []          # (group, param, contiguous fp32 grad)
        for group in self.param_groups:
            _adam_check_group(group)
            for p in group["params"]:
                if p.grad is None:
                    continue
                _adam_check_param(p)
                L.require_cuda(p.grad)
                items.append((group, p, L.f32c(p.grad)))
        if not items:
            return loss
        lib = L.lib()
        devices = {p.device for _, p, _ in items}
        if len(devices) != 1:
            raise L.Mi3dError("Adam: all parameters must be on one GPU")
        sumsq = None
        if self.clip_grad_norm > 0:
            sc = self._dev_scratch(items[0][1].device)
            sumsq = sc["sumsq"]
            for k, (_, _, g) in enumerate(items):
                L.check(lib.mi3d_sumsq(L.ptr(g), C.c_uint64(g.numel()), L.ptr(sumsq), C.c_int(1 if k else 0), L.ptr(sc["ws"]), L.stream()),
                        "sumsq")
        for group, p, g in items:
            st = self.state[p]
            if len(st) == 0:                                              # torch's Adam._init_group
                st["step"] = torch.tensor(0.0, dtype=torch.float32)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            if st["step"].is_cuda:
                raise L.Mi3dError("Adam: state['step'] must be a CPU tensor (a capturable / fused state dict was loaded)")
            st["step"] += 1                                               # CPU tensor: no synchronisation
            cfg = L.AdamCfg()
            cfg.lr = float(group["lr"]); cfg.beta1, cfg.beta2 = (float(b) for b in group["betas"]); cfg.eps = float(group["eps"])
            cfg.step = int(st["step"].item()); cfg.clip_grad_norm = self.clip_grad_norm
            L.check(lib.mi3d_adam_step(L.ptr(p.data), L.ptr(g), L.ptr(st["exp_avg"]), L.ptr(st["exp_avg_sq"]), C.c_uint64(p.numel()),
                                       L.ptr(sumsq), C.byref(cfg), L.stream()), "adam_step")
            if sumsq is not None and g.data_ptr() != p.grad.data_ptr():
                p.grad.copy_(g.view_as(p.grad))
        return loss


def _adam_check_world():
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise L.Mi3dError("Adam: multi-GPU (a process group of more than one rank) is not built; use Adan(group=...) there")


def _adam_check_group(group):
    for key, refused in (("amsgrad", True), ("maximize", True), ("capturable", True), ("differentiable", True), ("fused", True)):
        if group.get(key) == refused:
            raise L.Mi3dError(f"Adam: {key}=True is not built")
    if group.get("weight_decay", 0) != 0:
        raise L.Mi3dError(f"Adam: weight_decay={group['weight_decay']} is not built (main.py's Adam has none)")
    if torch.is_tensor(group["lr"]) and group["lr"].is_cuda:
        raise L.Mi3dError("Adam: a CUDA tensor lr would synchronise the host every step")


def _adam_check_param(p):
    if p.dtype != torch.float32 or not p.is_contiguous():
        raise L.Mi3dError("Adam: parameters must be contiguous fp32")
    if not p.is_cuda:
        raise L.Mi3dError("Adam: parameters must be CUDA tensors (there is no CPU path)")
