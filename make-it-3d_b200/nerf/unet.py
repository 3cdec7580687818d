"""B7 seam: the refine stage's gated U-Net, `UNet(num_input_channels=3+16)` of the reference's nerf/unet.py (nerf/utils.py:808, 863, 937),
on libmi3d.so.

`from mi3d_b200.nerf.unet import UNet` replaces the reference's import.  The module keeps the reference's constructor, submodule tree and
state_dict names (`start.block.conv_f.weight` .. `final.0.0.bias`, 41 entries with the BatchNorm buffers), and PyTorch's default
initialisation, so checkpoints load both ways and `torch.optim.Adam(unet.parameters())` works unchanged.

`forward([x0, x1, x2])` (x0 [N,19,H,W], x1 at H/2, x2 at H/4) runs in the engine of csrc/unet_engine.cu and returns [N,3,H,W] fp32.
The parameters are inputs of the autograd Function, so their gradients reach `.grad`; the engine reads their current values on every
call.  `.train()` uses batch statistics and updates the running statistics once per forward; `.eval()` uses the running statistics.
The backward may run more than once per forward (`retain_graph=True`).  One engine is planned per (N, H, W) on first use and cached.
Only the refine configuration is built, and there is no CPU or eager-PyTorch fallback.
"""
import contextlib
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib as L


class UNetCfg(C.Structure):
    _fields_ = [("N", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class UNetEngine:
    """Owns the device workspace and the planned launch lists of one (N, H, W) (mi3d_unet_create)."""

    def __init__(self, N, H, W, device, graph_replay=True):
        lib = L.lib()
        lib.mi3d_unet_workspace_bytes.restype = C.c_size_t
        lib.mi3d_unet_create.restype = C.c_void_p
        lib.mi3d_unet_param_name.restype = C.c_char_p
        self.cfg = UNetCfg(N, H, W)
        nbytes = lib.mi3d_unet_workspace_bytes(C.byref(self.cfg))
        if nbytes == 0:
            raise L.Mi3dError(f"unsupported U-Net shape N={N} H={H} W={W}")
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)
        h = lib.mi3d_unet_create(C.byref(self.cfg), L.ptr(self.workspace), C.c_size_t(nbytes))
        if not h:
            raise L.Mi3dError("mi3d_unet_create failed")
        self.h = C.c_void_p(h)
        self.names = [lib.mi3d_unet_param_name(self.h, C.c_int(i)).decode() for i in range(lib.mi3d_unet_num_params(self.h))]
        # an engine-owned stream, so the lists can replay as CUDA graphs (the legacy default stream cannot be captured)
        self.stream = torch.cuda.Stream(device) if graph_replay else None
        L.check(lib.mi3d_unet_set_graph_replay(self.h, C.c_int(1 if graph_replay else 0)), "unet_set_graph_replay")
        self.tape_id = 0          # bumped by every forward: each one replaces the engine's tape

    def graph_replays(self):
        return int(L.lib().mi3d_unet_graph_replays(self.h))

    @contextlib.contextmanager
    def on_stream(self):
        if self.stream is None:
            yield
            return
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            yield
        cur.wait_stream(self.stream)

    def forward(self, xs, state, train, need_grad):
        """state: registry name -> CUDA tensor (or None: a running statistic not to update)"""
        x0 = xs[0]
        out = torch.empty((x0.shape[0], 3, x0.shape[2], x0.shape[3]), dtype=torch.float32, device=x0.device)
        ptrs = (C.c_void_p * len(self.names))(*[None if state[n] is None else state[n].data_ptr() for n in self.names])
        with self.on_stream():
            L.check(L.lib().mi3d_unet_forward(self.h, L.ptr(xs[0]), L.ptr(xs[1]), L.ptr(xs[2]), ptrs, C.c_int(int(train)),
                                              C.c_int(int(need_grad)), L.ptr(out), L.stream()), "unet_forward")
        self.tape_id += 1
        return out

    def backward(self, dout, xs, params):
        """-> (dx0, dx1, dx2), {name: gradient} for the parameters named in `params`"""
        dout = L.f32c(dout)
        dxs = [torch.empty_like(x) for x in xs]
        grads = {n: torch.empty_like(p) for n, p in params.items()}
        ptrs = (C.c_void_p * len(self.names))(*[grads[n].data_ptr() if n in grads else None for n in self.names])
        with self.on_stream():
            L.check(L.lib().mi3d_unet_backward(self.h, L.ptr(dout), L.ptr(dxs[0]), L.ptr(dxs[1]), L.ptr(dxs[2]), ptrs, L.stream()),
                    "unet_backward")
        return dxs, grads

    def debug_tensor(self, name):
        """a named fp32 intermediate, as a view of the workspace"""
        p, n = C.c_void_p(), C.c_size_t()
        L.check(L.lib().mi3d_unet_debug_tensor(self.h, name.encode(), C.byref(p), C.byref(n)), f"unet_debug_tensor({name})")
        off = p.value - self.workspace.data_ptr()
        return self.workspace[off:off + n.value].view(torch.float32)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                L.lib().mi3d_unet_destroy(self.h)
        except Exception:
            pass


class _UNetFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, engine, train, need_grad, x0, x1, x2, *params):
        names = module._param_names
        state = dict(zip(names, params))
        for n, b in module.named_buffers():
            state[n] = b
        out = engine.forward((x0, x1, x2), state, train, need_grad)
        ctx.module, ctx.engine, ctx.train, ctx.tape_id = module, engine, train, engine.tape_id
        if need_grad:
            ctx.save_for_backward(x0, x1, x2, *params)
            # an eval-mode tape rebuild must read the running statistics this forward read
            ctx.eval_buffers = None if train else {n: b.detach().clone() for n, b in module.named_buffers()}
        return out

    @staticmethod
    def backward(ctx, dout):
        x0, x1, x2, *params = ctx.saved_tensors
        eng, names = ctx.engine, ctx.module._param_names
        pmap = dict(zip(names, params))
        if eng.tape_id != ctx.tape_id:
            # a later forward on this engine replaced its tape: rebuild it from the same inputs and parameters, without touching the
            # running statistics again (train mode) or with the ones the forward read (eval mode)
            state = dict(pmap)
            if ctx.train:
                state.update({n: None for n, _ in ctx.module.named_buffers()})
            else:
                state.update(ctx.eval_buffers)
            eng.forward((x0, x1, x2), state, ctx.train, True)
            ctx.tape_id = eng.tape_id
        need = {n: p for n, p, g in zip(names, params, ctx.needs_input_grad[7:]) if g}
        dxs, grads = eng.backward(dout, (x0, x1, x2), need)
        return (None, None, None, None, *[d if g else None for d, g in zip(dxs, ctx.needs_input_grad[4:7])],
                *[grads.get(n) for n in names])


class _Block(nn.Module):
    """GatedBlock(cin, c): its parameters live in `block` (conv_f, act_f, conv_m, act_m, norm), as in the reference"""

    def __init__(self, cin, c, norm=True):
        super().__init__()
        self.block = nn.ModuleDict({
            "conv_f": nn.Conv2d(cin, c, 3, padding=1), "act_f": nn.ELU(),
            "conv_m": nn.Conv2d(cin, c, 3, padding=1), "act_m": nn.Sigmoid(),
            "norm": nn.BatchNorm2d(c) if norm else nn.Identity(),
        })


class _Down(nn.Module):
    def __init__(self, cin, c):
        super().__init__()
        self.conv = _Block(cin, c)
        self.down = nn.AvgPool2d(2, 2)


class _Up(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.up = nn.Sequential(nn.Upsample(scale_factor=2, mode="bilinear"), nn.Sequential(nn.Conv2d(2 * c, c, 3, padding=1)))
        self.conv = _Block(2 * c, c, norm=False)


class UNet(nn.Module):
    r"""Rendering network with UNet architecture and multi-scale input (the refine stage's configuration only)."""

    def __init__(self, num_input_channels=3, num_output_channels=3, feature_scale=4, upsample_mode='bilinear', last_act='sigmoid',
                 conv_block='gated', graph_replay=True):
        super().__init__()
        if conv_block != 'gated':
            raise L.Mi3dError(f"conv_block={conv_block!r}: only 'gated' (the refine stage's) is built")
        if num_input_channels != 19:
            raise L.Mi3dError(f"num_input_channels={num_input_channels}: only 19 (3 + 16, the refine stage's) is built")
        if num_output_channels != 3:
            raise L.Mi3dError(f"num_output_channels={num_output_channels}: only 3 is built")
        if feature_scale != 4:
            raise L.Mi3dError(f"feature_scale={feature_scale}: only 4 is built")
        if upsample_mode != 'bilinear':
            raise L.Mi3dError(f"upsample_mode={upsample_mode!r}: only 'bilinear' is built")
        if last_act != 'sigmoid':
            raise L.Mi3dError(f"last_act={last_act!r}: only 'sigmoid' is built")
        self.feature_scale = feature_scale
        self.num_input_channels = num_input_channels
        self.graph_replay = graph_replay
        # constructed in the reference's order, so a seeded construction draws the same default initialisation
        self.start = _Block(19, 16)
        self.down1 = _Down(16, 13)
        self.down2 = _Down(32, 45)
        self.up2 = _Up(32)
        self.up1 = _Up(16)
        self.final = nn.Sequential(nn.Sequential(nn.Conv2d(16, 3, 1)), nn.Sigmoid())
        self._param_names = [n for n, _ in self.named_parameters()]
        self.engines = {}

    def engine(self, N, H, W, device):
        key = (N, H, W, device)
        if key not in self.engines:
            self.engines[key] = UNetEngine(N, H, W, device, graph_replay=self.graph_replay)
        return self.engines[key]

    def forward(self, inputs, **kwargs):
        if len(inputs) != 3:
            raise L.Mi3dError(f"UNet expects 3 input scales, got {len(inputs)}")
        x0, x1, x2 = inputs
        L.require_cuda(x0, x1, x2)
        params = [p for _, p in self.named_parameters()]
        L.require_cuda(*params)
        if x0.dim() != 4 or x0.shape[1] != 19:
            raise L.Mi3dError(f"x0 must be [N,19,H,W], got {tuple(x0.shape)}")
        N, _, H, W = x0.shape
        if H % 4 or W % 4:
            raise L.Mi3dError(f"H and W must be multiples of 4, got {H} x {W}")
        if tuple(x1.shape) != (N, 19, H // 2, W // 2) or tuple(x2.shape) != (N, 19, H // 4, W // 4):
            raise L.Mi3dError(f"input scales disagree: {tuple(x0.shape)}, {tuple(x1.shape)}, {tuple(x2.shape)}")
        if self.training and N * (H // 4) * (W // 4) < 2:
            raise L.Mi3dError(f"train-mode BatchNorm needs more than one value per channel at H/4 x W/4; got N={N}, {H} x {W}")
        for n, b in self.named_buffers():
            want = torch.long if n.endswith("num_batches_tracked") else torch.float32
            if b.dtype != want or not b.is_contiguous() or b.device != x0.device:
                raise L.Mi3dError(f"buffer {n} must be a contiguous {want} tensor on {x0.device}, got {b.dtype} on {b.device}")
        need = torch.is_grad_enabled() and (any(x.requires_grad for x in inputs) or any(p.requires_grad for p in params))
        xs = [L.f32c(x) if need else L.f32c(x.detach()) for x in inputs]
        eng = self.engine(N, H, W, x0.device)
        if not need:
            params = [p.detach() for p in params]
        return _UNetFn.apply(self, eng, self.training, need, *xs, *[L.f32c(p) for p in params])
