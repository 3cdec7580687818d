"""B6 seam: the `contextual_loss` package's `ContextualLoss(use_vgg=True, vgg_layer='relu5_4')` (nerf/utils.py:36, 810), on libmi3d.so.

`from mi3d_b200.nerf import contextual_loss as cl` replaces `import contextual_loss as cl`; `cl.ContextualLoss(...)` then has the
package's signature and state_dict names (`vgg_model.slice1.0.weight` .. `vgg_model.slice5.34.bias`, `vgg_mean`, `vgg_std`).  The package
loads torchvision's ImageNet VGG19; here `load_torchvision_vgg19(torchvision.models.vgg19(...).state_dict())` loads those weights, and
without them the module holds seeded stand-in weights.

Everything from the images to the loss runs in the engine of csrc/cx_engine.cu: VGG19 up to relu5_4 on [x; y] in one batched pass (tile
GEMM, fp16 storage, fp32 accumulation), then the contextual loss in fp32.  `forward(x, y)` returns the scalar loss with an autograd
backward for `x` only (the weights are frozen and `y` must not require a gradient, as the reference's `gt_rgb`).  One engine is planned
per (N, H, W) on first use and cached.  There is no CPU or eager-PyTorch fallback.
"""
import contextlib
import ctypes as C
import math

import torch
import torch.nn as nn

from .. import _lib as L

# torchvision vgg19().features indices of the 16 convs up to relu5_4, and the package's VGG19 slice holding each
CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25, 28, 30, 32, 34)
CONV_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512, 512, 512, 512, 512)


def _slice(idx):
    return 1 if idx < 4 else 2 if idx < 9 else 3 if idx < 18 else 4 if idx < 27 else 5


def package_name(tv_name):
    """'features.N.weight' (torchvision) -> 'vgg_model.sliceS.N.weight' (contextual_loss)"""
    _, idx, leaf = tv_name.split(".")
    return f"vgg_model.slice{_slice(int(idx))}.{idx}.{leaf}"


def torchvision_name(pkg_name):
    """'vgg_model.sliceS.N.weight' -> 'features.N.weight'"""
    _, _, idx, leaf = pkg_name.split(".")
    return f"features.{idx}.{leaf}"


class CxCfg(C.Structure):
    _fields_ = [("N", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class CxEngine:
    """Owns the device workspace and the planned launch lists of one (N, H, W) (mi3d_cx_create)."""

    def __init__(self, N, H, W, device, graph_replay=True):
        lib = L.lib()
        lib.mi3d_cx_workspace_bytes.restype = C.c_size_t
        lib.mi3d_cx_create.restype = C.c_void_p
        lib.mi3d_cx_param_name.restype = C.c_char_p
        self.cfg = CxCfg(N, H, W)
        nbytes = lib.mi3d_cx_workspace_bytes(C.byref(self.cfg))
        if nbytes == 0:
            raise L.Mi3dError(f"unsupported contextual-loss shape N={N} H={H} W={W}")
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        h = lib.mi3d_cx_create(C.byref(self.cfg), L.ptr(self.workspace), C.c_size_t(nbytes))
        if not h:
            raise L.Mi3dError("mi3d_cx_create failed (TMA descriptor encoding error)")
        self.h = C.c_void_p(h)
        self.names = [lib.mi3d_cx_param_name(self.h, C.c_int(i)).decode() for i in range(lib.mi3d_cx_num_params(self.h))]
        # as in ClipEngine: an engine-owned stream, so the lists can replay as CUDA graphs (the legacy default stream cannot be captured)
        self.stream = torch.cuda.Stream(device) if graph_replay else None
        L.check(lib.mi3d_cx_set_graph_replay(self.h, C.c_int(1 if graph_replay else 0)), "cx_set_graph_replay")
        self.tape_id = 0          # bumped by every forward: each one replaces the engine's tape

    def graph_replays(self):
        return int(L.lib().mi3d_cx_graph_replays(self.h))

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

    def load(self, tensors):
        """tensors: package state_dict name -> fp32 CUDA tensor"""
        lib = L.lib()
        for i, name in enumerate(self.names):
            if "#" in name:
                continue          # derived copies are written with their base tensor
            src = L.f32c(tensors[name])
            L.check(lib.mi3d_cx_load_param(self.h, C.c_int(i), L.ptr(src), L.stream()), f"cx_load_param({name})")
        torch.cuda.synchronize()

    def forward(self, x, y, band_width, need_grad):
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        with self.on_stream():
            L.check(L.lib().mi3d_cx_forward(self.h, L.ptr(x), L.ptr(y), C.c_float(band_width), C.c_int(int(need_grad)), L.ptr(loss),
                                            L.stream()), "cx_forward")
        self.tape_id += 1
        return loss

    def backward(self, dloss, shape):
        dloss = L.f32c(dloss)
        dx = torch.empty(shape, dtype=torch.float32, device=dloss.device)
        with self.on_stream():
            L.check(L.lib().mi3d_cx_backward(self.h, L.ptr(dloss), L.ptr(dx), L.stream()), "cx_backward")
        return dx

    def debug_tensor(self, name, dtype=torch.float16):
        """a named intermediate, as a view of the workspace ("relu5_4": fp16 NHWC [2N,H/16,W/16,512])"""
        p, n = C.c_void_p(), C.c_size_t()
        L.check(L.lib().mi3d_cx_debug_tensor(self.h, name.encode(), C.byref(p), C.byref(n)), f"cx_debug_tensor({name})")
        off = p.value - self.workspace.data_ptr()
        return self.workspace[off:off + n.value].view(dtype)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                L.lib().mi3d_cx_destroy(self.h)
        except Exception:
            pass


class _CxLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, engine, band_width, need_grad):
        loss = engine.forward(x, y, band_width, need_grad)
        ctx.engine, ctx.band_width, ctx.tape_id = engine, band_width, engine.tape_id
        if need_grad:
            ctx.save_for_backward(x, y)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, y = ctx.saved_tensors
        eng = ctx.engine
        if eng.tape_id != ctx.tape_id:
            # a later forward on this engine replaced its tape: rebuild it (same inputs, same result)
            eng.forward(x, y, ctx.band_width, True)
        dx = eng.backward(g.reshape(()), x.shape)
        return dx.to(x.dtype), None, None, None, None


class ContextualLoss(nn.Module):
    def __init__(self, band_width=0.5, loss_type='cosine', use_vgg=True, vgg_layer='relu5_4', device='cuda', state_dict=None, seed=0,
                 graph_replay=True):
        super().__init__()
        if not band_width > 0:
            raise L.Mi3dError("band_width must be positive")
        if loss_type != 'cosine':
            raise L.Mi3dError(f"loss_type={loss_type!r}: only 'cosine' (the refine stage's) is built")
        if not use_vgg:
            raise L.Mi3dError("use_vgg=False is not built: the refine stage uses the VGG features")
        if vgg_layer != 'relu5_4':
            raise L.Mi3dError(f"vgg_layer={vgg_layer!r}: only 'relu5_4' (the refine stage's) is built")
        self.band_width = float(band_width)
        self.vgg_layer = vgg_layer
        self.graph_replay = graph_replay
        self.dev = torch.device(device)
        gen = torch.Generator().manual_seed(seed)
        vgg = nn.Module()
        cin = 3
        for idx, cout in zip(CONV_INDICES, CONV_CHANNELS):
            name = f"vgg_model.slice{_slice(idx)}.{idx}"
            w = _default_weight(cout, cin, gen)
            b = torch.randn(cout, generator=gen) * 0.05
            if state_dict is not None:
                w = state_dict[name + ".weight"].detach().float().reshape(cout, cin, 3, 3)
                b = state_dict[name + ".bias"].detach().float().reshape(cout)
            s = vgg._modules.setdefault(f"slice{_slice(idx)}", nn.Module())
            conv = nn.Module()
            conv.register_parameter("weight", nn.Parameter(w.to(self.dev).contiguous(), requires_grad=False))
            conv.register_parameter("bias", nn.Parameter(b.to(self.dev).contiguous(), requires_grad=False))
            s.add_module(str(idx), conv)
            cin = cout
        self.vgg_model = vgg
        self.register_buffer("vgg_mean", torch.tensor([[[0.485]], [[0.456]], [[0.406]]], device=self.dev))
        self.register_buffer("vgg_std", torch.tensor([[[0.229]], [[0.224]], [[0.225]]], device=self.dev))
        self.engines = {}

    def load_torchvision_vgg19(self, sd):
        """load `torchvision.models.vgg19(...).state_dict()` (names `features.N.*`; entries past relu5_4 and the classifier are ignored)"""
        own = dict(self.named_parameters())
        with torch.no_grad():
            for k, p in own.items():
                p.copy_(sd[torchvision_name(k)].to(p.device, torch.float32).reshape(p.shape))
        self.reload()
        return self

    def reload(self):
        """push the current parameter values into every planned engine (after load_state_dict)"""
        tensors = {k: p.data for k, p in self.named_parameters()}
        for eng in self.engines.values():
            eng.load(tensors)

    def engine(self, N, H, W):
        key = (N, H, W)
        if key not in self.engines:
            eng = CxEngine(N, H, W, self.dev, graph_replay=self.graph_replay)
            eng.load({k: p.data for k, p in self.named_parameters()})
            self.engines[key] = eng
        return self.engines[key]

    def forward(self, x, y):
        L.require_cuda(x, y)
        if x.dim() != 4 or x.shape[1] != 3:
            raise L.Mi3dError(f"ContextualLoss expects [N,3,H,W] images, got {tuple(x.shape)}")
        if x.shape != y.shape:
            raise L.Mi3dError(f"x and y differ in shape: {tuple(x.shape)} vs {tuple(y.shape)}")
        N, _, H, W = x.shape
        if H < 16 or W < 16:
            raise L.Mi3dError(f"H and W must be >= 16 (relu5_4 is H/16 x W/16), got {H} x {W}")
        if y.requires_grad:
            raise L.Mi3dError("y must not require a gradient (the loss has no gradient for y)")
        need = torch.is_grad_enabled() and x.requires_grad
        eng = self.engine(N, H, W)
        return _CxLoss.apply(L.f32c(x) if need else L.f32c(x.detach()), L.f32c(y), eng, self.band_width, need)


def _default_weight(cout, cin, gen):
    """seeded stand-in weights (torchvision's VGG init is kaiming-normal; fan_in keeps the forward activations O(1))"""
    return torch.randn(cout, cin, 3, 3, generator=gen) * math.sqrt(2.0 / (cin * 9))
