"""B8 seam: the DPT-Hybrid depth model behind the reference image's depth prior (main.py:111-127, 196-214) on libmi3d.so.

`DPTDepthModel(path=None, non_negative=True, backbone="vitb_rn50_384", enable_attention_hooks=False, state_dict=None)` is a drop-in for
the reference's `DPT.dpt.models.DPTDepthModel` at the configuration main.py builds; it runs in the engine of csrc/dpt_engine.cu (tile
GEMMs, fused attention, GroupNorm / upsample / head kernels), with no CPU or eager-PyTorch fallback and no timm.

* Weights carry the reference's `state_dict()` names, so `path=` takes the reference's checkpoint (`dpt_hybrid-midas-501f0c75.pt`),
  unwrapped as DPT/dpt/base_model.py does.  Each tensor passes through the device on its way into the engine's fp16 copy.  Without
  weights the engine runs on seeded stand-ins.
* `forward(x)`: CUDA fp32 `[1, 3, 384, 384]` (resized, normalised) -> inverse depth fp32 `[1, 384, 384]`, no gradient.
* `reference_depth(model, ori_imgs, depth_mask)` is main.py:196-214 end to end: what that code leaves in `depth_prediction`.
"""
import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib as L

IGNORED_PREFIXES = ("pretrained.model.norm.", "pretrained.model.head.", "scratch.refinenet4.resConfUnit1.")


class DPTDepthModel(L.Engine):
    def __init__(self, path=None, non_negative=True, backbone="vitb_rn50_384", enable_attention_hooks=False, state_dict=None,
                 device="cuda"):
        if backbone != "vitb_rn50_384":
            raise L.Mi3dError(f"only the DPT-Hybrid backbone 'vitb_rn50_384' is built, not {backbone!r}")
        if not non_negative:
            raise L.Mi3dError("only non_negative=True (the final ReLU) is built")
        if enable_attention_hooks:
            raise L.Mi3dError("attention hooks are not built")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.Mi3dError("the DPT engine runs on sm_90a only; there is no CPU fallback")
        super().__init__("dpt", (), self.device, False, "DPT configuration")       # one eager forward per image: no graph replay
        if path is not None:
            state_dict = torch.load(path, map_location="cpu")
            if "optimizer" in state_dict:
                state_dict = state_dict["model"]
        self.load_state_dict(state_dict if state_dict is not None else _default_state(self.names, self.shapes))

    def to(self, device):
        if torch.device(device).type != "cuda":
            raise L.Mi3dError("the DPT engine runs on sm_90a only; there is no CPU fallback")
        return self

    def eval(self):
        return self

    def load_state_dict(self, state_dict):
        """the reference's DPTDepthModel.state_dict() names: every tensor the forward reads is required; of the others only
        pretrained.model.norm.*, pretrained.model.head.* and scratch.refinenet4.resConfUnit1.* are accepted (and ignored)"""
        return self.load_strict(state_dict, lambda k: k.startswith(IGNORED_PREFIXES))

    def forward(self, x):
        """x CUDA fp32 [1, 3, 384, 384] -> inverse depth fp32 [1, 384, 384]"""
        if not torch.is_tensor(x) or x.dtype != torch.float32:
            raise L.Mi3dError("DPT takes an fp32 image [1,3,384,384]")
        L.require_cuda(x)
        if tuple(x.shape) != (1, 3, 384, 384):
            raise L.Mi3dError(f"DPT takes an fp32 image [1,3,384,384]; got {tuple(x.shape)}")
        x = x.contiguous()
        out = torch.empty(1, 384, 384, dtype=torch.float32, device=x.device)
        L.check(L.lib().mi3d_dpt_forward(self.h, L.ptr(x), L.ptr(out), L.stream()), "dpt_forward")
        return out

    __call__ = forward

    def taps(self):
        """the last forward's reassembled backbone features layer_1 .. layer_4, fp32 NCHW"""
        shapes = ((1, 256, 96, 96), (1, 512, 48, 48), (1, 768, 24, 24), (1, 768, 12, 12))
        out = []
        for i, s in enumerate(shapes):
            t = torch.empty(s, dtype=torch.float32, device=self.device)
            L.check(L.lib().mi3d_dpt_tap(self.h, C.c_int(i), L.ptr(t), L.stream()), "dpt_tap")
            out.append(t)
        return out


def _default_state(names, shapes, seed=0):
    """seeded stand-in weights (no DPT checkpoint exists offline): normal(0, 0.02) linears and convs, zero biases, unit norms"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in zip(names, shapes):
        if ".norm" in name:
            out[name] = torch.ones(shape) if name.endswith("weight") else torch.zeros(shape)
        elif name.endswith("bias"):
            out[name] = torch.zeros(shape)
        else:
            out[name] = torch.randn(shape, generator=g) * 0.02
    return out


def depth_transform(ori_imgs):
    """main.py:120-125, as written there: T.Resize((384, 384)) then T.Normalize((0.5,) * 3, (0.5,) * 3)"""
    import torchvision.transforms as T
    return T.Compose([T.Resize((384, 384)), T.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])(ori_imgs)


def reference_depth(model, ori_imgs, depth_mask):
    """main.py:196-214: depth prior of the reference image.  ori_imgs fp32 [1, 3, H, W] in [0, 1] and depth_mask bool [1, 1, 512, 512]
    (True outside the object), both CUDA -> float64 [1, 1, 512, 512], what that code leaves in `depth_prediction`.  The uint16 PNG
    that write_depth_name(bits=2) writes and imageio reads back is a lossless round trip, so it is done in memory."""
    from scipy.ndimage import median_filter
    with torch.no_grad():
        pred = model.forward(depth_transform(ori_imgs))
        pred = F.interpolate(pred.unsqueeze(1), size=512, mode="bicubic", align_corners=True)
        depth = pred.squeeze().cpu().numpy()
        lo, hi = depth.min(), depth.max()
        if hi - lo > np.finfo("float").eps:
            out = 65535 * (depth - lo) / (hi - lo)
        else:
            out = np.zeros(depth.shape, dtype=depth.dtype)
        disparity = out.astype("uint16") / 65535.
        disparity = median_filter(disparity, size=5)
        depth = 1. / np.maximum(disparity, 1e-2)
    dev = ori_imgs.device
    d = torch.tensor(depth, device=dev)
    m = depth_mask.to(dev)
    d = d * (~m) + torch.ones_like(d) * m
    return ((d - 1.0) / (d.max() - 1.0)) * 0.9 + 0.1
