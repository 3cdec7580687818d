"""Functional restatement (torch.nn.functional) of the refine stage's gated U-Net: UNet(num_input_channels=19) of the reference's
nerf/unet.py with its defaults (feature_scale 4, bilinear upsampling, sigmoid output, gated blocks), parameters under the reference's
state_dict names.  The GPU tests compare csrc/unet_engine.cu against it; tests/golden/unet_ref.npz pins it to the reference's module.

round_fp16=True rounds every stored activation (block outputs, pre-activations, pooled and upsampled maps) to fp16 and back: the
difference to the fp32 result measures what fp16 activation storage alone costs, the floor the GPU tests scale their tolerance from.
"""
import math

import torch
import torch.nn.functional as F

# (prefix, cin, c, batch norm) of the five gated blocks and (name, cin, cout, k) of the plain convs, in state_dict order
GATED = (("start.block.", 19, 16, True), ("down1.conv.block.", 16, 13, True), ("down2.conv.block.", 32, 45, True),
         ("up2.conv.block.", 64, 32, False), ("up1.conv.block.", 32, 16, False))
CONVS = (("up2.up.1.0", 64, 32, 3), ("up1.up.1.0", 32, 16, 3), ("final.0.0", 16, 3, 1))
BN_EPS, BN_MOMENTUM = 1e-5, 0.1


def state_names():
    """the 41 state_dict entries, in the reference's order"""
    out = []
    for pre, _, _, bn in GATED[:3]:
        out += [pre + s for s in ("conv_f.weight", "conv_f.bias", "conv_m.weight", "conv_m.bias")]
        out += [pre + s for s in ("norm.weight", "norm.bias", "norm.running_mean", "norm.running_var", "norm.num_batches_tracked")]
    for (cname, *_), (pre, *_) in zip(CONVS[:2], GATED[3:]):
        out += [cname + ".weight", cname + ".bias"] + [pre + s for s in ("conv_f.weight", "conv_f.bias", "conv_m.weight", "conv_m.bias")]
    return out + ["final.0.0.weight", "final.0.0.bias"]


def shapes():
    s = {}
    for pre, cin, c, bn in GATED:
        for k in ("conv_f", "conv_m"):
            s[f"{pre}{k}.weight"], s[f"{pre}{k}.bias"] = (c, cin, 3, 3), (c,)
        if bn:
            for k in ("weight", "bias", "running_mean", "running_var"):
                s[f"{pre}norm.{k}"] = (c,)
            s[f"{pre}norm.num_batches_tracked"] = ()
    for name, cin, cout, k in CONVS:
        s[name + ".weight"], s[name + ".bias"] = (cout, cin, k, k), (cout,)
    return {n: s[n] for n in state_names()}


def seeded_params(seed=0, device="cpu", gamma_jitter=0.0):
    """PyTorch's default initialisation (kaiming-uniform(a=sqrt 5) convs: U(+-1/sqrt(fan_in)) weights and biases; BatchNorm weight 1,
    bias 0, running mean 0, var 1) from a seeded generator; gamma_jitter > 0 perturbs the BatchNorm affine parameters"""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for n, shp in shapes().items():
        if n.endswith("num_batches_tracked"):
            p[n] = torch.zeros((), dtype=torch.long)
        elif ".norm." in n:
            base = 1.0 if n.endswith(("weight", "running_var")) else 0.0
            t = torch.full(shp, base)
            if gamma_jitter and n.endswith(("norm.weight", "norm.bias")):
                t = t + gamma_jitter * (2 * torch.rand(shp, generator=g) - 1)
            p[n] = t
        else:
            wshape = shapes()[n.rsplit(".", 1)[0] + ".weight"]
            bound = 1.0 / math.sqrt(wshape[1] * wshape[2] * wshape[3])
            p[n] = (2 * torch.rand(shp, generator=g) - 1) * bound
    return {k: v.to(device) for k, v in p.items()}


def _r(x, round_fp16):
    return x.half().float() if round_fp16 else x


def _gated(x, p, pre, bn, train, rf):
    f = _r(F.conv2d(x, p[pre + "conv_f.weight"], p[pre + "conv_f.bias"], padding=1), rf)
    m = _r(F.conv2d(x, p[pre + "conv_m.weight"], p[pre + "conv_m.bias"], padding=1), rf)
    y = F.elu(f) * torch.sigmoid(m)
    if bn:
        y = F.batch_norm(y, p[pre + "norm.running_mean"], p[pre + "norm.running_var"], p[pre + "norm.weight"], p[pre + "norm.bias"],
                         training=train, momentum=BN_MOMENTUM, eps=BN_EPS)
        if train:
            p[pre + "norm.num_batches_tracked"].add_(1)
    return _r(y, rf)


def unet(xs, p, train=True, round_fp16=False):
    """xs = [x0 [N,19,H,W], x1 [N,19,H/2,W/2], x2 [N,19,H/4,W/4]] -> [N,3,H,W]; in train mode the running statistics in p are updated"""
    rf = round_fp16
    up = lambda t: _r(F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False), rf)
    in64 = _gated(xs[0], p, "start.block.", True, train, rf)
    d1 = torch.cat([_gated(_r(F.avg_pool2d(in64, 2, 2), rf), p, "down1.conv.block.", True, train, rf), xs[1]], 1)
    d2 = torch.cat([_gated(_r(F.avg_pool2d(d1, 2, 2), rf), p, "down2.conv.block.", True, train, rf), xs[2]], 1)
    u = _r(F.conv2d(up(d2), p["up2.up.1.0.weight"], p["up2.up.1.0.bias"], padding=1), rf)
    u = _gated(torch.cat([u, d1], 1), p, "up2.conv.block.", False, train, rf)
    u = _r(F.conv2d(up(u), p["up1.up.1.0.weight"], p["up1.up.1.0.bias"], padding=1), rf)
    u = _gated(torch.cat([u, in64], 1), p, "up1.conv.block.", False, train, rf)
    return torch.sigmoid(F.conv2d(u, p["final.0.0.weight"], p["final.0.0.bias"]))


def param_names():
    return [n for n in state_names() if not any(n.endswith(s) for s in ("running_mean", "running_var", "num_batches_tracked"))]
