"""Record tests/golden/unet_ref.npz from the reference's own nerf/unet.py (CPU, fp64).

    MI3D_REFERENCE_DIR=<checkout of the reference> python tests/golden/make_golden_unet.py

The module is imported unmodified and built as the refine stage builds it, UNet(num_input_channels=3+16), in train mode.  Recorded at
N = 2, 24 x 40: one train-mode forward (output and running statistics after it), the backward of sum(out * w) (the three input gradients
and every parameter gradient), then an eval-mode forward.  To keep the file small, inputs, weights and w are stored as integer codes that
decode exactly to fp32 (see decode()); the results are fp32.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

N, H, W = 2, 24, 40
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "unet_ref.npz")


def decode(z):
    """-> (params {name: fp32 tensor}, [x0, x1, x2], w) from the codes in the fixture"""
    names = [str(n) for n in z["names"]]
    params, off = {}, 0
    codes = z["param_codes"]
    for n, shp in zip(names, z["shapes"]):
        shp = tuple(int(s) for s in shp if s > 0)
        k = int(np.prod(shp)) if shp else 1
        c = codes[off:off + k].astype(np.float32).reshape(shp)
        off += k
        if n.endswith("num_batches_tracked"):
            params[n] = torch.tensor(int(c), dtype=torch.long)
        elif n.endswith("running_var"):
            params[n] = torch.from_numpy(1.0 + c / 64.0)
        elif n.endswith("norm.weight"):
            params[n] = torch.from_numpy(1.0 + c / 256.0)
        elif n.endswith("running_mean"):
            params[n] = torch.from_numpy(c / 64.0)
        else:
            params[n] = torch.from_numpy(c / 1024.0)
    xs = [torch.from_numpy(z[f"x{i}_codes"].astype(np.float32) / 255.0) for i in range(3)]
    w = torch.from_numpy(z["w_codes"].astype(np.float32) / 128.0)
    return params, xs, w


def main():
    ref = os.environ.get("MI3D_REFERENCE_DIR")
    if not ref:
        sys.exit("set MI3D_REFERENCE_DIR to a checkout of the reference")
    spec = importlib.util.spec_from_file_location("ref_unet", os.path.join(ref, "nerf", "unet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.manual_seed(0)
    net = mod.UNet(num_input_channels=3 + 16)
    sd = net.state_dict()
    rng = np.random.default_rng(0)
    names, shapes, codes = [], [], []
    for n, t in sd.items():
        names.append(n)
        shapes.append(list(t.shape) + [0] * (4 - t.dim()))
        if n.endswith("num_batches_tracked"):
            c = np.array([3])                                     # a checkpoint that has already trained a few steps
        elif ".norm." in n:
            c = rng.integers(-32, 33, size=t.numel())             # gamma 1 +- 1/8, beta / running mean +- 1/2, running var 1 +- 1/2
        else:
            bound = 1.0 / np.sqrt(t.numel() / t.shape[0]) if t.dim() > 1 else 1.0 / np.sqrt(sd[n[:-4] + "weight"][0].numel())
            lim = int(bound * 1024)
            c = rng.integers(-lim, lim + 1, size=t.numel())
        codes.append(c.astype(np.int16))
    xs_codes = [rng.integers(0, 256, size=(N, 19, H >> i, W >> i)).astype(np.uint8) for i in range(3)]
    w_codes = rng.integers(-128, 128, size=(N, 3, H, W)).astype(np.int8)
    z = {"names": np.array(names), "shapes": np.array(shapes, np.int32), "param_codes": np.concatenate(codes)}
    z.update({f"x{i}_codes": c for i, c in enumerate(xs_codes)})
    z["w_codes"] = w_codes
    params, xs, w = decode(z)
    net.load_state_dict(params)
    net = net.double().train()
    xs = [x.double().requires_grad_(True) for x in xs]
    out = net(xs)
    (out * w.double()).sum().backward()
    res = {"out": out.detach().float().numpy()}
    for i in range(3):
        res[f"dx{i}"] = xs[i].grad.float().numpy()
    for n, p in net.named_parameters():
        res["grad/" + n] = p.grad.float().numpy()
    for n, b in net.named_buffers():
        res["after/" + n] = b.detach().cpu().numpy().astype(np.int64 if b.dtype == torch.long else np.float32)
    net.eval()
    with torch.no_grad():
        res["eval_out"] = net([x.detach() for x in xs]).float().numpy()
    z.update(res)
    np.savez_compressed(OUT, **z)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
