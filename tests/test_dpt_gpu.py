"""GPU parity of the DPT-Hybrid depth model (csrc/dpt_engine.cu behind nerf/dpt.py) against the fp32 oracle (oracle/dpt_ref.py), with
seeded weights, plus the state_dict / path loading, input checks, and main.py:196-214 end to end (`reference_depth`).

Tolerance, as for the other engines: the engine stores fp16 between kernels, so the oracle also runs with every stored tensor rounded
to fp16 (e16) and the engine's relative L2 error must stay within max(2.5 x that fp16-storage error, 1e-3).  Observed values are
printed."""
import importlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dpt_ref

pytestmark = pytest.mark.gpu


def _mods():
    return importlib.import_module("make-it-3d_b200.nerf.dpt"), importlib.import_module("make-it-3d_b200._lib")


def _rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / b.norm())


def _image(seed, hw=384):
    g = torch.Generator().manual_seed(seed)
    x = F.interpolate(torch.rand(1, 3, hw // 16, hw // 16, generator=g), size=hw, mode="bilinear", align_corners=False)
    return (x + 0.05 * torch.randn(1, 3, hw, hw, generator=g)).clamp(0, 1)


@pytest.fixture(scope="module")
def setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dpt, _ = _mods()
    sd = dpt_ref.default_init(seed=3)
    model = dpt.DPTDepthModel(state_dict=sd)
    p = {k: v.cuda() for k, v in sd.items()}
    x = ((_image(4) - 0.5) / 0.5).cuda()
    with torch.no_grad():
        ref32 = dpt_ref.forward(p, x, taps=True)
        ref16 = dpt_ref.forward(p, x, e16=True, taps=True)
    return model, sd, p, x, ref32, ref16


def test_registry_is_the_reference_naming(setup):
    model = setup[0]
    shapes = dpt_ref.param_shapes()
    assert model.names == list(shapes)
    assert model.shapes == [tuple(s) for s in shapes.values()]


def test_forward_and_taps_match_oracle(setup):
    model, _, _, x, (o32, t32), (o16, t16) = setup
    out = model.forward(x)
    taps = model.taps()
    torch.cuda.synchronize()
    assert out.shape == (1, 384, 384) and out.dtype == torch.float32
    for name, got, a, b in [("depth", out, o32, o16)] + [(f"layer_{i + 1}", taps[i], t32[i], t16[i]) for i in range(4)]:
        assert got.shape == a.shape, name
        e, e16 = _rel(got, a), _rel(b, a)
        print(f"{name:10s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
        assert e <= max(2.5 * e16, 1e-3), (name, e, e16)


def test_bit_identical_across_calls(setup):
    model, x = setup[0], setup[3]
    a = model.forward(x).clone()
    b = model.forward(x.clone())
    assert torch.equal(a, b)


def test_path_loading(setup, tmp_path):
    dpt, _ = _mods()
    model, sd, _, x = setup[:4]
    full = dict(sd)                        # the reference's checkpoint also carries the tensors forward never reads
    full.update({k: torch.zeros(v) for k, v in dpt_ref.ignored_shapes().items()})
    want = model.forward(x).clone()
    torch.save(full, tmp_path / "plain.pt")
    torch.save({"model": full, "optimizer": {"state": {}}}, tmp_path / "wrapped.pt")
    for f in ("plain.pt", "wrapped.pt"):
        m = dpt.DPTDepthModel(path=str(tmp_path / f), backbone="vitb_rn50_384", non_negative=True, enable_attention_hooks=False)
        assert m.to("cuda") is m and m.eval() is m
        assert torch.equal(m.forward(x), want), f
        del m


def test_state_dict_mismatch_raises(setup):
    _, L = _mods()
    model, sd = setup[0], setup[1]
    extra = dict(sd, **{"pretrained.model.something.weight": torch.zeros(3)})
    with pytest.raises(L.Mi3dError):
        model.load_state_dict(extra)
    missing = dict(sd)
    missing.pop("scratch.refinenet1.out_conv.bias")
    with pytest.raises(L.Mi3dError):
        model.load_state_dict(missing)
    wrong = dict(sd, **{"scratch.refinenet1.out_conv.bias": torch.zeros(255)})
    with pytest.raises(L.Mi3dError):
        model.load_state_dict(wrong)
    model.load_state_dict(sd)              # still loads afterwards


def test_bad_inputs_raise(setup):
    dpt, L = _mods()
    model, x = setup[0], setup[3]
    for bad in (x.cpu(), x.half(), x[:, :, :383], torch.cat([x, x]), x[0]):
        with pytest.raises(L.Mi3dError):
            model.forward(bad)
    for kw in (dict(backbone="vitl16_384"), dict(backbone="vitb16_384"), dict(non_negative=False), dict(enable_attention_hooks=True)):
        with pytest.raises(L.Mi3dError):
            dpt.DPTDepthModel(**kw)
    with pytest.raises(L.Mi3dError):
        model.to("cpu")


def test_stand_in_weights_are_not_degenerate():
    dpt, _ = _mods()
    m = dpt.DPTDepthModel()
    out = m.forward(((_image(5) - 0.5) / 0.5).cuda())
    frac = float((out > 0).double().mean())
    print(f"stand-in weights: {frac:.3f} positive pixels, std {float(out.std()):.3e}")
    assert frac > 0.2 and float(out.std()) > 0 and bool(torch.isfinite(out).all())


def _main_py_restated(depth_model, ori_imgs, depth_mask, workspace):
    """main.py:120-125 and 196-214, line by line, with DPT/util/io.py's write_depth_name(bits=2) (its .pfm side file aside) and a real
    uint16 PNG round trip (cv2 writes, cv2 reads; imageio reads the same uint16 array)"""
    import os

    import cv2
    import torchvision.transforms as T
    from scipy.ndimage import median_filter
    device = ori_imgs.device
    depth_transform = T.Compose([T.Resize((384, 384)), T.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])

    def write_depth_name(path, depth, bits=1):
        depth_min = depth.min()
        depth_max = depth.max()
        max_val = (2 ** (8 * bits)) - 1
        if depth_max - depth_min > np.finfo("float").eps:
            out = max_val * (depth - depth_min) / (depth_max - depth_min)
        else:
            out = np.zeros(depth.shape, dtype=depth.dtype)
        cv2.imwrite(path + ".png", out.astype("uint16"), [cv2.IMWRITE_PNG_COMPRESSION, 0])

    with torch.no_grad():
        depth_prediction = depth_model.forward(depth_transform(ori_imgs))
        depth_prediction = torch.nn.functional.interpolate(depth_prediction.unsqueeze(1), size=512, mode="bicubic", align_corners=True)
        write_depth_name(os.path.join(workspace, "x_depth"), depth_prediction.squeeze().cpu().numpy(), bits=2)
        disparity = cv2.imread(os.path.join(workspace, "x_depth.png"), cv2.IMREAD_UNCHANGED) / 65535.
        disparity = median_filter(disparity, size=5)
        depth = 1. / np.maximum(disparity, 1e-2)
    depth_prediction = torch.tensor(depth, device=device)
    depth_mask = depth_mask.clone()
    depth_prediction = depth_prediction * (~depth_mask) + torch.ones_like(depth_prediction) * (depth_mask)
    depth_prediction = ((depth_prediction - 1.0) / (depth_prediction.max() - 1.0)) * 0.9 + 0.1
    return depth_prediction


class _Oracle:
    def __init__(self, p):
        self.p = p

    def forward(self, x):
        return dpt_ref.forward(self.p, x)


def test_reference_depth_matches_main_py(setup, tmp_path):
    pytest.importorskip("cv2")
    dpt, _ = _mods()
    model, _, p = setup[:3]
    ori = _image(6, hw=512).cuda()
    yy, xx = torch.meshgrid(torch.arange(512), torch.arange(512), indexing="ij")
    mask = (((yy - 256) ** 2 + (xx - 240) ** 2) > 180 ** 2)[None, None].cuda()
    want = _main_py_restated(_Oracle(p), ori, mask, str(tmp_path))
    # the pipeline alone, on the oracle's own output: exact
    got = dpt.reference_depth(_Oracle(p), ori, mask)
    assert got.shape == want.shape == (1, 1, 512, 512) and got.dtype == want.dtype == torch.float64
    assert torch.equal(got, want)
    # and on the engine
    got = dpt.reference_depth(model, ori, mask)
    e = _rel(got, want)
    print(f"reference_depth on the engine vs main.py on the fp32 oracle: rel-L2 {e:.3e}")
    assert bool(torch.isfinite(got).all()) and e < 5e-2
    assert float(got[mask].min()) == float(got[mask].max())      # the mask fill
