"""CPU: oracle/unet_ref.py (the restatement of the reference's gated U-Net the GPU tests compare against) pinned to
tests/golden/unet_ref.npz, recorded from the reference's own nerf/unet.py; the native module's state_dict layout and argument errors;
the ctypes mirror of mi3d_unet_shape."""
import ctypes
import importlib
import os
import re

import numpy as np
import pytest
import torch

from oracle import unet_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "unet_ref.npz")


def _golden():
    spec = importlib.util.spec_from_file_location("make_golden_unet", os.path.join(ROOT, "tests", "golden", "make_golden_unet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    z = np.load(GOLDEN)
    return z, *mod.decode(z)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_oracle_matches_reference_fixture():
    z, params, xs, w = _golden()
    p = {k: (v.double() if v.is_floating_point() else v.clone()) for k, v in params.items()}
    names = unet_ref.param_names()
    for n in names:
        p[n].requires_grad_(True)
    xr = [x.double().requires_grad_(True) for x in xs]
    out = unet_ref.unet(xr, p, train=True)
    (out * w.double()).sum().backward()
    assert _rel(out.detach(), z["out"]) <= 1e-5
    for i in range(3):
        assert _rel(xr[i].grad, z[f"dx{i}"]) <= 1e-5, i
    for n in names:
        assert _rel(p[n].grad, z["grad/" + n]) <= 1e-5, n
    for n in unet_ref.state_names():
        if n not in names:
            if n.endswith("num_batches_tracked"):
                assert int(p[n]) == int(z["after/" + n])
            else:
                assert _rel(p[n].detach(), z["after/" + n]) <= 1e-5, n
    with torch.no_grad():
        ev = unet_ref.unet([x.double() for x in xs], {k: v.detach() for k, v in p.items()}, train=False)
    assert _rel(ev, z["eval_out"]) <= 1e-5


def test_fixture_layout():
    z, params, _, _ = _golden()
    assert [str(n) for n in z["names"]] == unet_ref.state_names()
    assert len(params) == 41
    assert sum(params[n].numel() for n in unet_ref.param_names()) == 104_747
    assert os.path.getsize(GOLDEN) < 1_100_000


def test_native_module_state_dict():
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    torch.manual_seed(0)
    net = um.UNet(num_input_channels=3 + 16)
    sd = net.state_dict()
    z = np.load(GOLDEN)
    assert list(sd.keys()) == [str(n) for n in z["names"]]
    for n, shp in zip(sd.keys(), z["shapes"]):
        assert tuple(sd[n].shape) == tuple(int(s) for s in shp if s > 0), n
    assert sum(p.numel() for p in net.parameters()) == 104_747
    # the oracle's registry has the same names and shapes (the values of the default initialisation are compared with the reference's
    # module itself in test_native_module_default_init_matches_reference_module)
    ref = unet_ref.seeded_params(0)
    assert set(ref) == set(sd)
    assert all(tuple(ref[n].shape) == tuple(sd[n].shape) for n in sd)


def test_native_module_default_init_matches_reference_module():
    ref_dir = os.environ.get("MI3D_REFERENCE_DIR")
    if not ref_dir:
        pytest.skip("MI3D_REFERENCE_DIR not set")
    spec = importlib.util.spec_from_file_location("ref_unet", os.path.join(ref_dir, "nerf", "unet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    torch.manual_seed(5)
    a = um.UNet(num_input_channels=19).state_dict()
    torch.manual_seed(5)
    b = mod.UNet(num_input_channels=19).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("kw", [dict(num_input_channels=3), dict(num_input_channels=19, num_output_channels=4),
                                dict(num_input_channels=19, feature_scale=2), dict(num_input_channels=19, upsample_mode="nearest"),
                                dict(num_input_channels=19, upsample_mode="deconv"), dict(num_input_channels=19, last_act="tanh"),
                                dict(num_input_channels=19, conv_block="basic")])
def test_constructor_errors(kw):
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    L = importlib.import_module("make-it-3d_b200._lib")
    with pytest.raises(L.Mi3dError):
        um.UNet(**kw)


def test_argument_errors_without_gpu():
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    L = importlib.import_module("make-it-3d_b200._lib")
    net = um.UNet(num_input_channels=19)
    xs = [torch.rand(1, 19, 16 >> i, 16 >> i) for i in range(3)]
    with pytest.raises(L.Mi3dError):            # CPU tensors
        net(xs)
    with pytest.raises(L.Mi3dError):            # two scales
        net(xs[:2])


def test_shape_struct_matches_header():
    um = importlib.import_module("make-it-3d_b200.nerf.unet")
    hdr = open(os.path.join(ROOT, "include", "mi3d.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} mi3d_unet_shape;", hdr).group(1)
    fields = re.findall(r"int\s+([\w, ]+);", body)
    names = [f.strip() for grp in fields for f in grp.split(",")]
    assert names == [f for f, _ in um.UNetCfg._fields_]
    assert ctypes.sizeof(um.UNetCfg) == 4 * len(names)
