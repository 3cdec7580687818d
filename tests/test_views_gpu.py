"""GPU checks of the refine stage's point-cloud construction (csrc/views.cu behind nerf/refine_utils.load_views) against the reference's
own load_views run with the real cv2 (tests/golden/load_views_ref.npz):
- the mask kernels against the recorded erode / Canny / dilate outputs and masks, bit for bit;
- load_views end to end: the same points in the same order, positions within 1e-12 relative, colours within 1e-6;
- the npoint subsample against the recorded seeded multidepth2point_mask call; outputdir untouched; rejected inputs."""
import importlib
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import views_ref as vr
from test_views_oracle_cpu import case, check_quant, close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ru():
    return importlib.import_module("make-it-3d_b200.nerf.refine_utils")


@pytest.fixture(scope="module")
def gold():
    return load_golden("load_views_ref.npz")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def write_folder(g, root):
    """the golden case's decoded images written back as the mvimg folder Trainer.test leaves (PNG is lossless)"""
    import cv2
    os.makedirs(root, exist_ok=True)
    files = {"rgb": [], "depth": [], "mask": []}
    for i in range(g["poses"].shape[0]):
        for kind, im in (("depth", g["depth"][i]), ("mask", g["mask"][i]), ("rgb", g["rgb"][i][..., ::-1])):
            f = os.path.join(root, f"{i:04d}_{kind}.png")
            cv2.imwrite(f, np.ascontiguousarray(im))
            files[kind].append(f)
    return files


def blur_codes():
    """for each uint8 code b, a uint16 depth whose np.uint8(depth / 1000 * 255) is b"""
    d = np.arange(1001)
    b = vr.depth_blur(d / 1000.0, np.ones_like(d, bool))
    table = np.zeros(256, np.uint16)
    for code in range(256):
        table[code] = d[np.nonzero(b == code)[0][0]]
    assert np.array_equal(vr.depth_blur(table / 1000.0, np.ones(256, bool)), np.arange(256))
    return table


@pytest.mark.parametrize("name", ["a", "b"])
def test_mask_kernels_match_reference(ru, gold, name):
    g = case(gold, name)
    n, S = g["poses"].shape[0], g["depth"].shape[1]
    ind = (n - 1) // 2
    V = ru._Views(S, g["K"], torch.device("cuda"))
    cano_depth = torch.empty(S, S, device="cuda")
    m = V.mask(cu(g["depth"][ind]), cu(g["mask"][ind]), 21, -1, masked_depth=cano_depth)
    assert np.array_equal(m.cpu().numpy().astype(bool), g["cano_mask"])
    want = (g["depth"][ind] / 1000.0 * g["cano_mask"]).astype(np.float32)
    assert np.array_equal(cano_depth.cpu().numpy(), want)
    others = [i for i in range(n) if i != ind]
    for j, i in enumerate(others):
        er, ed, dl = (torch.empty(S, S, dtype=torch.uint8, device="cuda") for _ in range(3))
        out = V.mask(cu(g["depth"][i]), cu(g["mask"][i]), 11, 10, eroded=er, edges=ed, dilated=dl)
        assert np.array_equal(er.cpu().numpy() == 255, g["eroded"][j])
        assert np.array_equal(ed.cpu().numpy(), g["canny"][j])
        assert np.array_equal(dl.cpu().numpy(), g["dilated"][j])
        assert np.array_equal(out.cpu().numpy().astype(bool), g["eroded"][j] & ~(g["dilated"][j] == 255))


@pytest.mark.parametrize("name", ["a", "b"])
def test_cover_mask_matches_reference(ru, gold, name):
    """the canonical cloud (the recorded one) rendered into each view, quantised, eroded 15 x 15 and thresholded"""
    g = case(gold, name)
    n, S = g["poses"].shape[0], g["depth"].shape[1]
    ind = (n - 1) // 2
    V = ru._Views(S, g["K"], torch.device("cuda"))
    v32 = cu(g["v_cano"]).float()
    K32 = cu(g["K"]).float()
    for j, i in enumerate(i for i in range(n) if i != ind):
        w2c = np.linalg.inv(g["poses"][i])
        render = ru.render_point(v32, torch.ones(v32.shape[0], 1, device="cuda"), S, S, K32, cu(w2c), [S, S], 2.0 / S * 2.0, 8)
        alpha = V.mask(cu(g["depth"][i]), cu(g["mask"][i]), 11, 10)
        q = torch.empty(S, S, dtype=torch.uint8, device="cuda")
        out = V.cover(render.contiguous(), alpha, quant=q)
        check_quant(q.cpu().numpy(), g["quant"][j])
        assert np.array_equal(out.cpu().numpy().astype(bool), g["final_mask"][j])


@pytest.mark.parametrize("j", [0, 1, 2])
def test_erode_and_canny_on_random_images(ru, gold, j):
    im = gold[f"rand{j}_img"]
    h, w = im.shape
    s = min(h, w)
    im = np.ascontiguousarray(im[:s, :s])
    V = ru._Views(s, np.eye(3), torch.device("cuda"))
    er = torch.empty(s, s, dtype=torch.uint8, device="cuda")
    ones = np.full((s, s), 255, np.uint8)
    for k in (3, 11, 15, 21):
        V.mask(cu(np.zeros((s, s), np.uint16)), cu(im), k, -1, eroded=er)
        assert np.array_equal(er.cpu().numpy(), vr.erode(im, k))
    ed = torch.empty(s, s, dtype=torch.uint8, device="cuda")
    for t in (10, 30):
        V.mask(cu(blur_codes()[im]), cu(ones), 3, t, edges=ed)
        assert np.array_equal(ed.cpu().numpy(), vr.canny(im, t))
    assert np.array_equal(vr.canny(gold[f"rand{j}_img"], 10), gold[f"rand{j}_canny10"])


@pytest.mark.parametrize("name", ["a", "b"])
def test_load_views_matches_reference(ru, gold, name, tmp_path):
    g = case(gold, name)
    S = g["depth"].shape[1]
    f = write_folder(g, str(tmp_path / "mvimg"))
    outdir = tmp_path / "refine"
    outdir.mkdir()
    vc, cc, vn, cn = ru.load_views(g["gt_u8"] / 255., f["rgb"], f["depth"], f["mask"], g["poses"], S, S, g["K"], 2, 8, str(outdir), "cuda")
    assert os.listdir(outdir) == []
    assert vc.dtype == np.float64 and cc.dtype == np.float32 and vn.dtype == np.float64 and cn.dtype == np.float32
    assert vc.shape == g["v_cano"].shape and vn.shape == g["v_novel"].shape
    print(f"{name}: cano {len(vc)}, novel {len(vn)}; max |d v| {np.abs(vn - g['v_novel']).max():.2e}, "
          f"max |d c| {np.abs(cn - g['c_novel']).max():.2e}")
    assert close(vc, g["v_cano"], 1e-12) and close(vn, g["v_novel"], 1e-12)
    assert np.abs(cc - g["c_cano"]).max() <= 1e-6 and np.abs(cn - g["c_novel"]).max() <= 1e-6


def test_subsample_matches_reference(ru, gold, tmp_path):
    g = case(gold, "b")
    S = g["depth"].shape[1]
    f = write_folder(g, str(tmp_path / "mvimg"))
    np.random.seed(7)
    _, _, vn, cn = ru.load_views(g["gt_u8"] / 255., f["rgb"], f["depth"], f["mask"], g["poses"], S, S, g["K"], 2, 8, str(tmp_path), "cuda",
                                 npoint=int(g["sub_npoint"]))
    assert vn.shape == g["sub_v"].shape
    assert close(vn, g["sub_v"], 1e-12) and np.abs(cn - g["sub_c"]).max() <= 1e-6


def test_rejected_inputs(ru, gold, tmp_path):
    Mi3dError = importlib.import_module("make-it-3d_b200._lib").Mi3dError
    g = case(gold, "a")
    S = g["depth"].shape[1]
    f = write_folder(g, str(tmp_path / "mvimg"))
    args = (g["gt_u8"] / 255., f["rgb"], f["depth"], f["mask"], g["poses"], S, S, g["K"], 2, 8, str(tmp_path))
    with pytest.raises(Mi3dError):                      # not CUDA
        ru.load_views(*args, "cpu")
    with pytest.raises(Mi3dError):                      # non-square
        ru.load_views(g["gt_u8"] / 255., f["rgb"], f["depth"], f["mask"], g["poses"], S, S + 8, g["K"], 2, 8, str(tmp_path), "cuda")
    with pytest.raises(Mi3dError):                      # views at another size than H x W
        ru.load_views(np.zeros((2 * S, 2 * S, 3)), f["rgb"], f["depth"], f["mask"], g["poses"], 2 * S, 2 * S, g["K"], 2, 8, str(tmp_path),
                      "cuda")
    with pytest.raises(Mi3dError):                      # fewer than 2 views
        ru.load_views(args[0], f["rgb"][:1], f["depth"][:1], f["mask"][:1], g["poses"][:1], S, S, g["K"], 2, 8, str(tmp_path), "cuda")
