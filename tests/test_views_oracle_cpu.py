"""CPU: oracle/views_ref.py (load_views with numpy morphology and Canny) against the reference's own load_views run with the real cv2
(tests/golden/load_views_ref.npz): every mask and point count exactly, positions within 1e-12 relative, colours within 1e-6."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import views_ref as vr


@pytest.fixture(scope="module")
def gold():
    return load_golden("load_views_ref.npz")


def case(gold, name):
    return {k[len(name) + 1:]: v for k, v in gold.items() if k.startswith(name + "_")}


def check_quant(q, ref):
    """uint8(render * 255) of the canonical cloud.  render_point agrees with the reference's pytorch3d glue to 1e-6, not bit for bit
    (sqrt against pow(0.5) in the alpha), so a code whose product lands on an integer can differ by one (254 / 255 on fully covered
    pixels).  What the mask uses is the test code / 255 > 0.9, i.e. code >= 230: that must agree everywhere."""
    assert q.shape == ref.shape and np.abs(q.astype(int) - ref.astype(int)).max() <= 1
    assert np.array_equal(q >= 230, ref >= 230) and np.array_equal(q / 255 > 0.9, q >= 230)
    assert (ref >= 230).any() and ((ref > 0) & (ref < 230)).any()


def close(a, b, rel):
    assert a.shape == b.shape
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)) <= rel if a.size else True


@pytest.mark.parametrize("k", [3, 11, 15])
@pytest.mark.parametrize("j", [0, 1, 2])
def test_morphology_matches_cv2(gold, j, k):
    im = gold[f"rand{j}_img"]
    assert np.array_equal(vr.erode(im, k), gold[f"rand{j}_erode{k}"])
    assert np.array_equal(vr.dilate(im, k), gold[f"rand{j}_dilate{k}"])
    assert np.array_equal(vr.erode(im, 21), gold[f"rand{j}_erode11x2"])


@pytest.mark.parametrize("t", [10, 30])
@pytest.mark.parametrize("j", [0, 1, 2])
def test_canny_matches_cv2(gold, j, t):
    e = gold[f"rand{j}_canny{t}"]
    assert (e > 0).any()
    assert np.array_equal(vr.canny(gold[f"rand{j}_img"], t), e)


def test_depth_blur_wraps_like_numpy():
    d = np.array([300.7, 700.0, 0.5, 1.0]) / 255.0
    assert vr.depth_blur(d * 255.0 / 255.0, np.ones(4, bool)).tolist() == np.array([300.7, 700.0, 0.5, 1.0]).astype(np.uint8).tolist()
    assert vr.depth_blur(np.array([300.7 / 255.0]), np.ones(1, bool))[0] == 44


@pytest.mark.parametrize("name", ["a", "b"])
def test_load_views_matches_reference(gold, name):
    g = case(gold, name)
    n, S = g["poses"].shape[0], g["depth"].shape[1]
    rec = {}
    vc, cc, vn, cn = vr.load_views_ref(g["gt_u8"] / 255., list(g["depth"]), list(g["mask"]), list(g["rgb"]), g["poses"], S, S, g["K"], 2, 8,
                                       record=rec)
    assert np.array_equal(rec["cano_mask"], g["cano_mask"])
    for key in ("eroded", "canny", "dilated"):
        assert np.array_equal(np.stack(rec[key]), g[key]), key
    check_quant(np.stack(rec["quant"]), g["quant"])
    assert np.array_equal(np.stack(rec["mask"]), g["final_mask"])
    assert (g["canny"] > 0).any() and (g["eroded"] & (g["dilated"] == 255)).any()             # the edges remove masked pixels
    if name == "b":
        assert len(vn) < int(np.stack(rec["mask"]).sum())            # the canonical-depth test drops points
    assert vc.shape == g["v_cano"].shape and vn.shape == g["v_novel"].shape
    assert vc.dtype == np.float64 and cc.dtype == np.float32 and vn.dtype == np.float64 and cn.dtype == np.float32
    assert close(vc, g["v_cano"], 1e-12) and close(vn, g["v_novel"], 1e-12)
    assert np.abs(cc - g["c_cano"]).max() <= 1e-6 and np.abs(cn - g["c_novel"]).max() <= 1e-6
    assert n == len(rec["mask"]) + 1


def test_subsample_matches_reference(gold):
    g = case(gold, "b")
    S = g["depth"].shape[1]
    np.random.seed(7)
    _, _, vn, cn = vr.load_views_ref(g["gt_u8"] / 255., list(g["depth"]), list(g["mask"]), list(g["rgb"]), g["poses"], S, S, g["K"], 2, 8,
                                     npoint=int(g["sub_npoint"]))
    assert close(vn, g["sub_v"], 1e-12) and np.abs(cn - g["sub_c"]).max() <= 1e-6
