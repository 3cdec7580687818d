"""CPU checks of the point-renderer oracle (oracle/points_ref.py): it reproduces the reference's own render_point glue and z_buffer
(tests/golden/points_ref.npz), its vectorised and loop-form rasterisers agree, and hand cases pin the conventions."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import points_ref as pr


@pytest.fixture(scope="module")
def gold():
    return load_golden("points_ref.npz")


@pytest.mark.parametrize("case", ["a", "b"])
def test_oracle_reproduces_reference_glue(gold, case):
    g = pr.golden_case(gold, case + "_")
    S, radius = int(g["S"]), float(g["radius"])
    feats = torch.from_numpy(g["feats"])
    # on the cloud the reference's glue projected: the same image bit for bit
    ndc = torch.from_numpy(g["ndc"])
    idx_g, _, d2_g = pr.rasterize_ndc(ndc[:, 0], ndc[:, 1], ndc[:, 2], S, radius, 8)
    img_g, _ = pr.composite(idx_g, d2_g, feats, radius)
    assert torch.equal(img_g, torch.from_numpy(g["image"]))
    # with the oracle's own fixed-order projection: the same slots almost everywhere, the same image there
    image, idx, _, _, _ = pr.render_point_ref(torch.from_numpy(g["points"]), feats, S, S, torch.from_numpy(g["K"]),
                                              torch.from_numpy(g["w2c"]), [S, S], radius, 8)
    same = (idx == idx_g).all(-1)
    assert same.float().mean() >= 0.999, float(same.float().mean())
    err = (image[0] - torch.from_numpy(g["image"])[0]).abs().amax(0)[same]
    assert float(err.max()) <= 1e-5


@pytest.mark.parametrize("case", ["depth", "rand0", "rand1"])
def test_zbuffer_oracle_matches_reference(gold, case):
    g = pr.golden_case(gold, f"zb_{case}_")
    S = int(g["S"])
    mask = pr.z_buffer_ref(g["v"], g["w2c"], S, S, g["K"])
    assert np.array_equal(mask, g["mask"])


def test_loop_and_vectorised_rasterisers_agree():
    rng = np.random.default_rng(7)
    P, S, K = 60, 12, 3
    px = rng.uniform(-1.1, 1.1, P).astype(np.float32)
    py = rng.uniform(-1.1, 1.1, P).astype(np.float32)
    pz = rng.uniform(-0.2, 2.0, P).astype(np.float32)
    pz[5:10] = pz[4]                                # exact z ties
    px[20:24], py[20:24] = px[19], py[19]           # stacked points
    radius = 0.3
    idx_v, _, _ = pr.rasterize_ndc(*(torch.from_numpy(a) for a in (px, py, pz)), S, radius, K)
    idx_l = pr.rasterize_ndc_loop(px, py, pz, S, radius, K)
    assert (idx_l[..., -1] >= 0).sum() > 10          # queues overflowed somewhere
    assert np.array_equal(idx_v.numpy(), idx_l)


def _ndc_of_pixel(S, yi, xi):
    """NDC position of the centre of pixel (yi, xi), as a projected point"""
    c = pr.pixel_centres(S)
    return c[xi], c[yi]


def _one(px, py, pz, S=8, radius=0.3, K=2):
    t = lambda a: torch.tensor(a, dtype=torch.float32)
    return pr.rasterize_ndc(t(px), t(py), t(pz), S, radius, K)


def test_point_at_pixel_centre_has_zero_distance():
    x, y = _ndc_of_pixel(8, 2, 5)
    idx, zb, d2 = _one([float(x)], [float(y)], [1.5])
    assert idx[2, 5, 0] == 0 and d2[2, 5, 0] == 0 and zb[2, 5, 0] == 1.5


def test_not_mirrored():
    # pixel coordinates u = xi + 0.5, v = yi + 0.5 land on pixel (yi, xi): project a point through K and an identity pose
    S = 16
    K = torch.tensor([[20.0, 0, 8.0], [0, 20.0, 8.0], [0, 0, 1]])
    w2c = torch.eye(4)[:3]
    xi, yi, z = 3, 11, 2.0
    p = torch.tensor([[(xi + 0.5 - 8.0) * z / 20.0, (yi + 0.5 - 8.0) * z / 20.0, z]])
    _, idx, _, d2, _ = pr.render_point_ref(p, torch.ones(1, 1), S, S, K, w2c, [S, S], 0.5 / S, 1)
    hit = (idx[..., 0] >= 0).nonzero().tolist()
    assert hit == [[yi, xi]] and float(d2[yi, xi, 0]) < 1e-10


def test_behind_camera_is_culled():
    x, y = _ndc_of_pixel(8, 4, 4)
    idx, _, _ = _one([float(x)] * 2, [float(y)] * 2, [-0.5, 3.0])
    assert idx[4, 4].tolist() == [1, -1]


def test_farthest_of_three_dropped_with_k2():
    x, y = _ndc_of_pixel(8, 3, 3)
    idx, zb, _ = _one([float(x)] * 3, [float(y)] * 3, [2.0, 3.0, 1.0])
    assert idx[3, 3].tolist() == [2, 0] and zb[3, 3].tolist() == [1.0, 2.0]


def test_exact_z_tie_goes_to_lower_index():
    x, y = _ndc_of_pixel(8, 1, 6)
    idx, _, _ = _one([float(x)] * 3, [float(y)] * 3, [1.0, 1.0, 1.0])
    assert idx[1, 6].tolist() == [0, 1]
    idx_l = pr.rasterize_ndc_loop([float(x)] * 3, [float(y)] * 3, [1.0] * 3, 8, 0.3, 2)
    assert idx_l[1, 6].tolist() == [0, 1]
