"""CPU: the marching-cubes / atlas oracle (oracle/mesh_ref.py) that the GPU mesh export is checked against."""
import math

import numpy as np
import pytest

from oracle import mesh_ref as M


def _grid(n):
    g = np.linspace(-1, 1, n).astype(np.float32)
    return np.meshgrid(g, g, g, indexing="ij")


def _cube_faces():
    return [frozenset(m for m in range(8) if M.CORNERS[m][a] == s) for a in range(3) for s in (0, 1)]


def test_triangle_table_all_256_cases():
    """Each row uses exactly the crossing edges of its corner pattern; inside the cube every triangle edge is shared by exactly two
    of the row's triangles, in opposite directions (edges on a cube face belong to one triangle)."""
    faces = _cube_faces()
    for ci, row in enumerate(M.TRI_TABLE):
        outside = [(ci >> m) & 1 for m in range(8)]
        crossing = {e for e in range(12) if outside[M.EDGE_CORNERS[e, 0]] != outside[M.EDGE_CORNERS[e, 1]]}
        assert len(row) % 3 == 0 and len(row) <= 15, ci
        assert set(row) == crossing, ci
        use = {}
        for k in range(0, len(row), 3):
            a, b, c = row[k:k + 3]
            assert len({a, b, c}) == 3, ci
            for e in ((a, b), (b, c), (c, a)):
                use.setdefault(frozenset(e), []).append(e)
        for key, dirs in use.items():
            a, b = tuple(key)
            on_face = any(set(M.EDGE_CORNERS[a]) <= f and set(M.EDGE_CORNERS[b]) <= f for f in faces)
            if on_face:
                assert len(dirs) == 1, (ci, dirs)
            else:
                assert len(dirs) == 2 and dirs[0] == dirs[1][::-1], (ci, dirs)


def test_table_winding_points_out_of_the_solid():
    """case 1 (only corner 0 outside): the triangle's right-hand normal points toward corner 0"""
    mid = {e: (M.CORNERS[M.EDGE_CORNERS[e, 0]] + M.CORNERS[M.EDGE_CORNERS[e, 1]]) / 2 for e in range(12)}
    a, b, c = (mid[e] for e in M.TRI_TABLE[1])
    nrm = np.cross(b - a, c - a)
    assert np.dot(nrm, np.zeros(3) - a) > 0


def test_sphere_closed_genus0_volume_and_exact_vertices():
    X, Y, Z = _grid(64)
    r = 0.5
    vol = (r - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32)
    v, f = M.marching_cubes(vol, 0.0)
    assert len(f) > 1000
    assert M.is_closed_oriented(f)
    assert M.euler_characteristic(v, f) == 2
    h = 2.0 / 63
    vol_mesh = M.signed_volume(v * h, f)
    assert vol_mesh > 0 and abs(vol_mesh - 4 / 3 * math.pi * r ** 3) / (4 / 3 * math.pi * r ** 3) < 0.01
    # every vertex lies on its grid edge, at the fp32 interpolation point of the iso crossing
    ijk = np.floor(v).astype(np.int64)
    frac = v - ijk
    axis = np.argmax(frac, axis=1)
    assert ((frac > 0).sum(1) <= 1).all()
    s0 = vol[ijk[:, 0], ijk[:, 1], ijk[:, 2]]
    nb = ijk.copy()
    nb[np.arange(len(v)), axis] += 1
    s1 = vol[nb[:, 0], nb[:, 1], nb[:, 2]]
    assert ((s0 > 0) != (s1 > 0)).all()
    t = (np.float32(0) - s0) / (s1 - s0)
    np.testing.assert_array_equal(frac[np.arange(len(v)), axis], (ijk[np.arange(len(v)), axis].astype(np.float32) + t)
                                  - ijk[np.arange(len(v)), axis].astype(np.float32))


def test_torus_euler_characteristic_zero():
    X, Y, Z = _grid(64)
    vol = (0.2 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.5) ** 2 + Z ** 2)).astype(np.float32)
    v, f = M.marching_cubes(vol, 0.0)
    assert M.is_closed_oriented(f)
    assert M.euler_characteristic(v, f) == 0


@pytest.mark.parametrize("seed", range(6))
def test_random_volumes_closed_and_oriented(seed):
    """white-noise volumes visit every table row many times in every neighbourhood: a wrong row opens or flips the surface"""
    rng = np.random.default_rng(seed)
    vol = rng.standard_normal((14, 11, 17)).astype(np.float32)
    for sl in (np.s_[0], np.s_[-1]):
        vol[sl] = -1
        vol[:, sl] = -1
        vol[:, :, sl] = -1
    v, f = M.marching_cubes(vol, 0.25)
    assert len(f) > 100
    assert M.is_closed_oriented(f)
    assert M.signed_volume(v, f) > 0
    assert np.unique(f).size == len(v)                       # every vertex is used


def test_numbering_is_point_major_axis_minor():
    vol = np.zeros((3, 3, 3), np.float32)
    vol[1, 1, 1] = 1
    v, f = M.marching_cubes(vol, 0.5)
    # owners (0,1,1) x, (1,0,1) y, (1,1,0) z, then (1,1,1) x, y, z
    expect = np.array([[0.5, 1, 1], [1, 0.5, 1], [1, 1, 0.5], [1.5, 1, 1], [1, 1.5, 1], [1, 1, 1.5]], np.float32)
    np.testing.assert_array_equal(v, expect)
    assert len(f) == 8 and M.is_closed_oriented(f) and M.signed_volume(v, f) > 0


@pytest.mark.parametrize("F,T,c", [(1, 2048, 2048), (2, 2048, 2048), (131072, 2048, 8), (131073, 4096, 15)])
def test_atlas_layout(F, T, c):
    assert M.atlas_layout(F)[:2] == (T, c)


def test_atlas_layout_limit():
    with pytest.raises(ValueError):
        M.atlas_layout(2 * 2049 ** 2)


def _cheb_dist_to_triangle(p, tri):
    """Chebyshev distance from point p to a filled triangle (dense sampling of the triangle is exact enough at these sizes)"""
    w = np.stack(np.meshgrid(np.linspace(0, 1, 201), np.linspace(0, 1, 201), indexing="ij"), -1).reshape(-1, 2)
    w = w[w.sum(1) <= 1]
    q = tri[0] + w[:, :1] * (tri[1] - tri[0]) + w[:, 1:] * (tri[2] - tri[0])
    return np.abs(q - p).max(1).min()


def test_atlas_owner_rule():
    """a texel belongs to the face whose UV triangle its centre is within Chebyshev distance < 1 of, else to none"""
    F, T, c, n = 7, 64, 12, 2
    own = M.atlas_owner(T, c, n, F)
    uv = M.atlas_uv_corners(c).astype(np.float64)
    for r in range(0, 2 * c):
        for x in range(0, 2 * c):
            ctr = np.array([x + 0.5, r + 0.5])
            cell = (r // c) * n + x // c
            org = np.array([(x // c) * c, (r // c) * c], np.float64)
            hits = [2 * cell + s for s in (0, 1) if 2 * cell + s < F and _cheb_dist_to_triangle(ctr, org + uv[s]) < 1 - 1e-9]
            assert len(hits) <= 1
            assert own[r, x] == (hits[0] if hits else -1), (r, x)
    assert (own[2 * c:, :] == -1).all() and (own[:, 2 * c:] == -1).all()


@pytest.mark.parametrize("c", [8, 9, 15, 40])
def test_atlas_bilinear_footprint_stays_in_face(c):
    rng = np.random.default_rng(c)
    n, F = 3, 17
    T = 4 * c
    own = M.atlas_owner(T, c, n, F)
    uv = M.atlas_uv_corners(c).astype(np.float64)
    for f in range(F):
        cell = f // 2
        org = np.array([(cell % n) * c, (cell // n) * c], np.float64)
        tri = org + uv[f & 1]
        w = rng.random((200, 2))
        w[w.sum(1) > 1] = 1 - w[w.sum(1) > 1]
        p = tri[0] + w[:, :1] * (tri[1] - tri[0]) + w[:, 1:] * (tri[2] - tri[0])      # texel units (u, v)
        x0 = np.floor(p[:, 0] - 0.5).astype(int)
        r0 = np.floor(p[:, 1] - 0.5).astype(int)
        for dx in (0, 1):
            for dr in (0, 1):
                assert (own[r0 + dr, x0 + dx] == f).all(), f


def test_atlas_texel_points_and_vt():
    rng = np.random.default_rng(0)
    v = rng.uniform(-0.9, 0.9, (40, 3)).astype(np.float32)
    f = rng.integers(0, 40, (9, 3)).astype(np.int32)
    T, c, n = 64, 12, 3
    pts, own, vt = M.atlas_texels(v, f, T, c, n, bound=1.0)
    assert vt.shape == (27, 2)
    # the UV corners map back onto the face's vertices exactly enough, and owned points interpolate the face affinely
    for face in range(9):
        r, x = np.nonzero(own == face)
        assert len(r) > 0
        tri = vt[3 * face:3 * face + 3] * T
        ctr = np.stack([x + 0.5, r + 0.5], -1)
        A = np.stack([tri[1] - tri[0], tri[2] - tri[0]], -1)
        b = np.linalg.solve(A, (ctr - tri[0]).T).T
        expect = v[f[face, 0]] + b[:, :1] * (v[f[face, 1]] - v[f[face, 0]]) + b[:, 1:] * (v[f[face, 2]] - v[f[face, 0]])
        np.testing.assert_allclose(pts[r, x], np.clip(expect, -1, 1), atol=2e-6)
    assert (pts[own < 0] == 0).all()
