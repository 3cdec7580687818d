"""CPU restatement of the refine stage's point renderer (reference nerf/refine_utils.py:306-333 over pytorch3d's naive
`rasterize_points` and `alpha_composite`) and of its z_buffer (refine_utils.py:167-208), in the fp32 / fp64 op order that
csrc/points.cu evaluates, so slot selection and distances can be compared bit for bit.  Test infrastructure only.

pytorch3d is not available here, so its semantics are restated twice: `rasterize_ndc` (vectorised: every point's candidate pixel
window, then a sort by (pixel, z, index)) and `rasterize_ndc_loop` (per-pixel bounded priority queue, the structure of pytorch3d's
naive kernel).  The two agree on `idx`; parity with the real package is not pinned.
"""
import numpy as np
import torch


def project_ndc(points, K, world2cam, H, W):
    """fp32 [P,3] -> (x_ndc, y_ndc, z): c = R p + t, q = K c, u = q.x / q.z, x = -(u / W * 2 - 1), one rounding per op."""
    p = points.to(torch.float32)
    k = K.reshape(3, 3).to(torch.float32)
    rt = world2cam[:3, :4].to(torch.float32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    c = [((rt[r, 0] * x + rt[r, 1] * y) + rt[r, 2] * z) + rt[r, 3] for r in range(3)]
    q = [(k[r, 0] * c[0] + k[r, 1] * c[1]) + k[r, 2] * c[2] for r in range(3)]
    u, v = q[0] / q[2], q[1] / q[2]
    W32, H32 = torch.tensor(float(W), dtype=torch.float32), torch.tensor(float(H), dtype=torch.float32)
    return -((u / W32) * 2.0 - 1.0), -((v / H32) * 2.0 - 1.0), q[2]


def pixel_centres(S):
    """fp32 NDC centre of columns (= rows) 0..S-1: -1 + (2(S-1-i)+1)/S in double, rounded once."""
    i = np.arange(S, dtype=np.float64)
    return torch.from_numpy((-1.0 + (2.0 * (S - 1 - i) + 1.0) / S).astype(np.float32))


def rasterize_ndc(px, py, pz, S, radius, K):
    """naive rasterisation of NDC points: (idx [S,S,K] int64, zbuf, dist2 [S,S,K] fp32), empty slots -1."""
    px, py, pz = px.to(torch.float32), py.to(torch.float32), pz.to(torch.float32)
    r = torch.tensor(radius, dtype=torch.float32)
    rr = r * r
    cen = pixel_centres(S)
    P = px.shape[0]
    ok = ~(pz < 0) & torch.isfinite(px) & torch.isfinite(py)
    # nearest column / row of each point, then a window wide enough for the radius (+ 2 px of slack); the exact test decides
    half = int(np.ceil(float(radius) * S / 2.0)) + 2
    fx = torch.where(ok, ((1.0 - px.double()) * S - 1.0) / 2.0, torch.zeros_like(px, dtype=torch.float64)).round().clamp(-S, 2 * S).long()
    fy = torch.where(ok, ((1.0 - py.double()) * S - 1.0) / 2.0, torch.zeros_like(py, dtype=torch.float64)).round().clamp(-S, 2 * S).long()
    offs = torch.arange(-half, half + 1)
    oy, ox = torch.meshgrid(offs, offs, indexing="ij")
    oy, ox = oy.reshape(-1), ox.reshape(-1)
    ids_all, pix_all, d2_all = [], [], []
    chunk = max(1, (1 << 22) // oy.numel())
    for b in range(0, P, chunk):
        sl = slice(b, min(P, b + chunk))
        xi = fx[sl, None] + ox[None, :]
        yi = fy[sl, None] + oy[None, :]
        inb = (xi >= 0) & (xi < S) & (yi >= 0) & (yi < S) & ok[sl, None]
        dx = cen[xi.clamp(0, S - 1)] - px[sl, None]
        dy = cen[yi.clamp(0, S - 1)] - py[sl, None]
        d2 = dx * dx + dy * dy
        hit = inb & (d2 < rr)
        pid = torch.arange(b, sl.stop)[:, None].expand_as(xi)
        ids_all.append(pid[hit])
        pix_all.append((yi * S + xi)[hit])
        d2_all.append(d2[hit])
    ids, pix, d2 = torch.cat(ids_all), torch.cat(pix_all), torch.cat(d2_all)
    z = pz[ids]
    # sort by (pixel, z, index): stable sorts from the least significant key
    o = torch.argsort(ids, stable=True)
    o = o[torch.argsort(z[o], stable=True)]
    o = o[torch.argsort(pix[o], stable=True)]
    ids, pix, d2, z = ids[o], pix[o], d2[o], z[o]
    first = torch.searchsorted(pix, pix, right=False)
    rank = torch.arange(pix.numel()) - first
    keep = rank < K
    idx = torch.full((S * S, K), -1, dtype=torch.int64)
    zb = torch.full((S * S, K), -1.0, dtype=torch.float32)
    db = torch.full((S * S, K), -1.0, dtype=torch.float32)
    idx[pix[keep], rank[keep]] = ids[keep]
    zb[pix[keep], rank[keep]] = z[keep]
    db[pix[keep], rank[keep]] = d2[keep]
    return idx.reshape(S, S, K), zb.reshape(S, S, K), db.reshape(S, S, K)


def rasterize_ndc_loop(px, py, pz, S, radius, K):
    """the same, written as pytorch3d's naive kernel: per pixel, visit points in index order, keep a bounded queue of K (z, index)."""
    px, py, pz = (np.asarray(a, np.float32) for a in (px, py, pz))
    rr = np.float32(radius) * np.float32(radius)
    cen = pixel_centres(S).numpy()
    idx = np.full((S, S, K), -1, np.int64)
    for yi in range(S):
        for xi in range(S):
            q = []
            for p in range(px.shape[0]):
                if pz[p] < 0:
                    continue
                dx, dy = np.float32(cen[xi] - px[p]), np.float32(cen[yi] - py[p])
                d2 = np.float32(np.float32(dx * dx) + np.float32(dy * dy))
                if not d2 < rr:
                    continue
                if len(q) < K:
                    q.append((pz[p], p))
                else:
                    worst = max(q)
                    if (pz[p], p) < worst:
                        q[q.index(worst)] = (pz[p], p)
            for k, (_, p) in enumerate(sorted(q)):
                idx[yi, xi, k] = p
    return idx


def alphas_from_dist2(dist2, radius):
    """alpha = 1 - sqrt(clamp(fp32(0.1 * dist2) / fp32(radius^2), 1e-3, 1))  (refine_utils.py:320-325)"""
    r2 = torch.tensor(float(radius) ** 2, dtype=torch.float32)
    return 1.0 - torch.sqrt(((dist2 * torch.tensor(0.1, dtype=torch.float32)) / r2).clamp(min=1e-3, max=1.0))


def composite(idx, dist2, feats, radius):
    """front-to-back alpha composite of [S,S,K] slots over feats [P,C] (differentiable in feats) -> (image [1,C,S,S], w [S,S,K])."""
    S, _, K = idx.shape
    a = alphas_from_dist2(dist2, radius)
    valid = idx >= 0
    T = torch.ones(S, S, dtype=torch.float32)
    out = torch.zeros(S, S, feats.shape[1], dtype=torch.float32)
    ws = []
    for k in range(K):
        v = valid[..., k]
        w = torch.where(v, T * a[..., k], torch.zeros_like(T))
        f = feats[idx[..., k].clamp(min=0)]
        out = torch.where(v[..., None], out + w[..., None] * f, out)
        T = torch.where(v, T * (1.0 - a[..., k]), T)
        ws.append(w)
    return out.permute(2, 0, 1)[None], torch.stack(ws, -1)


def decode_feats(feats_u8):
    """fp32 features of the golden fixture's 8-bit codes: code / 255 (one IEEE division, exact on every platform)"""
    return np.asarray(feats_u8).astype(np.float32) / np.float32(255.0)


def golden_case(gold, prefix):
    """the entries of one case of tests/golden/points_ref.npz, prefix stripped, features / clouds decoded to what the reference saw"""
    g = {k[len(prefix):]: v for k, v in gold.items() if k.startswith(prefix)}
    if "feats_u8" in g:
        g["feats"] = decode_feats(g.pop("feats_u8"))
    if "v" in g:
        g["v"] = g["v"].astype(np.float64)
    return g


def render_point_ref(points, feats, H, W, K, world2cam, image_size, radius, ppp):
    """oracle of render_point: (image [1,C,h,w], idx, zbuf, dist2, w); image is differentiable in feats"""
    S = int(image_size[0])
    px, py, pz = project_ndc(points, K, world2cam, H, W)
    idx, zb, d2 = rasterize_ndc(px, py, pz, S, radius, ppp)
    image, w = composite(idx, d2, feats, radius)
    return image, idx, zb, d2, w


def z_buffer_ref(vertices, world2cam, H, W, K):
    """vectorised refine_utils.z_buffer in fp64 (same op order as the kernel): bool mask [P]"""
    v = np.asarray(vertices, np.float64)
    rt = np.asarray(world2cam, np.float64)[:3, :4]
    k = np.asarray(K, np.float64).reshape(3, 3)
    c = [((rt[r, 0] * v[:, 0] + rt[r, 1] * v[:, 1]) + rt[r, 2] * v[:, 2]) + rt[r, 3] for r in range(3)]
    q = [(k[r, 0] * c[0] + k[r, 1] * c[1]) + k[r, 2] * c[2] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, vv = np.rint(q[0] / q[2]), np.rint(q[1] / q[2])
    z = q[2]
    inb = (u >= 0) & (u <= W - 1) & (vv >= 0) & (vv <= H - 1)
    pix = np.where(inb, np.nan_to_num(vv) * W + np.nan_to_num(u), 0).astype(np.int64)
    zbuf = np.full(H * W, np.inf)
    np.minimum.at(zbuf, pix[inb], z[inb])
    with np.errstate(invalid="ignore"):
        return inb & ~((z - zbuf[pix]) > 1.0 / H)


# ---- scene helpers shared by the golden generator, the tests and tests/measure_points.py ----

def intrinsics(S, fov_deg=40.0):
    """K of nerf/utils.py:758-759 at an S x S image"""
    focal = 1 / (2 * np.tan(np.deg2rad(fov_deg) / 2))
    return np.array([[focal * S, 0, 0.5 * S], [0, focal * S, 0.5 * S], [0, 0, 1]], np.float64)


def lookat_c2w(radius, theta_deg, phi_deg):
    """camera-to-world pose looking at the origin, built like fix_poses (nerf/refine_utils.py:285-302); camera +z looks forward"""
    th, ph = np.deg2rad(theta_deg), np.deg2rad(phi_deg)
    centre = np.array([radius * np.sin(th) * np.sin(ph), radius * np.cos(th), radius * np.sin(th) * np.cos(ph)])
    fwd = -centre / np.linalg.norm(centre)
    right = np.cross(fwd, np.array([0.0, -1.0, 0.0]))
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    up /= np.linalg.norm(up)
    pose = np.eye(4)
    pose[:3, :3] = np.stack((right, up, fwd), axis=-1)
    pose[:3, 3] = centre
    return pose


def sphere_depth(c2w, K, S, R=0.5):
    """camera-z depth map [S,S] of a sphere of radius R at the origin (0 where the ray misses) and its mask"""
    ys, xs = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    d = np.stack([xs.ravel(), ys.ravel(), np.ones(S * S)], 0)
    d = (np.linalg.inv(K) @ d).T                     # camera rays with z = 1
    dw = d @ c2w[:3, :3].T
    o = c2w[:3, 3]
    a, b, c = (dw * dw).sum(1), 2 * dw @ o, o @ o - R * R
    disc = b * b - 4 * a * c
    t = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
    return t.reshape(S, S), (disc > 0).reshape(S, S)


def depth_cloud(D, mask, c2w, K):
    """world points of a depth map, built like depth2point (nerf/refine_utils.py:129-139)"""
    x, y = np.meshgrid(np.arange(D.shape[1]), np.arange(D.shape[0]))
    cam = np.vstack((x.reshape(-1), y.reshape(-1), np.ones(D.size)))
    v = np.linalg.inv(K).dot(cam).T * D.reshape(-1, 1)
    v = v[mask.reshape(-1)]
    return np.matmul(v, c2w[:3, :3].T) + c2w[:3, 3:].T


def surface_cloud(n_views, S, seed=0, R=0.5):
    """dense surface cloud: the union of the depth-map clouds of a sphere seen from n_views cameras around it (float32 [P,3])"""
    rng = np.random.default_rng(seed)
    clouds = []
    for i in range(n_views):
        c2w = lookat_c2w(1.0 + 0.5 * rng.random(), 20 + 80 * rng.random(), 360.0 * i / n_views)
        D, m = sphere_depth(c2w, intrinsics(S), S, R)
        clouds.append(depth_cloud(D, m, c2w, intrinsics(S)))
    return np.concatenate(clouds).astype(np.float32)
