"""CPU restatement of the refine stage's point-cloud construction: the reference's load_views (nerf/refine_utils.py:335-410) with its
helpers depth2point (:129-152) and multidepth2point_mask (:61-127).  Test infrastructure only.

OpenCV's erode, dilate and Canny are written out in numpy; the back-projection and projections use the reference's own numpy
expressions (so the fp64 products go through the same BLAS calls); grid_sample is torch's CPU kernel, as in the reference; the
point renderer and z_buffer are oracle/points_ref.py's.  The functions take decoded images (uint16 depth x 1000, uint8 masks, uint8 RGB)
instead of file names.  `make_mvimg` builds the synthetic multi-view folders the golden generator, the tests and
tests/measure_load_views.py share.
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import points_ref as pr


# ---- OpenCV's morphology and Canny ----

def _window(img, k, neutral, reduce):
    r = k // 2
    p = np.pad(img, r, mode="constant", constant_values=neutral)
    rows = reduce(np.lib.stride_tricks.sliding_window_view(p, k, axis=1), axis=-1)
    return reduce(np.lib.stride_tricks.sliding_window_view(rows, k, axis=0), axis=-1)


def erode(img, k):
    """cv2.erode(img, np.ones((k, k))) with the default +inf border: minimum over the k x k window clipped to the image"""
    return _window(img, k, np.inf if img.dtype.kind == "f" else np.iinfo(img.dtype).max, np.min)


def dilate(img, k):
    """cv2.dilate(img, np.ones((k, k))) with the default -inf border: maximum over the k x k window clipped to the image"""
    return _window(img, k, -np.inf if img.dtype.kind == "f" else np.iinfo(img.dtype).min, np.max)


def canny(img, thresh):
    """cv2.Canny(img, thresh, thresh) (aperture 3, L1 magnitude): with equal thresholds there are no weak pixels, so the edges are the
    non-maximum-suppression survivors with magnitude > thresh.  3x3 Sobel with a replicated border, magnitude 0 outside the image,
    OpenCV's fixed-point tan(22.5 deg) = 13573 / 2^15 sector test and its > / >= neighbour comparisons.  uint8 0 / 255."""
    H, W = img.shape
    p = np.pad(img.astype(np.int64), 1, mode="edge")
    dx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    m = np.abs(dx) + np.abs(dy)
    mp = np.pad(m, 1)

    def at(oy, ox):
        return mp[1 + oy:1 + oy + H, 1 + ox:1 + ox + W]

    ax, ay = np.abs(dx), np.abs(dy) << 15
    tg22x = ax * 13573
    horiz = ay < tg22x
    vert = ~horiz & (ay > tg22x + (ax << 16))
    neg = (dx ^ dy) < 0
    e_h = (m > at(0, -1)) & (m >= at(0, 1))
    e_v = (m > at(-1, 0)) & (m >= at(1, 0))
    e_d = np.where(neg, (m > at(-1, 1)) & (m > at(1, -1)), (m > at(-1, -1)) & (m > at(1, 1)))
    edge = (m > thresh) & np.where(horiz, e_h, np.where(vert, e_v, e_d))
    return np.where(edge, 255, 0).astype(np.uint8)


# ---- the masks of load_views ----

def depth_blur(depth, mask):
    """np.uint8(depth * mask * 255.0) (refine_utils.py:386-387): truncation, then wrap modulo 256 as numpy's cast does on x86-64"""
    return (np.trunc(depth * mask * 255.0).astype(np.int64) & 255).astype(np.uint8)


def view_mask(depth_u16, mask_u8):
    """a non-canonical view's mask (refine_utils.py:376-395): (mask, eroded == 1, Canny, dilated Canny)"""
    depth = depth_u16 / 1000.0
    eroded = erode(mask_u8 / 255.0, 11) == 1
    edges = canny(depth_blur(depth, eroded), 10)
    dil = dilate(edges, 11)
    return eroded & ~(dil == 255), eroded, edges, dil


def cano_mask(mask_u8):
    """the canonical view's mask (refine_utils.py:345-350): two 11 x 11 erosions == one 21 x 21, then == 1"""
    return erode(mask_u8 / 255.0, 21) == 1


def cover_quant(render):
    """uint8(render * 255) of the canonical cloud's [1,3,H,W] render as the reference writes it to PNG (refine_utils.py:79)"""
    return np.array(render[0].permute(1, 2, 0).detach().cpu().numpy() * 255, dtype=np.uint8)


def cover_mask(quant):
    """refine_utils.py:80-84 on the PNG round trip: erode each channel 15 x 15, OR over channels of > 0.9"""
    m = quant / 255.0
    e = np.stack([erode(m[..., c], 15) for c in range(m.shape[-1])], -1)
    return (e > 0.9).any(-1)


# ---- geometry, in the reference's numpy expressions ----

def backproject(D, mask, c2w, K):
    """world points of the mask's pixels (refine_utils.py:131-139), row-major pixel order"""
    x, y = np.meshgrid(np.arange(D.shape[1]), np.arange(D.shape[0]))
    cam_xyz = np.vstack((x.reshape(-1), y.reshape(-1), np.ones(len(D.reshape(-1)))))
    v = np.linalg.inv(K).dot(cam_xyz).T
    v = v * np.tile(D.reshape((-1, 1)), (1, 3))
    v = v[mask.reshape(-1) == 1]
    return np.matmul(v, c2w[:3, :3].T) + c2w[:3, 3:].T


def project(xyz, K, RT):
    xyz = np.dot(xyz, RT[:, :3].T) + RT[:, 3:].T
    xyz = np.dot(xyz, K.T)
    return xyz[:, :2] / xyz[:, 2:], xyz[:, 2:]


def sample(img_chw, xy, H):
    """F.grid_sample(img [1,C,H,W] float32, float32(xy) / H * 2 - 1) -> [N, C] float32 (bilinear, zeros, align_corners=False)"""
    g = torch.Tensor(np.asarray(xy)[None, None, ...]) / H * 2. - 1.
    return F.grid_sample(img_chw, g, align_corners=False)[0, :, 0].permute(1, 0).numpy()


def colourise(v, w2c, K, img_hwc, H, W):
    """z_buffer in the view, then the colours of the survivors (refine_utils.py:143-151 / :109-114)"""
    keep = pr.z_buffer_ref(v, w2c, H, W, K)
    v = v[keep, :]
    xy, _ = project(v, K, w2c[:3, :4])
    return v, sample(torch.Tensor(img_hwc[None, ...]).permute(0, 3, 1, 2), xy, H)


def occlusion_keep(v, K, cano_w2c, cano_D, H):
    """refine_utils.py:100-107: False for the points whose canonical depth sample d has -0.2 <= z - d <= 1/H"""
    xy1, xyz = project(v, K, cano_w2c[:3, :4])
    xy1 = np.round(xy1).astype(np.int32)
    d = sample(torch.Tensor(cano_D)[None, None], xy1, H)
    xy_mask = np.logical_and((xyz - d) <= (1 / H), (xyz - d) >= -0.2)
    return ~xy_mask[:, 0]


def load_views_ref(gt_rgb, depths_u16, masks_u8, rgbs_u8, cam2world_list, H, W, K, radius, ppp, npoint=1000000, record=None):
    """load_views on decoded images -> (vertices_cano, vertices_color_cano, vertices_novel, vertices_color_novel); `record` (a dict)
    receives the per-view intermediates"""
    rec = record if record is not None else {}
    n = len(cam2world_list)
    ind = (n - 1) // 2
    c2w_cano = cam2world_list[ind]
    depth_cano = depths_u16[ind] / 1000.0
    m_cano = cano_mask(masks_u8[ind])
    rec["cano_mask"] = m_cano
    # refine_utils.py:352-360 also computes a Canny edge mask of the canonical view, but never applies it (line 360 is commented out)
    w2c_cano = np.linalg.inv(c2w_cano)
    v = backproject(depth_cano, m_cano, c2w_cano, K)
    v_cano, c_cano = colourise(v, w2c_cano, K, np.asarray(gt_rgb), H, W)

    cano_v = torch.tensor(v_cano).float()
    cano_D = (depth_cano * m_cano).astype(np.float32)
    K32 = torch.tensor(K).float()
    r_ndc = float(radius) / float(H) * 2.0
    vs, cs = [], []
    for i in range(n):
        if i == ind:
            continue
        mask, eroded, edges, dil = view_mask(depths_u16[i], masks_u8[i])
        c2w = cam2world_list[i]
        w2c = np.linalg.inv(c2w)
        img = pr.render_point_ref(cano_v, torch.ones_like(cano_v), H, W, K32, torch.tensor(w2c), [H, W], r_ndc, ppp)[0]
        q = cover_quant(img)
        mask = np.logical_and(mask, ~cover_mask(q))
        rec.setdefault("eroded", []).append(eroded)
        rec.setdefault("canny", []).append(edges)
        rec.setdefault("dilated", []).append(dil)
        rec.setdefault("quant", []).append(q[..., 0])
        rec.setdefault("mask", []).append(mask)
        v = backproject(depths_u16[i] / 1000.0, mask, c2w, K)
        v = v[occlusion_keep(v, K, w2c_cano, cano_D, H)]
        v, c = colourise(v, w2c, K, rgbs_u8[i][..., :3] / 255., H, W)
        vs.append(v)
        cs.append(c)
    v_n, c_n = np.concatenate(vs), np.concatenate(cs)
    if len(v_n) >= npoint:
        arr = np.arange(len(v_n))
        np.random.shuffle(arr)
        arr = arr[:npoint]
        v_n, c_n = v_n[arr], c_n[arr]
    return v_cano, c_cano, v_n, c_n


# ---- synthetic multi-view folders, written the way Trainer.test writes them ----

# an object with a concavity: a large sphere and a smaller one that overlaps it (the crease between them is concave, and the small
# sphere hides part of the large one from some views)
SPHERES = ((np.array([0.0, 0.0, 0.0]), 0.42), (np.array([0.22, 0.12, 0.3]), 0.2), (np.array([-0.25, -0.2, 0.1]), 0.16))


def render_view(c2w, K, S):
    """camera-z depth [S,S] (0 where the rays miss), hit mask and an RGB uint8 image of the object"""
    ys, xs = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    d = (np.linalg.inv(K) @ np.stack([xs.ravel(), ys.ravel(), np.ones(S * S)], 0)).T
    dw = d @ c2w[:3, :3].T
    o = c2w[:3, 3]
    t = np.full(S * S, np.inf)
    for c, R in SPHERES:
        oc = o - c
        a, b, cc = (dw * dw).sum(1), 2 * dw @ oc, oc @ oc - R * R
        disc = b * b - 4 * a * cc
        th = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        t = np.minimum(t, np.where(th > 0, th, np.inf))
    hit = np.isfinite(t)
    p = o + dw * np.where(hit, t, 0)[:, None]
    rgb = (0.5 + 0.5 * np.sin(np.stack([7 * p[:, 0] + 1, 9 * p[:, 1] + 2, 11 * p[:, 2] + 3], -1))) * hit[:, None]
    return np.where(hit, t, 0).reshape(S, S), hit.reshape(S, S), np.round(rgb * 255).astype(np.uint8).reshape(S, S, 3)


def make_mvimg(folder, n_views, S, seed, fov=40.0):
    """write n_views views (uint16 depth x 1000, 0/255 mask, RGB png) and float32 poses into `folder`; returns
    (gt_rgb float64 [S,S,3], rgb_files, depth_files, mask_files, cam2world_list float32, K float64)"""
    import cv2
    os.makedirs(folder, exist_ok=True)
    rng = np.random.default_rng(seed)
    K = pr.intrinsics(S, fov)
    poses = []
    for i in range(n_views):
        c2w = pr.lookat_c2w(1.1 + 0.3 * rng.random(), 55 + 50 * rng.random(), 360.0 * i / n_views + 10 * rng.random())
        poses.append(c2w.astype(np.float32))
        depth, hit, rgb = render_view(poses[-1].astype(np.float64), K, S)
        cv2.imwrite(os.path.join(folder, f"{i:04d}_depth.png"), np.round(depth * 1000).astype(np.uint16))
        cv2.imwrite(os.path.join(folder, f"{i:04d}_mask.png"), (hit * 255).astype(np.uint8))
        cv2.imwrite(os.path.join(folder, f"{i:04d}_rgb.png"), rgb[..., ::-1])
    poses = np.stack(poses)
    np.save(os.path.join(folder, "0000_poses.npy"), poses)
    files = [sorted(os.path.join(folder, f) for f in os.listdir(folder) if f.endswith(s)) for s in ("rgb.png", "depth.png", "mask.png")]
    gt = render_view(poses[(n_views - 1) // 2].astype(np.float64), K, S)[2]
    return (gt / 255.0,) + tuple(files) + (np.load(os.path.join(folder, "0000_poses.npy")), K)
