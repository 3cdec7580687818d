"""B5 seam: the refine stage's point renderer and z-buffer (reference nerf/refine_utils.py:167-208, :306-333) on libmi3d.so.

* `render_point(points_xyz_org, points_color, H, W, K, world2cam, image_size, radius, ppp, bg_feat=None, acc='alphacomposite')`:
  drop-in for the reference function, which projects the cloud and runs pytorch3d's `rasterize_points` + `alpha_composite`.
  Returns `[1, C, h, w]` with a gradient for `points_color` only (the reference never asks for one on the points; `bg_feat` is
  accepted and ignored, as there).  Projection, rasterisation and compositing are fused in csrc/points.cu; the host never
  synchronises.
* `render_point_weights(...)`: `render_point` with the same arguments that also returns the composite weights `[h, w, ppp]` it
  saved for its backward (the refine loop derives its coverage mask from them instead of rasterising the cloud again).
* `rasterize_points(points_xyz_org, H, W, K, world2cam, image_size, radius, ppp)`: pytorch3d's `(idx [1,h,w,K] int32, zbuf, dists)`
  for the same projected cloud, for hosts that composite themselves.
* `z_buffer(vertices, world2cam_pose_cano, H, W, K)`: numpy in, numpy bool mask out, as the reference; runs in fp64 on the GPU.
* `load_views(gt_rgb, rgb_files, depth_files, mask_files, cam2world_list, H, W, K, radius, ppp, outputdir, device, npoint=1_000_000)`:
  drop-in for the reference function (refine_utils.py:335-410): the two coloured point clouds of the refine stage, built on
  csrc/views.cu and the two entry points above, point for point the reference's.

`H`, `W` normalise the projected pixel coordinates to NDC; `image_size` is the raster.  Only square rasters are supported.
"""
import ctypes as C

import numpy as np
import torch

from .. import _lib as L


def _cam32(K, world2cam):
    L.require_cuda(K, world2cam)
    k = K.reshape(3, 3).to(torch.float32).contiguous()
    rt = world2cam[:3, :4].to(torch.float32).contiguous()
    return k, rt


def _check(points, feats, image_size, acc="alphacomposite"):
    L.require_cuda(points, feats)
    if acc != "alphacomposite":
        raise L.Mi3dError(f"render_point: only acc='alphacomposite' is supported (got {acc!r})")
    h, w = int(image_size[0]), int(image_size[1])
    if h != w:
        raise L.Mi3dError(f"render_point: only square images are supported (got {h}x{w})")
    if points.requires_grad:
        raise L.Mi3dError("render_point: no gradient with respect to the point positions (pass them detached)")
    if points.dim() != 2 or points.shape[1] != 3:
        raise L.Mi3dError(f"render_point: points must be [P,3] (got {tuple(points.shape)})")
    return h


def _forward(points, feats, k, rt, H, W, S, radius, ppp, want_image, want_extra):
    lib = L.lib()
    P = points.shape[0]
    Cn = feats.shape[1] if feats is not None else 1
    nbytes = lib.mi3d_points_workspace_bytes(C.c_uint32(P), C.c_uint32(S), C.c_uint32(S), C.c_double(radius))
    if nbytes == 0:
        raise L.Mi3dError(f"render_point: invalid arguments (P={P}, image {S}x{S}, radius={radius})")
    dev = points.device
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    idx = torch.empty(S, S, ppp, dtype=torch.int32, device=dev)
    wts = torch.empty(S, S, ppp, dtype=torch.float32, device=dev) if want_image else None
    image = torch.empty(1, Cn, S, S, dtype=torch.float32, device=dev) if want_image else None
    zbuf = torch.empty(S, S, ppp, dtype=torch.float32, device=dev) if want_extra else None
    dist2 = torch.empty(S, S, ppp, dtype=torch.float32, device=dev) if want_extra else None
    L.check(lib.mi3d_points_render_forward(L.ptr(points), L.ptr(feats), C.c_uint32(P), C.c_uint32(Cn), L.ptr(k), L.ptr(rt),
                                           C.c_float(W), C.c_float(H), C.c_uint32(S), C.c_uint32(S), C.c_double(radius), C.c_uint32(ppp),
                                           L.ptr(image), L.ptr(idx), L.ptr(wts), L.ptr(zbuf), L.ptr(dist2), L.ptr(ws), C.c_size_t(nbytes),
                                           L.stream()), "points_render_forward")
    return image, idx, wts, zbuf, dist2


class _RenderPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, feats, k, rt, H, W, S, radius, ppp):
        image, idx, wts, _, _ = _forward(points, feats, k, rt, H, W, S, radius, ppp, True, False)
        ctx.save_for_backward(points, k, rt, idx, wts)
        ctx.args = (H, W, S, radius, ppp, feats.shape[1])
        return image

    @staticmethod
    def backward(ctx, grad_image):
        points, k, rt, idx, wts = ctx.saved_tensors
        H, W, S, radius, ppp, Cn = ctx.args
        g = L.f32c(grad_image)
        grad_feats = torch.empty(points.shape[0], Cn, dtype=torch.float32, device=points.device)
        L.check(L.lib().mi3d_points_render_backward(L.ptr(points), C.c_uint32(points.shape[0]), C.c_uint32(Cn), L.ptr(k), L.ptr(rt),
                                                    C.c_float(W), C.c_float(H), C.c_uint32(S), C.c_uint32(S), C.c_double(radius),
                                                    C.c_uint32(ppp), L.ptr(idx), L.ptr(wts), L.ptr(g), L.ptr(grad_feats), L.stream()),
                "points_render_backward")
        return None, grad_feats, None, None, None, None, None, None, None


def render_point(points_xyz_org, points_color, H, W, K, world2cam, image_size, radius, ppp, bg_feat=None, acc='alphacomposite'):
    """[1, C, h, w] alpha-composited splats of the cloud (reference refine_utils.py:306-333); bg_feat is ignored, as there."""
    S = _check(points_xyz_org, points_color, image_size, acc)
    k, rt = _cam32(K, world2cam)
    pts = L.f32c(points_xyz_org)
    feats = points_color if points_color.dtype == torch.float32 else points_color.float()
    return _RenderPoint.apply(pts, feats.contiguous(), k, rt, float(H), float(W), S, float(radius), int(ppp))


class _RenderPointWeights(_RenderPoint):
    """_RenderPoint that also returns its composite weights (no gradient through them)"""

    @staticmethod
    def forward(ctx, points, feats, k, rt, H, W, S, radius, ppp):
        image, idx, wts, _, _ = _forward(points, feats, k, rt, H, W, S, radius, ppp, True, False)
        ctx.save_for_backward(points, k, rt, idx, wts)
        ctx.args = (H, W, S, radius, ppp, feats.shape[1])
        ctx.mark_non_differentiable(wts)
        return image, wts

    @staticmethod
    def backward(ctx, grad_image, grad_wts):
        return _RenderPoint.backward(ctx, grad_image)


def render_point_weights(points_xyz_org, points_color, H, W, K, world2cam, image_size, radius, ppp):
    """(render_point(...) with the same arguments, its composite weights fp32 [h, w, ppp]); summing a pixel's weights in slot order
    gives, bit for bit, the image render_point makes with unit colours"""
    S = _check(points_xyz_org, points_color, image_size)
    k, rt = _cam32(K, world2cam)
    feats = points_color if points_color.dtype == torch.float32 else points_color.float()
    return _RenderPointWeights.apply(L.f32c(points_xyz_org), feats.contiguous(), k, rt, float(H), float(W), S, float(radius), int(ppp))


def rasterize_points(points_xyz_org, H, W, K, world2cam, image_size, radius, ppp):
    """pytorch3d's (idx [1,h,w,ppp] int32, zbuf, dists) for the cloud render_point projects with the same arguments."""
    S = _check(points_xyz_org, None, image_size)
    k, rt = _cam32(K, world2cam)
    _, idx, _, zbuf, dist2 = _forward(L.f32c(points_xyz_org), None, k, rt, float(H), float(W), S, float(radius), int(ppp), False, True)
    return idx[None], zbuf[None], dist2[None]


def z_buffer(vertices, world2cam_pose_cano, H, W, K, device="cuda"):
    """bool mask [P] of the points that survive the reference's z-buffer test (refine_utils.py:167-208)."""
    v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)).to(device)
    k = torch.from_numpy(np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(3, 3))).to(device)
    rt = torch.from_numpy(np.ascontiguousarray(np.asarray(world2cam_pose_cano, dtype=np.float64)[:3, :4])).to(device)
    P = v.shape[0]
    mask = torch.empty(P, dtype=torch.uint8, device=device)
    zbuf = torch.empty(int(H) * int(W), dtype=torch.int64, device=device)
    L.check(L.lib().mi3d_points_zbuffer_visible(L.ptr(v), C.c_uint32(P), L.ptr(k), L.ptr(rt), C.c_uint32(int(H)), C.c_uint32(int(W)),
                                                L.ptr(zbuf), L.ptr(mask), L.stream()), "points_zbuffer_visible")
    return mask.cpu().numpy().astype(bool)


# ---- load_views: the two coloured point clouds of the refine stage (reference refine_utils.py:61-152, :335-410) ----

def _read(path, flags):
    import cv2
    im = cv2.imread(path, flags)
    if im is None:
        raise L.Mi3dError(f"load_views: cannot read {path}")
    return im


def _read_first_channel(path):
    """load_depth: cv2.IMREAD_UNCHANGED, then the first channel"""
    import cv2
    im = _read(path, cv2.IMREAD_UNCHANGED)
    return im[:, :, 0] if im.ndim > 2 else im


def _read_rgb(path):
    """imageio.imread(path)[:, :, :3] as uint8 RGB"""
    import cv2
    im = _read(path, cv2.IMREAD_UNCHANGED)
    if im.ndim != 3 or im.shape[2] < 3 or im.dtype != np.uint8:
        raise L.Mi3dError(f"load_views: {path} is not an 8-bit RGB(A) image")
    return np.ascontiguousarray(im[:, :, 2::-1])


class _Views:
    """device buffers and C-ABI calls of one load_views run at S x S"""

    def __init__(self, S, K, device):
        self.S, self.dev = S, device
        lib = L.lib()
        nbytes = lib.mi3d_views_workspace_bytes(C.c_uint32(S), C.c_uint32(S))
        if nbytes == 0:
            raise L.Mi3dError(f"load_views: unsupported view size {S}x{S}")
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.nbytes = C.c_size_t(nbytes)
        K = np.asarray(K, dtype=np.float64).reshape(3, 3)
        self.k = self._f64(K)
        self.kinv = self._f64(np.linalg.inv(K))
        self.zbuf = torch.empty(S * S, dtype=torch.int64, device=device)

    def _f64(self, a):
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float64))).reshape(-1).to(self.dev)

    def rows(self, pose):
        """rows 0..2 of a 4x4 pose (R | t), its own dtype's values held exactly in fp64"""
        return self._f64(np.asarray(pose)[:3, :4])

    def mask(self, depth, mask, erode_k, canny, eroded=None, edges=None, dilated=None, masked_depth=None):
        S = self.S
        out = torch.empty(S, S, dtype=torch.uint8, device=self.dev)
        L.check(L.lib().mi3d_views_mask(L.ptr(depth), L.ptr(mask), C.c_uint32(S), C.c_uint32(S), C.c_uint32(erode_k), C.c_int(canny),
                                        C.c_uint32(11), L.ptr(out), L.ptr(masked_depth), L.ptr(eroded), L.ptr(edges), L.ptr(dilated),
                                        L.ptr(self.ws), self.nbytes, L.stream()), "views_mask")
        return out

    def cover(self, render, alphamask, quant=None):
        S = self.S
        out = torch.empty(S, S, dtype=torch.uint8, device=self.dev)
        L.check(L.lib().mi3d_views_cover_mask(L.ptr(render), L.ptr(alphamask), C.c_uint32(S), C.c_uint32(S), C.c_uint32(15), L.ptr(out),
                                              L.ptr(quant), L.ptr(self.ws), self.nbytes, L.stream()), "views_cover_mask")
        return out

    def backproject(self, depth, mask, c2w, cano_w2c=None, cano_depth=None):
        S = self.S
        pts = torch.empty(S * S, 3, dtype=torch.float64, device=self.dev)
        count = torch.empty(1, dtype=torch.int32, device=self.dev)
        L.check(L.lib().mi3d_views_backproject(L.ptr(depth), L.ptr(mask), C.c_uint32(S), C.c_uint32(S), L.ptr(self.kinv), L.ptr(c2w),
                                               L.ptr(self.k), L.ptr(cano_w2c), L.ptr(cano_depth), L.ptr(pts), L.ptr(count), L.ptr(self.ws),
                                               self.nbytes, L.stream()), "views_backproject")
        return pts, count

    def visible(self, pts, w2c):
        """z_buffer of the (NaN-padded) back-projection in the view w2c"""
        S, P = self.S, pts.shape[0]
        keep = torch.empty(P, dtype=torch.uint8, device=self.dev)
        L.check(L.lib().mi3d_points_zbuffer_visible(L.ptr(pts), C.c_uint32(P), L.ptr(self.k), L.ptr(w2c), C.c_uint32(S), C.c_uint32(S),
                                                    L.ptr(self.zbuf), L.ptr(keep), L.stream()), "points_zbuffer_visible")
        return keep

    def compact_colour(self, pts, keep, w2c, img_f32=None, img_u8=None):
        S, P = self.S, pts.shape[0]
        out = torch.empty(P, 3, dtype=torch.float64, device=self.dev)
        col = torch.empty(P, 3, dtype=torch.float32, device=self.dev)
        count = torch.empty(1, dtype=torch.int32, device=self.dev)
        L.check(L.lib().mi3d_views_compact_colour(L.ptr(pts), C.c_uint32(P), L.ptr(keep), L.ptr(self.k), L.ptr(w2c), L.ptr(img_f32),
                                                  L.ptr(img_u8), C.c_uint32(S), C.c_uint32(S), L.ptr(out), L.ptr(col), L.ptr(count),
                                                  L.ptr(self.ws), self.nbytes, L.stream()), "views_compact_colour")
        return out, col, count


def load_views(gt_rgb, rgb_files, depth_files, mask_files, cam2world_list, H, W, K, radius, ppp, outputdir, device, npoint=1_000_000):
    """the refine stage's two coloured point clouds (reference refine_utils.py:335-410) ->
    (vertices_cano fp64 [P,3], vertices_color_cano fp32 [P,3], vertices_novel fp64 [Q,3], vertices_color_novel fp32 [Q,3]).

    Files are only decoded on the host; every mask, the back-projection, the visibility tests and the colour lookups run in
    csrc/views.cu and csrc/points.cu.  Nothing is written to `outputdir` (the reference's mask PNG round trip is lossless, so the
    uint8 quantisation happens in memory).  When the novel points reach `npoint`, they are subsampled with the reference's
    `np.random.shuffle(np.arange(n))`, which consumes numpy's global RNG as the reference does.  Square views (H == W) at H x W,
    at least 2 views and a CUDA device only."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise L.Mi3dError(f"load_views: runs on CUDA only (got device {device!r})")
    H, W = int(H), int(W)
    if H != W:
        raise L.Mi3dError(f"load_views: only square views are supported (got {H}x{W})")
    n = len(cam2world_list)
    if n < 2 or len(depth_files) != n or len(mask_files) != n or len(rgb_files) != n:
        raise L.Mi3dError(f"load_views: need at least 2 views with a depth, mask and RGB file each (got {n} poses, {len(depth_files)} "
                          f"depth, {len(mask_files)} mask and {len(rgb_files)} RGB files)")
    gt = np.asarray(gt_rgb)
    if gt.shape != (H, W, 3):
        raise L.Mi3dError(f"load_views: gt_rgb must be [{H},{W},3] (got {gt.shape})")
    S = H
    V = _Views(S, K, dev)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    def read_view(i):
        d, m = _read_first_channel(depth_files[i]), _read_first_channel(mask_files[i])
        if d.shape != (S, S) or m.shape != (S, S) or d.dtype != np.uint16 or m.dtype != np.uint8:
            raise L.Mi3dError(f"load_views: view {i} must be a uint16 depth and a uint8 mask at {S}x{S} "
                              f"(got {d.dtype} {d.shape}, {m.dtype} {m.shape})")
        return up(d), up(m)

    ind = (n - 1) // 2
    c2w_cano = np.asarray(cam2world_list[ind])
    w2c_cano = np.linalg.inv(c2w_cano)
    # canonical view: 11 x 11 erosion twice (= 21 x 21).  The reference also computes a Canny edge mask here (refine_utils.py:352-359)
    # but never applies it, because line 360 is commented out; it is not computed.
    d_cano, m_cano = read_view(ind)
    cano_depth = torch.empty(S, S, dtype=torch.float32, device=dev)
    mask_cano = V.mask(d_cano, m_cano, 21, -1, masked_depth=cano_depth)
    pts, _ = V.backproject(d_cano, mask_cano, V.rows(c2w_cano))
    w2c_cano_d = V.rows(w2c_cano)
    v_cano, c_cano, n_cano = V.compact_colour(pts, V.visible(pts, w2c_cano_d), w2c_cano_d,
                                              img_f32=up(gt.astype(np.float64).astype(np.float32)))
    P = int(n_cano.item())                                                   # the one count read of the canonical view
    v_cano, c_cano = v_cano[:P], c_cano[:P]

    # the canonical cloud rendered into each other view with unit colours: every channel of the reference's 3-channel render is the
    # same sum, so one channel is rendered
    cano_v32 = v_cano.float().contiguous()
    ones = torch.ones(P, 1, dtype=torch.float32, device=dev)
    K32 = torch.from_numpy(np.asarray(K, dtype=np.float64)).float().to(dev)
    r_ndc = float(radius) / float(S) * 2.0
    outs = []
    for i in range(n):
        if i == ind:
            continue
        d, m = read_view(i)
        rgb = _read_rgb(rgb_files[i])
        if rgb.shape != (S, S, 3):
            raise L.Mi3dError(f"load_views: view {i}'s RGB image must be {S}x{S} (got {rgb.shape[:2]})")
        alphamask = V.mask(d, m, 11, 10)
        c2w = np.asarray(cam2world_list[i])
        w2c = np.linalg.inv(c2w)
        render = render_point(cano_v32, ones, S, S, K32, torch.from_numpy(np.asarray(w2c)).to(dev), [S, S], r_ndc, ppp)
        mask = V.cover(render.detach().contiguous(), alphamask)
        pts, _ = V.backproject(d, mask, V.rows(c2w), w2c_cano_d, cano_depth)
        w2c_d = V.rows(w2c)
        outs.append(V.compact_colour(pts, V.visible(pts, w2c_d), w2c_d, img_u8=up(rgb)))
    counts = torch.cat([o[2] for o in outs]).cpu().tolist()
    v_n = torch.cat([o[0][:c] for o, c in zip(outs, counts)])
    c_n = torch.cat([o[1][:c] for o, c in zip(outs, counts)])
    if v_n.shape[0] >= npoint:
        arr = np.arange(v_n.shape[0])
        np.random.shuffle(arr)
        sel = torch.from_numpy(arr[:npoint]).to(dev)
        v_n, c_n = v_n[sel], c_n[sel]
    return v_cano.cpu().numpy(), c_cano.cpu().numpy(), v_n.cpu().numpy(), c_n.cpu().numpy()
