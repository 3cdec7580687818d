"""B5 seam: the refine stage's point renderer and z-buffer (reference nerf/refine_utils.py:167-208, :306-333) on libmi3d.so.

* `render_point(points_xyz_org, points_color, H, W, K, world2cam, image_size, radius, ppp, bg_feat=None, acc='alphacomposite')`:
  drop-in for the reference function, which projects the cloud and runs pytorch3d's `rasterize_points` + `alpha_composite`.
  Returns `[1, C, h, w]` with a gradient for `points_color` only (the reference never asks for one on the points; `bg_feat` is
  accepted and ignored, as there).  Projection, rasterisation and compositing are fused in csrc/points.cu; the host never
  synchronises.
* `rasterize_points(points_xyz_org, H, W, K, world2cam, image_size, radius, ppp)`: pytorch3d's `(idx [1,h,w,K] int32, zbuf, dists)`
  for the same projected cloud, for hosts that composite themselves.
* `z_buffer(vertices, world2cam_pose_cano, H, W, K)`: numpy in, numpy bool mask out, as the reference; runs in fp64 on the GPU.

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
    lib.mi3d_points_workspace_bytes.restype = C.c_size_t
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
