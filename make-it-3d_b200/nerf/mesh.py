"""B10 seam: mesh export (NeRFRenderer.export_mesh, nerf/renderer.py:157-330) without PyMCubes, xatlas, nvdiffrast, sklearn or scipy.

* ``marching_cubes(volume, isovalue)``  PyMCubes' call contract (``from mi3d_b200.nerf import mesh as mcubes``), on the GPU
* ``extract_mesh(model, resolution, S)`` the density volume of renderer.py:167-180 (one fused field call per S^3 chunk, no
                                         tape) -> marching cubes with the export's [-1, 1] scaling -> (v, f) CUDA tensors
* ``bake_texture(model, v, f)``        closed-form per-face atlas: texels -> surface points -> field albedo
* ``export_mesh(model, path, ...)``    mesh.obj / mesh.mtl / albedo.png as the reference writes them

The surface is the one PyMCubes extracts (same algorithm and triangle table; csrc/mesh.cu).  The atlas is not xatlas's: faces 2p and
2p+1 share one square cell of c x c texels, and every texel whose centre lies within Chebyshev distance 1 of a face's UV triangle is
baked from that face's (extrapolated) surface point, so bilinear lookups inside a triangle only read its own texels.  That gutter
replaces the reference's kd-tree inpainting ring.  One host synchronisation reads the vertex / face counts; the file write is the other.
"""
import ctypes as C
import math
import os

import numpy as np
import torch

from .. import _lib as L
from . import field_ops

ATLAS_T0, ATLAS_T_MAX, ATLAS_MIN_CELL = 2048, 16384, 8     # 2048 = the reference's h0 = w0 (renderer.py:193)

MTL_TEXT = ("newmtl mat0 \n"
            "Ka 1.000000 1.000000 1.000000 \n"
            "Kd 1.000000 1.000000 1.000000 \n"
            "Ks 0.000000 0.000000 0.000000 \n"
            "Tr 1.000000 \n"
            "illum 1 \n"
            "Ns 0.000000 \n"
            "map_Kd albedo.png \n")


# ----------------------------------------------------------------------------------------------------------------------------
# marching cubes
# ----------------------------------------------------------------------------------------------------------------------------
def _check_volume(volume):
    if not torch.is_tensor(volume) or not volume.is_cuda:
        raise L.Mi3dError("marching cubes runs on the GPU: pass a CUDA tensor (or a numpy array to marching_cubes)")
    if volume.dtype != torch.float32 or not volume.is_contiguous() or volume.dim() != 3:
        raise L.Mi3dError(f"volume must be a contiguous fp32 [nx, ny, nz] tensor; got {volume.dtype} {tuple(volume.shape)}")
    nx, ny, nz = volume.shape
    if L.lib().mi3d_mc_workspace_bytes(C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(nz)) == 0:
        raise L.Mi3dError(f"volume {tuple(volume.shape)}: every dimension must be >= 2 and the vertex / face counts must fit int32")
    return nx, ny, nz


def _iso_args(isovalue, iso_dev):
    if iso_dev is not None:
        if not (torch.is_tensor(iso_dev) and iso_dev.is_cuda and iso_dev.dtype == torch.float32 and iso_dev.numel() >= 1):
            raise L.Mi3dError("iso_dev must be a CUDA fp32 scalar tensor")
        iso_dev = iso_dev.reshape(-1)[:1].contiguous()
    return C.c_float(float(isovalue)), iso_dev


def mc_count(volume, isovalue, iso_dev=None):
    """Count pass: -> (workspace, counts) with counts a CUDA int32 [2] = (V, F).  The threshold is isovalue, or
    min(isovalue, iso_dev) when iso_dev (CUDA fp32 scalar) is given, read on the device."""
    nx, ny, nz = _check_volume(volume)
    iso, iso_dev = _iso_args(isovalue, iso_dev)
    lib = L.lib()
    ws = torch.empty(lib.mi3d_mc_workspace_bytes(C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(nz)), dtype=torch.uint8, device=volume.device)
    counts = torch.empty(2, dtype=torch.int32, device=volume.device)
    L.check(lib.mi3d_mc_count(L.ptr(volume), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(nz), iso, L.ptr(iso_dev), L.ptr(ws), L.ptr(counts),
                              L.stream()), "mc_count")
    return ws, counts


def mc_emit(volume, isovalue, ws, V, F, iso_dev=None, scale=1.0, offset=0.0):
    """Emit pass on the workspace of mc_count (same volume and threshold): -> vertices fp32 [V,3] (* scale + offset), faces int32 [F,3]"""
    nx, ny, nz = _check_volume(volume)
    iso, iso_dev = _iso_args(isovalue, iso_dev)
    v = torch.empty(V, 3, dtype=torch.float32, device=volume.device)
    f = torch.empty(F, 3, dtype=torch.int32, device=volume.device)
    if V > 0 or F > 0:
        L.check(L.lib().mi3d_mc_emit(L.ptr(volume), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(nz), iso, L.ptr(iso_dev), L.ptr(ws),
                                     C.c_float(scale), C.c_float(offset), C.c_void_p(v.data_ptr()), C.c_void_p(f.data_ptr()), L.stream()),
                "mc_emit")
    return v, f


def _marching_cubes_cuda(volume, isovalue, iso_dev=None, scale=1.0, offset=0.0):
    ws, counts = mc_count(volume, isovalue, iso_dev)
    V, F = (int(x) for x in counts.cpu().tolist())            # the one host synchronisation: sizes the outputs
    return mc_emit(volume, isovalue, ws, V, F, iso_dev, scale, offset)


def marching_cubes(volume, isovalue):
    """PyMCubes' marching_cubes(volume, isovalue) on the GPU (current CUDA device; there is no CPU path).
    numpy volume -> (vertices float64 [V,3] in index coordinates, triangles int64 [F,3]) as numpy;
    CUDA fp32 tensor -> (vertices float32, triangles int32) CUDA tensors.  Vertices lie where the volume crosses isovalue (rounded
    to fp32); triangles wind with their right-hand normal pointing toward values <= isovalue."""
    if isinstance(volume, np.ndarray):
        vol = torch.from_numpy(np.ascontiguousarray(volume, dtype=np.float32)).cuda()
        v, f = _marching_cubes_cuda(vol, isovalue)
        return v.cpu().numpy().astype(np.float64), f.cpu().numpy().astype(np.int64)
    if torch.is_tensor(volume) and not volume.is_cuda:
        raise L.Mi3dError("marching_cubes: CPU tensors are not accepted (pass a numpy array or a CUDA tensor)")
    return _marching_cubes_cuda(volume, isovalue)


# ----------------------------------------------------------------------------------------------------------------------------
# field evaluation (mi3d_field_forward directly: one evaluation per point, no tape)
# ----------------------------------------------------------------------------------------------------------------------------
def _field_sigma_albedo(model, pts, sigmas, rgbs):
    table, mlp_params, hg, cfg = model._field_handles()
    field_ops._check_params(table, mlp_params)
    m = pts.shape[0]
    if m == 0:
        return
    io = L.FieldIO()
    io.xyzs = pts.data_ptr(); io.dirs = None; io.counter = None; io.m_fixed = m; io.align = 0; io.cap = m
    cf = field_ops._cfg_struct(dict(cfg, n_evals=1, shading='albedo', ambient_ratio=1.0), None)
    mlp = field_ops._mlp_struct(mlp_params)
    null = C.c_void_p(0)
    L.check(L.lib().mi3d_field_forward(C.byref(io), L.ptr(table), C.byref(hg), C.byref(mlp), C.byref(cf), L.ptr(sigmas), L.ptr(rgbs),
                                       null, null, null, null, null, L.stream()), "field_forward")


@torch.no_grad()
def density_volume(model, resolution, S=128):
    """sigmas[x, y, z] of renderer.py:167-180: float32 torch.linspace(-1, 1, resolution) coordinates made on the CPU, 'ij' grid,
    chunks of S^3 points; bit-identical to model.density(pts)['sigma'] over the same loop."""
    dev = model.aabb_train.device
    lin = torch.linspace(-1, 1, resolution).to(dev)
    vol = torch.empty(resolution, resolution, resolution, dtype=torch.float32, device=dev)
    sig = torch.empty(min(S, resolution) ** 3, dtype=torch.float32, device=dev)
    for x0 in range(0, resolution, S):
        for y0 in range(0, resolution, S):
            for z0 in range(0, resolution, S):
                xs, ys, zs = lin[x0:x0 + S], lin[y0:y0 + S], lin[z0:z0 + S]
                xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing='ij')
                pts = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], dim=-1)
                m = pts.shape[0]
                _field_sigma_albedo(model, pts, sig[:m], None)
                vol[x0:x0 + len(xs), y0:y0 + len(ys), z0:z0 + len(zs)] = sig[:m].view(len(xs), len(ys), len(zs))
    return vol


def density_threshold(model):
    """min(model.mean_density, model.density_thresh) (renderer.py:163) as (float, CUDA scalar or None): a device mean_density stays
    on the device (the kernels take the minimum), so no .item() is needed."""
    md = model.mean_density
    if torch.is_tensor(md) and md.is_cuda:
        return float(model.density_thresh), md
    return float(min(float(md), float(model.density_thresh))), None


@torch.no_grad()
def extract_mesh(model, resolution, S=128):
    """-> (v fp32 [V,3] in [-1, 1], f int32 [F,3]) CUDA tensors: the export's surface (renderer.py:159-189)"""
    vol = density_volume(model, resolution, S)
    iso, iso_dev = density_threshold(model)
    return _marching_cubes_cuda(vol, iso, iso_dev, scale=2.0 / (resolution - 1.0), offset=-1.0)


# ----------------------------------------------------------------------------------------------------------------------------
# texture atlas
# ----------------------------------------------------------------------------------------------------------------------------
def atlas_layout(F):
    """-> (T, c, n): P = ceil(F/2) cells, n = ceil(sqrt(P)) per row, texture side T = smallest 2048 * 2^k with cell side
    c = floor(T / n) >= 8.  Raises Mi3dError past T = 16384."""
    if F < 1:
        raise L.Mi3dError("the atlas needs at least one face")
    P = (F + 1) // 2
    n = math.isqrt(P)
    if n * n < P:
        n += 1
    T = ATLAS_T0
    while T // n < ATLAS_MIN_CELL:
        T *= 2
        if T > ATLAS_T_MAX:
            raise L.Mi3dError(f"{F} faces need a texture larger than {ATLAS_T_MAX} x {ATLAS_T_MAX} (8-texel cells)")
    return T, T // n, n


@torch.no_grad()
def bake_texture(model, v, f):
    """-> (vt fp32 [3F,2], ft int32 [F,3], albedo fp32 [T,T,3], owner int32 [T,T]).  Owned texels carry the field albedo at their
    surface point; texels that belong to no face are 0 (as in the reference before its inpainting)."""
    L.require_cuda(v, f)
    if v.dtype != torch.float32 or f.dtype != torch.int32 or v.dim() != 2 or f.dim() != 2 or v.shape[1] != 3 or f.shape[1] != 3:
        raise L.Mi3dError("bake_texture needs v fp32 [V,3] and f int32 [F,3]")
    v, f = v.contiguous(), f.contiguous()
    F = f.shape[0]
    T, c, n = atlas_layout(F)
    dev = v.device
    points = torch.empty(T * T, 3, dtype=torch.float32, device=dev)
    owner = torch.empty(T * T, dtype=torch.int32, device=dev)
    vt = torch.empty(3 * F, 2, dtype=torch.float32, device=dev)
    L.check(L.lib().mi3d_mesh_atlas_texels(L.ptr(v), L.ptr(f), C.c_uint32(F), C.c_uint32(T), C.c_uint32(c), C.c_uint32(n),
                                           C.c_float(float(model.bound)), L.ptr(points), L.ptr(owner), L.ptr(vt), L.stream()),
            "mesh_atlas_texels")
    sig = torch.empty(T * T, dtype=torch.float32, device=dev)
    rgb = torch.empty(T * T, 3, dtype=torch.float32, device=dev)
    _field_sigma_albedo(model, points, sig, rgb)
    albedo = torch.where(owner[:, None] >= 0, rgb, torch.zeros((), dtype=torch.float32, device=dev))
    ft = torch.arange(3 * F, dtype=torch.int32, device=dev).view(F, 3)
    return vt, ft, albedo.view(T, T, 3), owner.view(T, T)


# ----------------------------------------------------------------------------------------------------------------------------
# files
# ----------------------------------------------------------------------------------------------------------------------------
def write_files(path, v, f, vt, ft, albedo, name=''):
    """mesh.obj / mesh.mtl / albedo.png in the reference's format (renderer.py:290-328).  Coordinates are printed with 9 significant
    digits, which parse back to the same float32; vt lines carry 1 - v like the reference's."""
    import cv2
    v_np, f_np = v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    vt_np, ft_np = vt.cpu().numpy(), ft.cpu().numpy().astype(np.int64)
    feats = (albedo.cpu().numpy() * 255).astype(np.uint8)            # renderer.py:265-266
    feats = cv2.cvtColor(feats, cv2.COLOR_RGB2BGR)
    cv2.imwrite(os.path.join(path, f'{name}albedo.png'), feats)
    vt_out = np.stack([vt_np[:, 0], np.float32(1) - vt_np[:, 1]], axis=-1)
    fidx = np.stack([f_np + 1, ft_np + 1], axis=-1).reshape(-1)        # f v/vt, 1-based
    with open(os.path.join(path, f'{name}mesh.obj'), "w") as fp:
        fp.write(f'mtllib {name}mesh.mtl \n')
        fp.write(('v %.9g %.9g %.9g \n' * len(v_np)) % tuple(v_np.reshape(-1).tolist()))
        fp.write(('vt %.9g %.9g \n' * len(vt_out)) % tuple(vt_out.reshape(-1).tolist()))
        fp.write('usemtl mat0 \n')
        fp.write(('f %d/%d %d/%d %d/%d \n' * len(f_np)) % tuple(fidx.tolist()))
    with open(os.path.join(path, f'{name}mesh.mtl'), "w") as fp:
        fp.write(MTL_TEXT.replace('albedo.png', f'{name}albedo.png'))


@torch.no_grad()
def export_mesh(model, path, resolution=None, S=128):
    """NeRFRenderer.export_mesh (renderer.py:157-330): writes path/mesh.obj, mesh.mtl, albedo.png; returns None.  An empty surface at
    the density threshold raises Mi3dError before any file is written."""
    if resolution is None:
        resolution = model.grid_size
    v, f = extract_mesh(model, int(resolution), S)
    if f.shape[0] == 0:
        raise L.Mi3dError(f"no surface at the density threshold (resolution {resolution}): nothing to export")
    vt, ft, albedo, _ = bake_texture(model, v, f)
    write_files(path, v, f, vt, ft, albedo)
