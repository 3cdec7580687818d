"""torch.autograd.Function wrappers over the fused field / render kernels of libmi3d.so.

* ``field_eval``      -- NeRFNetwork.forward / density / normal on an explicit point set (B2 unfused seam)
* ``render_train``    -- the whole training branch of NeRFRenderer.run_cuda (nerf/renderer.py:481-524,553-583):
                         march (fused near/far, look-back compaction) -> fused field -> composite (+epilogue),
                         three launches, zero host synchronisation; backward = composite-bwd + fused field-bwd.
Gradients flow to (table, w1, b1, w2, b2, w3, b3) only, exactly the leaves the reference optimises
(nerf/network_tcnn.py:195-206); positions get none (tcnn is asked for none, SURVEY.md 8a-E1).
"""
import ctypes as C

import torch
from torch.autograd import Function

from .. import _lib as L


# Optional live kernel timing (bench.py roofline leg): a list that receives (kernel_name, start_event, end_event, info) tuples,
# recorded on the launching stream around the C-ABI call.  None = off (no events, no overhead).
PROFILE = None


def _timed(name, info, fn):
    if PROFILE is None:
        return fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    r = fn()
    e.record()
    PROFILE.append((name, s, e, info))
    return r


_BWD_SCRATCH = {}


def bwd_scratch(device):
    """per-device staging buffer of the split backward pipeline (mi3d_field_backward_workspace_bytes), allocated once"""
    key = str(device)
    if key not in _BWD_SCRATCH:
        _BWD_SCRATCH[key] = torch.empty(L.lib().mi3d_field_backward_workspace_bytes(), dtype=torch.uint8, device=device)
    return _BWD_SCRATCH[key]


def make_hashgrid(n_levels=16, base_resolution=16, per_level_scale=1.3819128274917603, log2_hashmap_size=19):
    hg = L.HashGrid()
    L.check(L.lib().mi3d_hashgrid_make(C.c_uint32(n_levels), C.c_uint32(base_resolution), C.c_double(per_level_scale),
                                       C.c_uint32(log2_hashmap_size), C.byref(hg)), "hashgrid_make")
    return hg


def _mlp_struct(ws):
    m = L.Mlp()
    for name, t in zip(("w1", "b1", "w2", "b2", "w3", "b3"), ws):
        setattr(m, name, t.data_ptr())
    return m


def _cfg_struct(cfg, light_d):
    c = L.FieldCfg()
    c.bound = cfg["bound"]; c.blob_density = cfg["blob_density"]; c.blob_radius = cfg["blob_radius"]
    c.n_evals = cfg["n_evals"]; c.shading = L.SHADING[cfg["shading"]]; c.ambient_ratio = cfg["ambient_ratio"]
    c.light_d = light_d.data_ptr() if light_d is not None else None
    return c


def _check_params(table, ws):
    L.require_cuda(table, *ws)
    shapes = [(64, 32), (64,), (64, 64), (64,), (4, 64), (4,)]
    for t, s in zip(ws, shapes):
        if tuple(t.shape) != s or t.dtype != torch.float32 or not t.is_contiguous():
            raise L.Mi3dError(f"sigma_net must be MLP(32,4,64,3) fp32 contiguous; got {tuple(t.shape)} {t.dtype}")
    if table.dtype != torch.float32 or not table.is_contiguous():
        raise L.Mi3dError("encoder.params must be a contiguous fp32 tensor")


def _grad_or_none(g):
    return None if g is None else L.f32c(g)


class _FieldEval(Function):
    """sigma, color, normal, loss_orient, loss_smooth = field(table, mlp..., xyzs, dirs, light_d)"""

    @staticmethod
    def forward(ctx, table, w1, b1, w2, b2, w3, b3, xyzs, dirs, light_d, smooth_noise, hg, cfg, seed):
        ws = (w1, b1, w2, b2, w3, b3)
        _check_params(table, ws)
        xyzs = L.f32c(xyzs)
        dirs = L.f32c(dirs) if dirs is not None else None
        L.require_cuda(xyzs, dirs, light_d, smooth_noise)
        m = xyzs.shape[0]
        dev = xyzs.device
        sigmas = torch.empty(m, dtype=torch.float32, device=dev)
        rgbs = torch.empty(m, 3, dtype=torch.float32, device=dev)
        normals = torch.empty(m, 3, dtype=torch.float32, device=dev) if cfg["n_evals"] >= 7 else None
        tape = torch.empty(m, 16, dtype=torch.float32, device=dev)
        nct = L.lib().mi3d_field_grid_ctas(C.c_int(0))
        partials = torch.empty(2 * nct, dtype=torch.float32, device=dev)
        losses = torch.zeros(2, dtype=torch.float32, device=dev)
        io = L.FieldIO()
        io.xyzs = xyzs.data_ptr(); io.dirs = dirs.data_ptr() if dirs is not None else None
        io.counter = None; io.m_fixed = m; io.align = 0; io.cap = m
        io.smooth_noise = smooth_noise.data_ptr() if smooth_noise is not None else None
        io.seed = seed
        mlp, cf = _mlp_struct(ws), _cfg_struct(cfg, light_d)
        if m > 0:
            L.check(L.lib().mi3d_field_forward(C.byref(io), L.ptr(table), C.byref(hg), C.byref(mlp), C.byref(cf), L.ptr(sigmas),
                                               L.ptr(rgbs), L.ptr(normals), L.ptr(tape), L.ptr(partials),
                                               C.c_void_p(losses.data_ptr()), C.c_void_p(losses.data_ptr() + 4), L.stream()),
                    "field_forward")
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(table, w1, b1, w2, b2, w3, b3, xyzs, dirs, light_d, smooth_noise, tape)
        ctx.hg, ctx.cfg, ctx.seed, ctx.m = hg, cfg, seed, m
        if normals is None:
            normals = torch.zeros(m, 3, dtype=torch.float32, device=dev)
        return sigmas, rgbs, normals, losses[0], losses[1]

    @staticmethod
    def backward(ctx, g_sigmas, g_rgbs, g_normals, g_lo, g_ls):
        table, w1, b1, w2, b2, w3, b3, xyzs, dirs, light_d, smooth_noise, tape = ctx.saved_tensors
        ws = (w1, b1, w2, b2, w3, b3)
        g_table = torch.zeros_like(table)
        g_ws = [torch.zeros_like(w) for w in ws]
        if ctx.m > 0:
            io = L.FieldIO()
            io.xyzs = xyzs.data_ptr(); io.dirs = dirs.data_ptr() if dirs is not None else None
            io.counter = None; io.m_fixed = ctx.m; io.align = 0; io.cap = ctx.m
            io.smooth_noise = smooth_noise.data_ptr() if smooth_noise is not None else None
            io.seed = ctx.seed
            mlp, cf = _mlp_struct(ws), _cfg_struct(ctx.cfg, light_d)
            gm = _mlp_struct(g_ws)
            g_sigmas, g_rgbs, g_normals = _grad_or_none(g_sigmas), _grad_or_none(g_rgbs), _grad_or_none(g_normals)
            g_lo, g_ls = _grad_or_none(g_lo), _grad_or_none(g_ls)
            if ctx.cfg["n_evals"] < 7:
                g_normals = None
            L.check(L.lib().mi3d_field_backward(C.byref(io), L.ptr(table), C.byref(ctx.hg), C.byref(mlp), C.byref(cf), L.ptr(tape),
                                                L.ptr(g_sigmas), L.ptr(g_rgbs), L.ptr(g_normals), L.ptr(g_lo), L.ptr(g_ls),
                                                L.ptr(g_table), C.byref(gm), L.ptr(bwd_scratch(table.device)), L.stream()), "field_backward")
        return (g_table, *g_ws, None, None, None, None, None, None, None)


def field_eval(table, mlp_params, xyzs, dirs, light_d, hg, cfg, smooth_noise=None, seed=0):
    return _FieldEval.apply(table, *mlp_params, xyzs, dirs, light_d, smooth_noise, hg, cfg, seed)


def _blob_view(blob, ptr, shape, dtype):
    """tensor view of a carved sub-buffer of the workspace blob (ptr = absolute device address inside blob)"""
    item = torch.empty(0, dtype=dtype).element_size()
    n = 1
    for d in shape:
        n *= d
    off = ptr - blob.data_ptr()
    return blob[off:off + n * item].view(dtype).view(*shape)


class RenderWorkspace:
    """Capacity-sized per-sample / per-ray buffers carved by the library out of ONE device blob (mi3d_render_workspace_carve),
    allocated once and reused every step: no zero-fill, no empty_cache (the 268 MB/step torch.zeros + allocator flush of
    raymarching.py:217-243 disappears).  The tensor attributes are views into the blob (tests and tools read them)."""

    def __init__(self, N, max_steps, device, max_samples=None, n_views=1):
        lib = L.lib()
        self.N, self.device, self.n_views = N, device, n_views
        # hash-grid encodings of the first 8192 tiles (1 M samples x 13 evaluation points, 1.7 GB at full size): written by the
        # forward, read back by the backward passes of the same step instead of re-gathering the table
        args = (C.c_uint32(N), C.c_uint32(max_steps), C.c_uint32(max_samples or 0), C.c_uint32(n_views), C.c_uint32(8192))
        self.c = L.RenderWs()
        L.check(lib.mi3d_render_workspace_carve(C.c_void_p(0), *args, C.byref(self.c)), "render_workspace_carve")
        self.blob = torch.empty(self.c.bytes, dtype=torch.uint8, device=device)
        L.check(lib.mi3d_render_workspace_carve(C.c_void_p(self.blob.data_ptr()), *args, C.byref(self.c)), "render_workspace_carve")
        c, cap = self.c, self.c.cap
        self.cap = cap
        f32, i32 = torch.float32, torch.int32
        v = lambda name, shape, dt=f32: _blob_view(self.blob, getattr(c, name), shape, dt)
        self.xyzs, self.dirs, self.deltas = v("xyzs", (cap, 3)), v("dirs", (cap, 3)), v("deltas", (cap, 2))
        self.sigmas, self.rgbs, self.tape = v("sigmas", (cap,)), v("rgbs", (cap, 3)), v("tape", (cap, 16))
        self.g_sigmas, self.g_rgbs = v("g_sigmas", (cap,)), v("g_rgbs", (cap, 3))
        self.rays, self.counter = v("rays", (N, 3), i32), v("counter", (2,), i32)
        self.nears, self.fars = v("nears", (N,)), v("fars", (N,))
        self.ws_raw, self.depth_raw, self.image_raw = v("ws_raw", (N,)), v("depth_raw", (N,)), v("image_raw", (N, 3))
        self.depth_scale = v("depth_scale", (N,))
        self.scan_ws = _blob_view(self.blob, c.scan_ws, (lib.mi3d_march_rays_train_workspace_bytes(C.c_uint32(N)),), torch.uint8)
        self.partials = v("loss_partials", (2 * n_views * lib.mi3d_field_grid_ctas(C.c_int(0)),))
        self.view_counts = v("view_counts", (L.MAX_VIEWS,), i32)
        self.counter.zero_(); self.view_counts.zero_()
        self.enc_tiles = c.enc_cache_tiles
        self.enc_cache = _blob_view(self.blob, c.enc_cache, (lib.mi3d_field_enc_cache_bytes(C.c_uint32(self.enc_tiles)),), torch.uint8)
        self.generation = 0

    def segs(self):
        """host copy of the device segment table of the last multi-view forward (debug / tests; synchronises)"""
        raw = _blob_view(self.blob, self.c.segs, (C.sizeof(L.ViewSegs) // 4,), torch.int32).cpu().numpy().tobytes()
        return L.ViewSegs.from_buffer_copy(raw)


def _render_args(ws, N, rays_o, rays_d, depth_scale, raygen, bitfield, aabb, noises, smooth_noise, bg_color, opts, par):
    ra = L.RenderArgs()
    ra.rays_o = rays_o.data_ptr() if rays_o is not None else None
    ra.rays_d = rays_d.data_ptr() if rays_d is not None else None
    ra.depth_scale = depth_scale.data_ptr() if depth_scale is not None else None
    ra.raygen = C.pointer(raygen) if raygen is not None else None
    ra.N = N; ra.n_views = opts.get("n_views", 1)
    ra.density_bitfield = bitfield.data_ptr(); ra.C = opts["cascade"]; ra.H = opts["grid_size"]
    ra.bound = opts["bound"]; ra.dt_gamma = opts["dt_gamma"]; ra.max_steps = opts["max_steps"]; ra.min_near = opts["min_near"]
    ra.aabb = aabb.data_ptr(); ra.noises = noises.data_ptr() if noises is not None else None; ra.seed = opts["seed"]
    ra.T_thresh = opts["T_thresh"]; ra.bg_color = bg_color.data_ptr() if bg_color is not None else None; ra.bg_scalar = 1.0
    ra.max_depth = opts["max_depth"]
    ra.smooth_noise = smooth_noise.data_ptr() if smooth_noise is not None else None
    ra.noise_mode = opts.get("noise_mode", 0)
    ra.all_counts = par["all_counts"].data_ptr() if par is not None else None
    ra.n_ranks = par["world"] if par is not None else 1
    ra.pad_view_mask = opts.get("pad_view_mask", (1 << ra.n_views) - 1)
    return ra


class _RenderTrain(Function):
    """image, depth, weights_sum, loss_orient, loss_smooth = render(...) through mi3d_render_forward / mi3d_render_backward: ONE C call
    per direction (march [+ray generation] -> fused field -> composite + epilogue).  With `par` (parallel.RayParallel) the batch is
    this rank's share of every view of the step: per-view sample counts are all-gathered between the march and the field (device
    side, no host sync), image fragments travel to the view's owner in one all-to-all, and the backward sends the gradient
    fragments back the same way (DESIGN.md section 5)."""

    @staticmethod
    def forward(ctx, table, w1, b1, w2, b2, w3, b3, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color,
                depth_scale, ws, hg, cfg, opts, raygen, par):
        P = (w1, b1, w2, b2, w3, b3)
        _check_params(table, P)
        if rays_o is not None:
            rays_o, rays_d = L.f32c(rays_o).view(-1, 3), L.f32c(rays_d).view(-1, 3)
        L.require_cuda(rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color, depth_scale)
        N = ws.N
        if rays_o is not None and rays_o.shape[0] != N:
            raise L.Mi3dError(f"workspace built for {ws.N} rays, got {rays_o.shape[0]}")
        dev = table.device
        lib = L.lib()
        nv = opts.get("n_views", 1)
        ws.generation += 1
        pdict = None
        if par is not None:
            pdict = dict(world=par.world, all_counts=torch.empty(par.world, nv, dtype=torch.int32, device=dev))
        ra = _render_args(ws, N, rays_o, rays_d, depth_scale, raygen, bitfield, aabb, noises, smooth_noise, bg_color, opts, pdict)
        mlp, cf = _mlp_struct(P), _cfg_struct(cfg, light_d)
        multi = nv > 1 or par is not None
        losses = torch.zeros(2, nv if multi else 1, dtype=torch.float32, device=dev)
        image = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        weights_sum = torch.empty(N, dtype=torch.float32, device=dev)

        def call(phases):
            L.check(lib.mi3d_render_forward(C.byref(ra), L.ptr(table), C.byref(hg), C.byref(mlp), C.byref(cf), C.byref(ws.c), C.c_int(phases),
                                            L.ptr(image), L.ptr(depth), L.ptr(weights_sum), C.c_void_p(losses[0].data_ptr()),
                                            C.c_void_p(losses[1].data_ptr()), L.stream()), "render_forward")
        if par is None:
            call(L.RENDER_PHASE_ALL)
        else:
            call(L.RENDER_PHASE_MARCH)
            par.gather_counts(ws.view_counts[:nv], pdict["all_counts"])
            call(L.RENDER_PHASE_SHADE)
        ctx.set_materialize_grads(False)        # unused outputs arrive as None -> the backward skips evaluations that get no gradient
        ctx.save_for_backward(table, w1, b1, w2, b2, w3, b3, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color, depth_scale)
        ctx.ws, ctx.hg, ctx.cfg, ctx.opts, ctx.N, ctx.generation, ctx.raygen, ctx.par, ctx.pdict = ws, hg, cfg, opts, N, ws.generation, raygen, par, pdict
        if par is not None:
            # fragments [view][ray-in-fragment] -> the owner of each view; own view comes back complete
            packed = torch.cat([image, depth[:, None], weights_sum[:, None]], dim=1)           # [N, 5]
            full = par.fragments_to_owner(packed, nv)                                           # [N, 5] of this rank's view
            lsum = par.reduce_losses(losses)                                                    # [2, nv] summed over ranks
            image, depth, weights_sum = full[:, :3].contiguous(), full[:, 3].contiguous(), full[:, 4].contiguous()
            return image, depth, weights_sum, lsum[0, par.rank], lsum[1, par.rank]
        if multi:
            return image, depth, weights_sum, losses[0], losses[1]
        return image, depth, weights_sum, losses[0, 0], losses[1, 0]

    @staticmethod
    def backward(ctx, g_image, g_depth, g_ws, g_lo, g_ls):
        (table, w1, b1, w2, b2, w3, b3, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color, depth_scale) = ctx.saved_tensors
        ws, N, opts, par = ctx.ws, ctx.N, ctx.opts, ctx.par
        if ws.generation != ctx.generation:
            raise L.Mi3dError("render workspace was reused by a later forward before this backward ran")
        P = (w1, b1, w2, b2, w3, b3)
        lib = L.lib()
        dev = table.device
        nv = opts.get("n_views", 1)
        g_image = L.f32c(g_image) if g_image is not None else torch.zeros(N, 3, dtype=torch.float32, device=dev)
        g_depth, g_ws = _grad_or_none(g_depth), _grad_or_none(g_ws)
        g_lo, g_ls = _grad_or_none(g_lo), _grad_or_none(g_ls)
        if par is not None:
            z = torch.zeros(N, dtype=torch.float32, device=dev)
            packed = torch.cat([g_image, (g_depth if g_depth is not None else z)[:, None], (g_ws if g_ws is not None else z)[:, None]], dim=1)
            frag = par.owner_to_fragments(packed, nv)                                            # [N, 5] in batch order
            g_image, g_depth, g_ws = frag[:, :3].contiguous(), frag[:, 3].contiguous(), frag[:, 4].contiguous()
            zero = torch.zeros((), dtype=torch.float32, device=dev)
            gl = par.gather_loss_grads(torch.stack([g_lo if g_lo is not None else zero, g_ls if g_ls is not None else zero]))   # [world, 2]
            had_lo, had_ls = g_lo is not None, g_ls is not None
            g_lo, g_ls = (gl[:, 0].contiguous() if had_lo else None), (gl[:, 1].contiguous() if had_ls else None)
        ra = _render_args(ws, N, rays_o, rays_d, depth_scale, ctx.raygen, bitfield, aabb, noises, smooth_noise, bg_color, opts, ctx.pdict)
        g_table = torch.zeros_like(table)
        g_P = [torch.zeros_like(w) for w in P]
        mlp, cf, gm = _mlp_struct(P), _cfg_struct(ctx.cfg, light_d), _mlp_struct(g_P)
        full = (g_lo is not None) or (g_ls is not None) or ctx.cfg["shading"] != "albedo"
        _timed("render_bwd", dict(n_evals=ctx.cfg["n_evals"], N=N, full=full), lambda: L.check(lib.mi3d_render_backward(
            C.byref(ra), L.ptr(table), C.byref(ctx.hg), C.byref(mlp), C.byref(cf), C.byref(ws.c), L.ptr(g_image), L.ptr(g_depth), L.ptr(g_ws),
            L.ptr(g_lo), L.ptr(g_ls), L.ptr(g_table), C.byref(gm), L.ptr(bwd_scratch(table.device)), C.c_int(1), L.stream()), "render_backward"))
        return (g_table, *g_P) + (None,) * 15


def render_train(table, mlp_params, rays_o, rays_d, bitfield, aabb, ws, hg, cfg, opts, noises=None, light_d=None,
                 smooth_noise=None, bg_color=None, depth_scale=None, raygen=None, par=None):
    """Returns (image[N,3], depth[N], weights_sum[N], loss_orient, loss_smooth).  rays_o / rays_d explicit, or raygen (L.RayGen)
    to generate them inside the march kernel.  opts['n_views'] > 1: multi-view batch (losses are [n_views]).  par: ray-parallel
    multi-GPU step, outputs are this rank's own complete view."""
    if PROFILE is not None and par is None and opts.get("n_views", 1) == 1 and rays_o is not None:
        # bench.py's per-kernel roofline leg: the same kernels through the unfused entry points, CUDA events around the field calls
        return _RenderTrainUnfused.apply(table, *mlp_params, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color,
                                         depth_scale, ws, hg, cfg, opts)
    return _RenderTrain.apply(table, *mlp_params, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color,
                              depth_scale, ws, hg, cfg, opts, raygen, par)


class _RenderTrainUnfused(Function):
    """The same step through the separate B1 / B2 entry points (march, field, composite: three C calls + torch glue).  Kept as the
    A/B arm of tests/test_field_gpu.py::test_fused_entry_points_match_unfused and for per-kernel CUDA-event timing (bench.py)."""

    @staticmethod
    def forward(ctx, table, w1, b1, w2, b2, w3, b3, rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color,
                depth_scale, ws, hg, cfg, opts):
        P = (w1, b1, w2, b2, w3, b3)
        _check_params(table, P)
        rays_o, rays_d = L.f32c(rays_o).view(-1, 3), L.f32c(rays_d).view(-1, 3)
        L.require_cuda(rays_o, rays_d, bitfield, aabb, noises, light_d, smooth_noise, bg_color, depth_scale)
        N = rays_o.shape[0]
        if N != ws.N:
            raise L.Mi3dError(f"workspace built for {ws.N} rays, got {N}")
        dev = rays_o.device
        lib = L.lib()
        ws.generation += 1
        ws.counter.zero_()                                                     # renderer.py:504
        L.check(lib.mi3d_march_rays_train(
            L.ptr(rays_o), L.ptr(rays_d), L.ptr(bitfield), C.c_float(opts["bound"]), C.c_float(opts["dt_gamma"]),
            C.c_uint32(opts["max_steps"]), C.c_uint32(N), C.c_uint32(opts["cascade"]), C.c_uint32(opts["grid_size"]),
            C.c_uint32(ws.cap - 128), C.c_void_p(0), C.c_void_p(0), L.ptr(aabb), C.c_float(opts["min_near"]), L.ptr(ws.nears),
            L.ptr(ws.fars), L.ptr(noises), C.c_uint64(opts["seed"]), L.ptr(ws.xyzs), L.ptr(ws.dirs), L.ptr(ws.deltas), L.ptr(ws.rays),
            L.ptr(ws.counter), L.ptr(ws.scan_ws), L.stream()), "march_rays_train")
        io = L.FieldIO()
        io.xyzs = ws.xyzs.data_ptr(); io.dirs = ws.dirs.data_ptr(); io.counter = ws.counter.data_ptr()
        io.m_fixed = 0; io.align = 128; io.cap = ws.cap
        io.smooth_noise = smooth_noise.data_ptr() if smooth_noise is not None else None
        io.seed = opts["seed"] + 1; io.noise_mode = opts.get("noise_mode", 0)
        io.enc_cache = ws.enc_cache.data_ptr(); io.enc_cache_tiles = ws.enc_tiles; io.enc_cache_valid = 0
        mlp, cf = _mlp_struct(P), _cfg_struct(cfg, light_d)
        losses = torch.zeros(2, dtype=torch.float32, device=dev)
        _timed("k_field_fwd", dict(n_evals=cfg["n_evals"], N=N), lambda: L.check(lib.mi3d_field_forward(
            C.byref(io), L.ptr(table), C.byref(hg), C.byref(mlp), C.byref(cf), L.ptr(ws.sigmas), L.ptr(ws.rgbs), C.c_void_p(0),
            L.ptr(ws.tape), L.ptr(ws.partials), C.c_void_p(losses.data_ptr()), C.c_void_p(losses.data_ptr() + 4), L.stream()),
            "field_forward"))
        ep = L.Epilogue()
        ep.bg_color = bg_color.data_ptr() if bg_color is not None else None
        ep.bg_scalar = 1.0
        ep.max_depth = opts["max_depth"]
        ep.depth_scale = depth_scale.data_ptr() if depth_scale is not None else None
        image = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        L.check(lib.mi3d_composite_rays_train_forward(
            L.ptr(ws.sigmas), L.ptr(ws.rgbs), L.ptr(ws.deltas), L.ptr(ws.rays), C.c_uint32(ws.cap - 128), C.c_uint32(N),
            C.c_float(opts["T_thresh"]), L.ptr(ws.ws_raw), L.ptr(ws.depth_raw), L.ptr(ws.image_raw), C.byref(ep), L.ptr(image),
            L.ptr(depth), L.stream()), "composite_rays_train_forward")
        weights_sum = ws.ws_raw.clone()
        ctx.set_materialize_grads(False)        # unused outputs arrive as None -> the backward skips evaluations that get no gradient
        ctx.save_for_backward(table, w1, b1, w2, b2, w3, b3, light_d, smooth_noise, bg_color, depth_scale)
        ctx.ws, ctx.hg, ctx.cfg, ctx.opts, ctx.N, ctx.generation = ws, hg, cfg, opts, N, ws.generation
        ctx.io_seed = io.seed
        return image, depth, weights_sum, losses[0], losses[1]

    @staticmethod
    def backward(ctx, g_image, g_depth, g_ws, g_lo, g_ls):
        table, w1, b1, w2, b2, w3, b3, light_d, smooth_noise, bg_color, depth_scale = ctx.saved_tensors
        ws, N, opts = ctx.ws, ctx.N, ctx.opts
        if ws.generation != ctx.generation:
            raise L.Mi3dError("render workspace was reused by a later forward before this backward ran")
        P = (w1, b1, w2, b2, w3, b3)
        lib = L.lib()
        dev = table.device
        g_image = L.f32c(g_image) if g_image is not None else torch.zeros(N, 3, dtype=torch.float32, device=dev)
        g_depth, g_ws = _grad_or_none(g_depth), _grad_or_none(g_ws)
        ep = L.Epilogue()
        ep.bg_color = bg_color.data_ptr() if bg_color is not None else None
        ep.bg_scalar = 1.0
        ep.max_depth = opts["max_depth"]
        ep.depth_scale = depth_scale.data_ptr() if depth_scale is not None else None
        L.check(lib.mi3d_composite_rays_train_backward(
            L.ptr(g_ws), L.ptr(g_image), L.ptr(g_depth), L.ptr(ws.sigmas), L.ptr(ws.rgbs), L.ptr(ws.deltas), L.ptr(ws.rays),
            L.ptr(ws.ws_raw), L.ptr(ws.image_raw), C.c_uint32(ws.cap - 128), C.c_uint32(N), C.c_float(opts["T_thresh"]), C.byref(ep),
            L.ptr(ws.g_sigmas), L.ptr(ws.g_rgbs), C.c_int(1), L.stream()), "composite_rays_train_backward")
        g_table = torch.zeros_like(table)
        g_P = [torch.zeros_like(w) for w in P]
        io = L.FieldIO()
        io.xyzs = ws.xyzs.data_ptr(); io.dirs = ws.dirs.data_ptr(); io.counter = ws.counter.data_ptr()
        io.m_fixed = 0; io.align = 128; io.cap = ws.cap
        io.smooth_noise = smooth_noise.data_ptr() if smooth_noise is not None else None
        io.seed = ctx.io_seed; io.noise_mode = opts.get("noise_mode", 0)
        io.enc_cache = ws.enc_cache.data_ptr(); io.enc_cache_tiles = ws.enc_tiles; io.enc_cache_valid = 1 if ctx.generation == ws.generation else 0
        mlp, cf, gm = _mlp_struct(P), _cfg_struct(ctx.cfg, light_d), _mlp_struct(g_P)
        g_lo, g_ls = _grad_or_none(g_lo), _grad_or_none(g_ls)
        full = (g_lo is not None) or (g_ls is not None) or ctx.cfg["shading"] != "albedo"
        _timed("k_field_bwd", dict(n_evals=ctx.cfg["n_evals"], N=N, full=full), lambda: L.check(lib.mi3d_field_backward(
            C.byref(io), L.ptr(table), C.byref(ctx.hg), C.byref(mlp), C.byref(cf), L.ptr(ws.tape), L.ptr(ws.g_sigmas), L.ptr(ws.g_rgbs),
            C.c_void_p(0), L.ptr(g_lo), L.ptr(g_ls), L.ptr(g_table), C.byref(gm), L.ptr(bwd_scratch(table.device)), L.stream()), "field_backward"))
        return (g_table, *g_P) + (None,) * 13


