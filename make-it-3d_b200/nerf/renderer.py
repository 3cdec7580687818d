"""B2 seam: NeRFRenderer with the reference's attribute / buffer / method names (nerf/renderer.py:99-677).

Only the CUDA-ray path exists (main.py:95 hard-sets cuda_ray=True; the reference's pure-PyTorch `run()` is dead code).
`run_cuda`'s training branch is three launches of libmi3d.so with no host synchronisation; `update_extra_state`
keeps the mean density and the packing threshold on the device.  state_dict keys (density_grid, density_bitfield,
step_counter, aabb_train, aabb_infer) match the reference so checkpoints interchange (nerf/utils.py:1075-1186).
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from .. import _lib as L
from .. import raymarching
from . import field_ops
from .utils import safe_normalize


class NeRFRenderer(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.bound = opt.bound
        self.cascade = 1 + math.ceil(math.log2(opt.bound))
        self.grid_size = 128
        self.cuda_ray = True
        self.min_near = opt.min_near
        self.density_thresh = opt.density_thresh
        self.bg_radius = getattr(opt, "bg_radius", -1)
        aabb_train = torch.FloatTensor([-opt.bound, -opt.bound, -opt.bound, opt.bound, opt.bound, opt.bound])
        self.register_buffer('aabb_train', aabb_train)
        self.register_buffer('aabb_infer', aabb_train.clone())
        self.register_buffer('density_grid', torch.zeros([self.cascade, self.grid_size ** 3]))
        self.register_buffer('density_bitfield', torch.zeros(self.cascade * self.grid_size ** 3 // 8, dtype=torch.uint8))
        self.register_buffer('step_counter', torch.zeros(16, 2, dtype=torch.int32))
        self.mean_density = 0
        self.iter_density = 0
        self.mean_count = 0
        self.local_step = 0
        self._mean_density_dev = None
        self._workspaces = {}
        self._grid_ws = None

    # --- to be provided by the field subclass ---
    def forward(self, x, d):
        raise NotImplementedError()

    def density(self, x):
        raise NotImplementedError()

    def _field_handles(self):
        """-> (table, (w1,b1,w2,b2,w3,b3), hashgrid struct, base cfg dict)"""
        raise NotImplementedError()

    def reset_extra_state(self):
        self.density_grid.zero_()
        self.mean_density = 0
        self.iter_density = 0
        self.step_counter.zero_()
        self.mean_count = 0
        self.local_step = 0

    def _workspace(self, N, max_steps, device, n_views=1):
        key = (N, max_steps, str(device), n_views)
        ws = self._workspaces.get(key)
        if ws is None:
            # keep one workspace per shape, two shapes at most: a training loop alternates single views (front views) with one
            # multi-view batch size (coarse.train_one_epoch's views_per_step), and re-carving on every switch costs a large allocation
            ws = field_ops.RenderWorkspace(N, max_steps, device, max_samples=getattr(self.opt, "max_samples", None), n_views=n_views)
        # most recently used first (callers read the current one as list(_workspaces.values())[0]), then at most one other
        others = [(k, w) for k, w in self._workspaces.items() if k != key][:1]
        self._workspaces = dict([(key, ws)] + others)
        return ws

    def run_cuda(self, rays_o, rays_d, depth_scale=None, bg_color=None, dt_gamma=0, light_d=None, ambient_ratio=1.0,
                 shading='albedo', perturb=False, force_all_rays=False, max_steps=1024, T_thresh=1e-4, **kwargs):
        """nerf/renderer.py:481-583.  Additive optional kwargs (none collides with a reference `opt` field):
          noises[N], smooth_noise[m,3]  inject the random draws of raymarching.py:226 / renderer.py:522 (reproducible parity tests)
          cam_poses [G,4,4], cam_intrinsics (fx,fy,cx,cy) or [G,4], cam_hw (H, W)
                                        generate the rays of G views inside the march kernel (rays_o / rays_d may be None);
                                        G > 1 = a multi-view batch: image [G,HW,3], per-view losses [G]
          cam_table [G,16]              the same, as the ready device table of nerf/utils.py::camera_table (instead of cam_poses)
          ray_parallel                  parallel.RayParallel: this rank renders every world-th pixel of each of `world` views and
                                        returns the complete image of ITS OWN view (rank r owns cam_poses[r]); needs step_seed
          step_seed                     int shared by all ranks of a step (march jitter, smoothness perturbation, light directions)
        Explicit rays_o / rays_d [G,H*W,3] (depth_scale [G,H*W]) with G > 1 are a multi-view batch in training, as cam_poses are."""
        device = self.density_bitfield.device
        cam_poses = kwargs.get('cam_poses')
        cam_table = kwargs.get('cam_table')
        if cam_table is not None:
            L.require_cuda(cam_table)
            cam_poses = cam_table
        par = kwargs.get('ray_parallel')
        if cam_poses is None:
            prefix = rays_o.shape[:-1]
            rays_o = L.f32c(rays_o).view(-1, 3)
            rays_d = L.f32c(rays_d).view(-1, 3)
            L.require_cuda(rays_o, rays_d)
            N = rays_o.shape[0]
            device = rays_o.device
        elif not self.training:
            raise L.Mi3dError("cam_poses (in-kernel ray generation) is a training-path option; pass rays for evaluation")
        results = {}

        if self.training:
            table, mlp_params, hg, cfg = self._field_handles()
            cfg = dict(cfg, n_evals=13 if self.opt.lambda_smooth > 0 else 7, shading=shading, ambient_ratio=float(ambient_ratio))
            step_seed = kwargs.get('step_seed')
            if par is not None and step_seed is None:
                raise L.Mi3dError("ray_parallel needs step_seed (a value shared by all ranks, e.g. parallel.shared_seed(base, step))")
            seed = int(step_seed) if step_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())   # CPU generator: no device sync
            G, raygen, origins = 1, None, None
            if cam_poses is None and len(prefix) == 2 and prefix[0] > 1:
                G = prefix[0]
                if G > L.MAX_VIEWS or par is not None:
                    raise L.Mi3dError(f"a multi-view batch of explicit rays takes 2..{L.MAX_VIEWS} views on one rank; got {G}")
                origins = rays_o.view(G, -1, 3)[:, 0]
            if cam_poses is not None:
                from . import utils as U
                Hc, Wc = kwargs['cam_hw']
                if cam_table is not None:
                    cams = L.f32c(cam_table).view(-1, 16)
                else:
                    cam_poses = torch.as_tensor(cam_poses, dtype=torch.float32)
                    if cam_poses.dim() == 2:
                        cam_poses = cam_poses[None]
                    cams = U.camera_table(cam_poses, kwargs['cam_intrinsics'], device)
                G = cams.shape[0]
                if par is not None:
                    if G != par.world or (Hc * Wc) % par.world:
                        raise L.Mi3dError(f"ray_parallel: need one view per rank and H*W divisible by the world size (G={G}, world={par.world})")
                    rpv = Hc * Wc // par.world
                    raygen = U.raygen_struct(cams, Hc, Wc, rpv, par.world, par.rank)
                else:
                    rpv = Hc * Wc
                    raygen = U.raygen_struct(cams, Hc, Wc, rpv, 1, 0)
                self._cams = cams                                      # keep the device table alive until the backward ran
                N = G * rpv
                origins = cams[:, [3, 7, 11]]
                rays_o = rays_d = None
                prefix = (1, Hc * Wc) if (par is not None or G == 1) else (G, Hc * Wc)
            elif par is not None:
                raise L.Mi3dError("ray_parallel needs cam_poses (every rank generates its share of every view's rays)")
            multi = G > 1 or par is not None
            if light_d is None:                                        # renderer.py:496-499, one direction per view
                gen = torch.Generator().manual_seed(seed % (2 ** 63)) if step_seed is not None else None
                o = origins if origins is not None else rays_o[:1]
                light_d = safe_normalize(o + torch.randn(o.shape, generator=gen).to(device))
                if not multi:
                    light_d = light_d[0]
            light_d = L.f32c(light_d.to(device))
            ws = self._workspace(N, max_steps, device, G)
            opts = dict(bound=float(self.bound), dt_gamma=float(dt_gamma), max_steps=int(max_steps), cascade=self.cascade,
                        grid_size=self.grid_size, min_near=0.2,          # wrapper default, NOT opt.min_near (raymarching.py:34)
                        T_thresh=float(T_thresh), max_depth=float(self.opt.max_depth), seed=seed, n_views=G,
                        noise_mode=1 if (multi or step_seed is not None) else 0, pad_view_mask=(1 << par.rank) if par is not None else (1 << G) - 1)
            noises = kwargs.get('noises')
            if noises is None and not perturb:
                noises = torch.zeros(N, dtype=torch.float32, device=device)
            if bg_color is not None and not torch.is_tensor(bg_color):
                bg_color = torch.full((3,), float(bg_color), device=device)
            if bg_color is not None:
                bg_color = L.f32c(bg_color.to(device))
                if multi and bg_color.dim() == 1:
                    bg_color = bg_color.expand(G, 3).contiguous()
            ds = L.f32c(depth_scale).view(-1) if (depth_scale is not None and raygen is None) else None
            self.local_step += 1
            image, depth, weights_sum, loss_orient, loss_smooth = field_ops.render_train(
                table, mlp_params, rays_o, rays_d, self.density_bitfield, self.aabb_train, ws, hg, cfg, opts,
                noises=noises, light_d=light_d, smooth_noise=kwargs.get('smooth_noise'), bg_color=bg_color, depth_scale=ds,
                raygen=raygen, par=par)
            results['loss_orient'] = loss_orient
            if self.opt.lambda_smooth > 0:
                results['loss_smooth'] = loss_smooth
            nears, fars = ws.nears, ws.fars
            image = image.view(*prefix, 3)
            depth = depth.view(*prefix, 1)
            if par is not None:                                        # nears / fars cover this rank's ray share only
                results['image'], results['depth'], results['weights_sum'] = image, depth, weights_sum.reshape(*prefix)
                return results
        else:
            if light_d is None:                                        # renderer.py:496-499
                light_d = safe_normalize(rays_o[0] + torch.randn(3, device=device, dtype=torch.float))
            light_d = L.f32c(light_d)
            if kwargs.get('eval_loop', 'device') == 'device':
                # the whole alive-ray loop in ONE C call, loop state on the device (mi3d_render_eval; SURVEY 8f-2)
                weights_sum, depth, image, normal, nears, fars = self._render_eval_device(
                    rays_o, rays_d, depth_scale, bg_color, dt_gamma, light_d, ambient_ratio, shading, perturb, max_steps, T_thresh)
                image, normal = image.view(*prefix, 3), normal.view(*prefix, 3)
                depth = depth.view(*prefix, 1)
            else:
                weights_sum, depth, image, normal, nears, fars = self._render_eval_host_loop(
                    rays_o, rays_d, depth_scale, bg_color, dt_gamma, light_d, ambient_ratio, shading, perturb, max_steps, T_thresh, prefix)
            results['normal'] = normal

        results['image'] = image
        results['depth'] = depth
        results['weights_sum'] = weights_sum.reshape(*prefix)
        results['mask'] = (nears < fars).reshape(*prefix)
        return results

    def _render_eval_host_loop(self, rays_o, rays_d, depth_scale, bg_color, dt_gamma, light_d, ambient_ratio, shading, perturb, max_steps,
                               T_thresh, prefix):
        """The reference's host-driven loop (renderer.py:526-551) over the B1 / B2 entry points, one device->host sync per iteration
        (the boolean-mask compaction).  Kept as the A/B arm of the device-controlled loop (`eval_loop='host'`)."""
        N, device = rays_o.shape[0], rays_o.device
        nears, fars = raymarching.near_far_from_aabb(rays_o, rays_d, self.aabb_infer)
        dtype = torch.float32
        weights_sum = torch.zeros(N, dtype=dtype, device=device)
        depth = torch.zeros(N, dtype=dtype, device=device)
        image = torch.zeros(N, 3, dtype=dtype, device=device)
        normal = torch.zeros(N, 3, dtype=dtype, device=device)
        n_alive = N
        rays_alive = torch.arange(n_alive, dtype=torch.int32, device=device)
        rays_t = nears.clone()
        step = 0
        while step < max_steps:                                   # renderer.py:535-551
            n_alive = rays_alive.shape[0]
            if n_alive <= 0:
                break
            n_step = max(min(N // n_alive, 8), 1)
            xyzs, dirs, deltas = raymarching.march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, self.bound,
                                                        self.density_bitfield, self.cascade, self.grid_size, nears, fars, 128,
                                                        perturb if step == 0 else False, dt_gamma, max_steps)
            sigmas, rgbs, normals = self(xyzs, dirs, light_d, ratio=ambient_ratio, shading=shading)
            normals = (normals + 1) / 2
            raymarching.composite_rays(n_alive, n_step, rays_alive, rays_t, sigmas, rgbs, normals, deltas, weights_sum, depth,
                                       image, normal, T_thresh)
            rays_alive = rays_alive[rays_alive >= 0]
            step += n_step
        bg = 1 if bg_color is None else bg_color
        image = (image + (1 - weights_sum).unsqueeze(-1) * bg).view(*prefix, 3)
        normal = (normal + (1 - weights_sum).unsqueeze(-1) * bg).view(*prefix, 3)
        depth = depth + (1 - weights_sum) * self.opt.max_depth
        if depth_scale is not None:
            depth = depth.view(*prefix, 1) * depth_scale.view(*prefix, 1)
        else:
            depth = depth.view(*prefix, 1)
        return weights_sum, depth, image, normal, nears, fars

    def _render_eval_device(self, rays_o, rays_d, depth_scale, bg_color, dt_gamma, light_d, ambient_ratio, shading, perturb, max_steps, T_thresh):
        table, mlp_params, hg, cfg = self._field_handles()
        N, dev = rays_o.shape[0], rays_o.device
        lib = L.lib()
        key = (N, str(dev))
        if getattr(self, "_eval_ws_key", None) != key:
            self._eval_ws = torch.empty(lib.mi3d_render_eval_workspace_bytes(C.c_uint32(N)), dtype=torch.uint8, device=dev)
            self._eval_done = torch.zeros(1, dtype=torch.int32).pin_memory()      # device-written, host-polled (no sync)
            self._eval_ws_key = key
        self._eval_done.zero_()
        cfg = dict(cfg, n_evals=7, shading=shading, ambient_ratio=float(ambient_ratio))
        cf = field_ops._cfg_struct(cfg, light_d)
        mlp = field_ops._mlp_struct(mlp_params)
        if bg_color is not None and not torch.is_tensor(bg_color):
            bg_color = torch.full((3,), float(bg_color), device=dev)
        if bg_color is not None:
            bg_color = L.f32c(bg_color.to(dev))
        ds = L.f32c(depth_scale).view(-1) if depth_scale is not None else None
        a = L.RenderEvalArgs()
        a.rays_o = rays_o.data_ptr(); a.rays_d = rays_d.data_ptr(); a.depth_scale = ds.data_ptr() if ds is not None else None; a.N = N
        a.density_bitfield = self.density_bitfield.data_ptr(); a.C = self.cascade; a.H = self.grid_size
        a.bound = float(self.bound); a.dt_gamma = float(dt_gamma); a.max_steps = int(max_steps); a.min_near = 0.2
        a.aabb = self.aabb_infer.data_ptr(); a.T_thresh = float(T_thresh); a.perturb = 1 if perturb else 0
        a.seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        a.bg_color = bg_color.data_ptr() if bg_color is not None else None; a.bg_scalar = 1.0; a.max_depth = float(self.opt.max_depth)
        f32 = dict(dtype=torch.float32, device=dev)
        weights_sum, depth = torch.empty(N, **f32), torch.empty(N, **f32)
        image, normal = torch.empty(N, 3, **f32), torch.empty(N, 3, **f32)
        L.check(lib.mi3d_render_eval(C.byref(a), L.ptr(table), C.byref(hg), C.byref(mlp), C.byref(cf), L.ptr(self._eval_ws),
                                     C.c_void_p(self._eval_done.data_ptr()), L.ptr(weights_sum), L.ptr(depth), L.ptr(image), L.ptr(normal), L.stream()),
                "render_eval")
        # nears / fars live at fixed offsets of the workspace (control block 256 B, two alive lists, rays_t, then nears, fars)
        stride = (N * 4 + 255) // 256 * 256
        nears = self._eval_ws[256 + 3 * stride:256 + 3 * stride + 4 * N].view(torch.float32)
        fars = self._eval_ws[256 + 4 * stride:256 + 4 * stride + 4 * N].view(torch.float32)
        return weights_sum, depth, image, normal, nears, fars

    @torch.no_grad()
    def update_extra_state(self, decay=0.95, S=128, jitter=None, seed=None):
        """nerf/renderer.py:587-637 as ONE C-ABI call (positions, field, EMA-max, mean, packbits); no .item().
        `seed` (additive kwarg) keys the in-kernel cell jitter.  Multi-GPU callers MUST pass the same value on every rank
        (parallel.shared_seed(base, iteration)): the view-/ray-parallel step relies on bit-identical bitfields without a
        broadcast.  None draws from this process's CPU generator (single-process behaviour of the reference)."""
        table, mlp_params, hg, cfg = self._field_handles()
        dev = table.device
        lib = L.lib()
        if self._grid_ws is None or self._grid_ws.device != dev:
            nbytes = lib.mi3d_density_grid_workspace_bytes(C.c_uint32(self.cascade), C.c_uint32(self.grid_size))
            self._grid_ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            self._mean_density_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        cf = field_ops._cfg_struct(dict(cfg, n_evals=1, shading='albedo', ambient_ratio=1.0), None)
        mlp = field_ops._mlp_struct(mlp_params)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        if jitter is not None:
            jitter = L.f32c(jitter)
        L.check(lib.mi3d_density_grid_update(
            L.ptr(self.density_grid), L.ptr(self.density_bitfield), C.c_uint32(self.cascade), C.c_uint32(self.grid_size),
            C.c_float(self.bound), C.c_float(decay), C.c_float(self.density_thresh), L.ptr(table), C.byref(hg), C.byref(mlp),
            C.byref(cf), L.ptr(jitter), C.c_uint64(seed), L.ptr(self._mean_density_dev), L.ptr(self._grid_ws), L.stream()),
            "density_grid_update")
        self.mean_density = self._mean_density_dev     # device scalar; float(...) only when a checkpoint is written
        self.iter_density += 1
        self.mean_count = 0                            # unused under force_all_rays=True (nerf/utils.py:498)
        self.local_step = 0

    @torch.no_grad()
    def export_mesh(self, path, resolution=None, S=128):
        """nerf/renderer.py:157-330: marching cubes over the density volume and a baked albedo atlas, written as path/mesh.obj,
        mesh.mtl and albedo.png (nerf/mesh.py)."""
        from . import mesh
        mesh.export_mesh(self, path, resolution, S)

    def render(self, rays_o, rays_d, depth_scale=None, staged=False, max_ray_batch=4096, **kwargs):
        """nerf/renderer.py:642-677 (cuda_ray never stages)."""
        return self.run_cuda(rays_o, rays_d, depth_scale, **kwargs)
