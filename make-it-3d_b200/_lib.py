"""ctypes binding of libmi3d.so (C ABI declared in include/mi3d.h).

The product path has NO fallback: if the shared library is missing, or a call returns non-zero, we raise.
"""
import contextlib
import ctypes as C
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MI3D_LIB_PATH") or os.path.join(_HERE, "libmi3d.so")      # override: A/B builds under tools/
_lib = None


class Mi3dError(RuntimeError):
    pass


class HashGrid(C.Structure):
    _fields_ = [("n_levels", C.c_uint32), ("n_entries", C.c_uint32), ("offsets", C.c_uint32 * 16),
                ("sizes", C.c_uint32 * 16), ("ress", C.c_uint32 * 16), ("scales", C.c_float * 16)]


class RayGen(C.Structure):
    _fields_ = [("cams", C.c_void_p), ("n_views", C.c_uint32), ("H", C.c_uint32), ("W", C.c_uint32), ("rays_per_view", C.c_uint32),
                ("pixel_stride", C.c_uint32), ("pixel_phase", C.c_uint32)]


class Mlp(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1", "b1", "w2", "b2", "w3", "b3")]


class Epilogue(C.Structure):
    _fields_ = [("bg_color", C.c_void_p), ("bg_scalar", C.c_float), ("max_depth", C.c_float), ("depth_scale", C.c_void_p),
                ("rays_per_view", C.c_uint32)]


class FieldCfg(C.Structure):
    _fields_ = [("bound", C.c_float), ("blob_density", C.c_float), ("blob_radius", C.c_float), ("n_evals", C.c_int),
                ("shading", C.c_int), ("ambient_ratio", C.c_float), ("light_d", C.c_void_p)]


class FieldIO(C.Structure):
    _fields_ = [("xyzs", C.c_void_p), ("dirs", C.c_void_p), ("counter", C.c_void_p), ("m_fixed", C.c_uint32),
                ("align", C.c_uint32), ("cap", C.c_uint32), ("smooth_noise", C.c_void_p), ("seed", C.c_uint64),
                ("enc_cache", C.c_void_p), ("enc_cache_tiles", C.c_uint32), ("enc_cache_valid", C.c_uint32),
                ("segs", C.c_void_p), ("n_views", C.c_uint32), ("noise_mode", C.c_uint32)]


MAX_VIEWS = 8


class ViewSegs(C.Structure):
    _fields_ = [("n_views", C.c_uint32), ("bounds", C.c_uint32 * (2 * MAX_VIEWS + 1)), ("mpad", C.c_uint32 * MAX_VIEWS)]


class AdanCfg(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("beta3", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("max_grad_norm", C.c_float), ("clip_grad_norm", C.c_float), ("no_prox", C.c_int),
                ("step", C.c_int), ("reset_prev", C.c_int)]


class AdamCfg(C.Structure):
    """mi3d_adam_cfg: one clip + torch.optim.Adam step of mi3d_adam_step"""
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double), ("step", C.c_int),
                ("clip_grad_norm", C.c_float)]


class RenderArgs(C.Structure):
    _fields_ = [("rays_o", C.c_void_p), ("rays_d", C.c_void_p), ("depth_scale", C.c_void_p), ("raygen", C.POINTER(RayGen)), ("N", C.c_uint32),
                ("n_views", C.c_uint32), ("density_bitfield", C.c_void_p), ("C", C.c_uint32), ("H", C.c_uint32), ("bound", C.c_float),
                ("dt_gamma", C.c_float), ("max_steps", C.c_uint32), ("min_near", C.c_float), ("aabb", C.c_void_p), ("noises", C.c_void_p),
                ("seed", C.c_uint64), ("T_thresh", C.c_float), ("bg_color", C.c_void_p), ("bg_scalar", C.c_float), ("max_depth", C.c_float),
                ("smooth_noise", C.c_void_p), ("noise_mode", C.c_uint32), ("all_counts", C.c_void_p), ("n_ranks", C.c_uint32),
                ("pad_view_mask", C.c_uint32)]


class RenderEvalArgs(C.Structure):
    _fields_ = [("rays_o", C.c_void_p), ("rays_d", C.c_void_p), ("depth_scale", C.c_void_p), ("N", C.c_uint32), ("density_bitfield", C.c_void_p),
                ("C", C.c_uint32), ("H", C.c_uint32), ("bound", C.c_float), ("dt_gamma", C.c_float), ("max_steps", C.c_uint32), ("min_near", C.c_float),
                ("aabb", C.c_void_p), ("T_thresh", C.c_float), ("perturb", C.c_int), ("seed", C.c_uint64), ("bg_color", C.c_void_p),
                ("bg_scalar", C.c_float), ("max_depth", C.c_float)]


class RenderWs(C.Structure):
    _fields_ = [("N", C.c_uint32), ("cap", C.c_uint32), ("n_views", C.c_uint32)] + \
               [(n, C.c_void_p) for n in ("xyzs", "dirs", "deltas", "sigmas", "rgbs", "tape", "g_sigmas", "g_rgbs", "rays", "counter", "nears",
                                          "fars", "ws_raw", "depth_raw", "image_raw", "depth_scale", "scan_ws", "loss_partials", "view_counts",
                                          "segs", "enc_cache")] + [("enc_cache_tiles", C.c_uint32), ("bytes", C.c_size_t)]


class OpGemmArgs(C.Structure):
    """mi3d_op_gemm_args: one plan::Builder::gemm (test path)"""
    _fields_ = [("a", C.c_void_p), ("lda", C.c_longlong), ("a_rows", C.c_longlong), ("K", C.c_int), ("a_z1", C.c_int), ("a_sz1", C.c_longlong),
                ("a_z2", C.c_int), ("a_sz2", C.c_longlong),
                ("b", C.c_void_p), ("ldb", C.c_longlong), ("b_rows", C.c_longlong), ("b_z1", C.c_int), ("b_sz1", C.c_longlong),
                ("b_z2", C.c_int), ("b_sz2", C.c_longlong),
                ("N", C.c_int), ("batch", C.c_int), ("b_batched", C.c_int),
                ("out16", C.c_void_p), ("out32", C.c_void_p), ("ldc", C.c_longlong), ("out_z1", C.c_int), ("out_s_lo", C.c_longlong),
                ("out_s_hi", C.c_longlong),
                ("bias", C.c_void_p), ("row_bias", C.c_void_p), ("rows_per_group", C.c_int), ("residual", C.c_void_p), ("ld_res", C.c_longlong),
                ("mode", C.c_int), ("alpha", C.c_float), ("aux", C.c_void_p)]


class AdamSegment(C.Structure):
    """mi3d_adam_segment: one parameter tensor of mi3d_refine_adam"""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("offset", C.c_ulonglong), ("n", C.c_ulonglong)]


RENDER_PHASE_MARCH, RENDER_PHASE_SHADE, RENDER_PHASE_ALL = 1, 2, 3

SHADING = {"albedo": 0, "lambertian": 1, "textureless": 2, "normal": 3}

# every symbol include/mi3d.h declares (tests/test_abi.py checks the .so exports exactly these)
SYMBOLS = [
    "mi3d_near_far_from_aabb", "mi3d_morton3D", "mi3d_morton3D_invert", "mi3d_packbits",
    "mi3d_march_rays_train_workspace_bytes", "mi3d_march_rays_train", "mi3d_march_rays_train_cam", "mi3d_get_rays",
    "mi3d_composite_rays_train_forward", "mi3d_composite_rays_train_backward",
    "mi3d_march_rays", "mi3d_composite_rays",
    "mi3d_hashgrid_make", "mi3d_hashgrid_forward", "mi3d_hashgrid_backward",
    "mi3d_field_grid_ctas", "mi3d_field_forward", "mi3d_field_backward", "mi3d_field_backward_workspace_bytes", "mi3d_field_enc_cache_bytes",
    "mi3d_render_workspace_bytes", "mi3d_render_workspace_carve", "mi3d_render_forward", "mi3d_render_backward",
    "mi3d_render_eval_workspace_bytes", "mi3d_render_eval",
    "mi3d_density_grid_workspace_bytes", "mi3d_density_grid_update", "mi3d_version",
    "mi3d_sumsq_workspace_bytes", "mi3d_sumsq", "mi3d_adan_step", "mi3d_adam_step",
    "mi3d_gemm_f16", "mi3d_gemm_f16_splitk", "mi3d_flash_attn_f16", "mi3d_conv3x3_f16", "mi3d_tf32_tile_test", "mi3d_gemm_f16_bt",
    "mi3d_op_gemm", "mi3d_op_conv3", "mi3d_op_conv3_block", "mi3d_op_attention", "mi3d_op_attention_core", "mi3d_op_layernorm", "mi3d_op_layernorm_bwd",
    "mi3d_op_softmax", "mi3d_op_softmax_bwd", "mi3d_op_transpose",
    "mi3d_engine_destroy", "mi3d_engine_num_params", "mi3d_engine_param_name", "mi3d_engine_param_shape", "mi3d_engine_load_param",
    "mi3d_engine_set_graph_replay", "mi3d_engine_graph_replays", "mi3d_engine_debug_tensor",
    "mi3d_sd_workspace_bytes", "mi3d_sd_create", "mi3d_sd_encode", "mi3d_sd_encode_backward", "mi3d_sd_unet_sds", "mi3d_sd_profile",
    "mi3d_sd_profile_dump", "mi3d_sd_ddim_step", "mi3d_sd_decode", "mi3d_sd_sample",
    "mi3d_sd_text_workspace_bytes", "mi3d_sd_text_create", "mi3d_sd_text_act_workspace_bytes", "mi3d_sd_text_act_create",
    "mi3d_sd_text_encode",
    "mi3d_clip_workspace_bytes", "mi3d_clip_create", "mi3d_clip_encode_image", "mi3d_clip_encode_image_backward", "mi3d_clip_encode_text",
    "mi3d_points_workspace_bytes", "mi3d_points_render_forward", "mi3d_points_render_backward", "mi3d_points_zbuffer_visible",
    "mi3d_cx_workspace_bytes", "mi3d_cx_create", "mi3d_cx_forward", "mi3d_cx_backward",
    "mi3d_unet_workspace_bytes", "mi3d_unet_create", "mi3d_unet_forward", "mi3d_unet_backward",
    "mi3d_dpt_workspace_bytes", "mi3d_dpt_create", "mi3d_dpt_forward", "mi3d_dpt_tap",
    "mi3d_blip2_workspace_bytes", "mi3d_blip2_create", "mi3d_blip2_encode", "mi3d_blip2_generate", "mi3d_blip2_tap",
    "mi3d_stream_gemm_workspace_bytes", "mi3d_stream_gemm_f16",
    "mi3d_mc_workspace_bytes", "mi3d_mc_count", "mi3d_mc_emit", "mi3d_mesh_atlas_texels",
    "mi3d_views_workspace_bytes", "mi3d_views_mask", "mi3d_views_cover_mask", "mi3d_views_backproject", "mi3d_views_compact_colour",
    "mi3d_refine_image_losses_workspace_bytes", "mi3d_refine_image_losses", "mi3d_refine_image_losses_backward",
    "mi3d_refine_adam_workspace_bytes", "mi3d_refine_adam",
    "mi3d_coarse_losses_workspace_bytes", "mi3d_coarse_losses", "mi3d_coarse_losses_backward",
]


def build(verbose=False):
    """Compile libmi3d.so in-tree with nvcc for sm_90a (no GPU needed)."""
    out = subprocess.run(["make", "-C", os.path.join(_HERE, "csrc")], capture_output=True, text=True)
    if out.returncode != 0:
        raise Mi3dError("building libmi3d.so failed:\n" + out.stdout[-4000:] + out.stderr[-4000:])
    if verbose:
        print(out.stdout[-2000:])


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Mi3dError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU / PyTorch fallback for the hot path)")
        _lib = C.CDLL(LIB_PATH)
        for name in SYMBOLS:
            if name.endswith("_workspace_bytes"):
                getattr(_lib, name).restype = C.c_size_t
            elif name.endswith("_create"):
                getattr(_lib, name).restype = C.c_void_p           # mi3d_engine_t
        _lib.mi3d_field_enc_cache_bytes.restype = C.c_size_t
        _lib.mi3d_engine_param_name.restype = C.c_char_p
        _lib.mi3d_version.restype = C.c_char_p
    return _lib


def check(code, what):
    if code != 0:
        if code == 1000001:
            raise Mi3dError(f"{what}: invalid argument (MI3D_ERR_ARG)")
        raise Mi3dError(f"{what}: CUDA error {code}")


def ptr(t):
    """device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise Mi3dError("mi3d kernels need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise Mi3dError("mi3d kernels need contiguous tensors")
    return C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def f32c(t):
    return t.contiguous().float() if (t.dtype != torch.float32 or not t.is_contiguous()) else t


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise Mi3dError("mi3d operators run on sm_90a only; got a CPU tensor and there is no CPU fallback")


class Engine:
    """A planned engine of libmi3d.so (mi3d_<kind>_create): the device workspace it is carved from (zeroed: padding rows and channels
    are never written), its handle, its parameter registry (`names`, `shapes`) and, with graph_replay, the stream its launch lists
    run on so that they can replay as CUDA graphs (torch's legacy default stream cannot be captured; graph_replay=False keeps plain
    launches on the caller's stream).  Subclasses add their configuration struct, their compute calls and their state_dict policy."""

    debug_dtype = torch.float16          # element type of the workspace's intermediates (debug_tensor's default view)

    def __init__(self, kind, cfg_args, device, graph_replay, what):
        """cfg_args: the arguments mi3d_<kind>_workspace_bytes takes (and mi3d_<kind>_create before the workspace); what: the
        configuration, for the error message when the engine cannot run it"""
        lib_ = lib()
        nbytes = getattr(lib_, f"mi3d_{kind}_workspace_bytes")(*cfg_args)
        if nbytes == 0:
            raise Mi3dError(f"unsupported {what}")
        self.nbytes = nbytes
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        h = getattr(lib_, f"mi3d_{kind}_create")(*cfg_args, ptr(self.workspace), C.c_size_t(nbytes))
        if not h:
            raise Mi3dError(f"mi3d_{kind}_create failed (TMA descriptor encoding error)")
        self.h = C.c_void_p(h)
        self.names, self.shapes = [], []
        shp = (C.c_int * 4)()
        for i in range(lib_.mi3d_engine_num_params(self.h)):
            self.names.append(lib_.mi3d_engine_param_name(self.h, C.c_int(i)).decode())
            r = lib_.mi3d_engine_param_shape(self.h, C.c_int(i), shp)
            self.shapes.append(tuple(shp[k] for k in range(r)))
        self.stream = torch.cuda.Stream(device) if graph_replay else None
        check(lib_.mi3d_engine_set_graph_replay(self.h, C.c_int(1 if graph_replay else 0)), f"{kind}: set_graph_replay")

    def graph_replays(self):
        """number of launch lists currently instantiated as CUDA graphs"""
        return int(lib().mi3d_engine_graph_replays(self.h))

    @contextlib.contextmanager
    def on_stream(self):
        """Engine calls inside run on self.stream, ordered after the caller's pending work; the caller's stream then waits for them."""
        if self.stream is None:
            yield
            return
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            yield
        cur.wait_stream(self.stream)

    def partner(self, name, tensors):
        """the second tensor of a pair the engine writes together with entry `name` (None: none)"""
        return None

    def load(self, tensors):
        """tensors: name -> tensor (any float dtype, any device) for every registry entry; an entry 'base#suffix' is a derived copy
        and is written from tensors[base]"""
        lib_ = lib()
        dev = self.workspace.device
        for i, name in enumerate(self.names):
            base = name.split("#")[0]
            if base not in tensors:
                raise Mi3dError(f"missing parameter {base}")
            src = tensors[base].detach().to(dev, torch.float32).contiguous()
            partner = self.partner(name, tensors)
            if partner is not None:
                partner = partner.detach().to(dev, torch.float32).contiguous()
            # the caching allocator reuses src's memory only after the load kernel queued behind it on this stream
            check(lib_.mi3d_engine_load_param(self.h, C.c_int(i), ptr(src), ptr(partner), stream()), f"load_param({name})")
        torch.cuda.synchronize(dev)

    def load_strict(self, state_dict, ignored=lambda key: False):
        """load() after checking that state_dict holds every registry entry with its shape and no other key but those `ignored` accepts"""
        known = set(self.names)
        missing = [n for n in self.names if n not in state_dict]
        unexpected = [k for k in state_dict if k not in known and not ignored(k)]
        if missing or unexpected:
            raise Mi3dError(f"{type(self).__name__} state_dict mismatch: missing {missing[:4]}, unexpected {unexpected[:4]}")
        for name, shape in zip(self.names, self.shapes):
            if tuple(state_dict[name].shape) != shape:
                raise Mi3dError(f"{name}: shape {tuple(state_dict[name].shape)}, expected {shape}")
        self.load(state_dict)
        return self

    def debug_tensor(self, name, dtype=None):
        """a named intermediate, as a view of the workspace"""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib().mi3d_engine_debug_tensor(self.h, name.encode(), C.byref(p), C.byref(n)), f"debug_tensor({name})")
        off = p.value - self.workspace.data_ptr()
        return self.workspace[off:off + n.value].view(dtype or self.debug_dtype)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                lib().mi3d_engine_destroy(self.h)
        except Exception:
            pass
