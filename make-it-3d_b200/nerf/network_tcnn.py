"""B2 seam: the default field of the reference (`--backbone tcnn`, nerf/network_tcnn.py:37-205) on libmi3d.so.

Same constructor, attribute names and state_dict keys as the reference:
    encoder.params                      flat fp32 [12 196 240]  (tcnn.Encoding's single parameter tensor)
    sigma_net.net.{0,1,2}.{weight,bias} MLP(32, 4, 64, 3)
so reference checkpoints load here and vice versa.  forward / density / normal / common_forward run the fused
field kernels (hash-grid gather + MLP + activations + finite-difference normals + shading in one launch).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib as L
from . import field_ops
from .renderer import NeRFRenderer


class HashGridEncoding(nn.Module):
    """tinycudann.Encoding(3, {otype: HashGrid, ...}, dtype=float32) stand-in (nerf/network_tcnn.py:54-65)."""

    def __init__(self, n_input_dims=3, encoding_config=None, dtype=torch.float32, seed=None):
        super().__init__()
        cfg = dict(otype="HashGrid", n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16,
                   per_level_scale=1.3819128274917603)
        cfg.update(encoding_config or {})
        if n_input_dims != 3 or cfg["otype"] != "HashGrid" or cfg["n_features_per_level"] != 2 or dtype != torch.float32:
            raise L.Mi3dError("only the reference's configuration is built: 3-D HashGrid, 2 features/level, fp32")
        self.encoding_config = cfg
        self.hg = field_ops.make_hashgrid(cfg["n_levels"], cfg["base_resolution"], float(cfg["per_level_scale"]),
                                          cfg["log2_hashmap_size"])
        self.n_input_dims = 3
        self.n_output_dims = 2 * cfg["n_levels"]
        g = None
        if seed is not None:
            g = torch.Generator().manual_seed(seed)
        # tcnn initialises grid parameters U(-1e-4, 1e-4)
        self.params = nn.Parameter((torch.rand(self.hg.n_entries * 2, generator=g) * 2 - 1) * 1e-4)

    def forward(self, x):
        return _Encode.apply(x, self.params, self.hg)


class _Encode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, params, hg):
        import ctypes as C
        x = L.f32c(x).view(-1, 3)
        L.require_cuda(x, params)
        E = x.shape[0]
        out = torch.empty(E, 2 * hg.n_levels, dtype=torch.float32, device=x.device)
        L.check(L.lib().mi3d_hashgrid_forward(L.ptr(x), C.c_uint32(E), L.ptr(params), C.byref(hg), L.ptr(out), L.stream()),
                "hashgrid_forward")
        ctx.save_for_backward(x, params)
        ctx.hg = hg
        return out

    @staticmethod
    def backward(ctx, g):
        import ctypes as C
        x, params = ctx.saved_tensors
        g = L.f32c(g)
        gp = torch.zeros_like(params)
        L.check(L.lib().mi3d_hashgrid_backward(L.ptr(x), C.c_uint32(x.shape[0]), L.ptr(g), C.byref(ctx.hg), L.ptr(gp), L.stream()),
                "hashgrid_backward")
        return None, gp, None


class MLP(nn.Module):
    """nerf/network_tcnn.py:13-32 (parameter container; the fused kernels read the weights in place)."""

    def __init__(self, dim_in, dim_out, dim_hidden, num_layers, bias=True):
        super().__init__()
        self.dim_in, self.dim_out, self.dim_hidden, self.num_layers = dim_in, dim_out, dim_hidden, num_layers
        self.net = nn.ModuleList([
            nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=bias)
            for l in range(num_layers)])

    def forward(self, x):
        for l in range(self.num_layers):
            x = self.net[l](x)
            if l != self.num_layers - 1:
                x = F.relu(x, inplace=True)
        return x


class NeRFNetwork(NeRFRenderer):
    def __init__(self, opt, bg_color=None, num_layers=3, hidden_dim=64, num_layers_bg=2, hidden_dim_bg=64):
        super().__init__(opt)
        if num_layers != 3 or hidden_dim != 64:
            raise L.Mi3dError("the fused field kernel is built for the reference's MLP(32,4,64,3)")
        self.num_layers, self.hidden_dim = num_layers, hidden_dim
        per_level_scale = np.exp2(np.log2(2048 * self.bound / 16) / (16 - 1))
        self.encoder = HashGridEncoding(3, {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2,
                                            "log2_hashmap_size": 19, "base_resolution": 16,
                                            "per_level_scale": float(per_level_scale)}, dtype=torch.float32)
        self.sigma_net = MLP(32, 4, hidden_dim, num_layers, bias=True)
        if self.bg_radius > 0:
            raise L.Mi3dError("bg_radius > 0 (background network) is out of scope: main.py:54 fixes it to -1")
        self.bg_net = None

    def set_device(self, device):
        self.encoder.to(device)
        self.sigma_net.to(device)

    # ---- handles for the fused kernels ----
    def _field_handles(self):
        net = self.sigma_net.net
        mlp_params = (net[0].weight, net[0].bias, net[1].weight, net[1].bias, net[2].weight, net[2].bias)
        cfg = dict(bound=float(self.bound), blob_density=float(self.opt.blob_density), blob_radius=float(self.opt.blob_radius),
                   n_evals=7, shading='albedo', ambient_ratio=1.0)
        return self.encoder.params, mlp_params, self.encoder.hg, cfg

    def _eval(self, x, d, l, n_evals, shading, ratio):
        table, mlp_params, hg, cfg = self._field_handles()
        cfg = dict(cfg, n_evals=n_evals, shading=shading, ambient_ratio=float(ratio))
        x = L.f32c(x).view(-1, 3)
        return field_ops.field_eval(table, mlp_params, x, d, l, hg, cfg)

    def gaussian(self, x):                                    # network_tcnn.py:94-100
        d = (x ** 2).sum(-1)
        return self.opt.blob_density * torch.exp(-d / (2 * self.opt.blob_radius ** 2))

    def common_forward(self, x):                              # :102-112
        sigma, albedo, _, _, _ = self._eval(x, None, None, 1, 'albedo', 1.0)
        return sigma, albedo

    def normal(self, x):                                      # :115-138
        _, _, normal, _, _ = self._eval(x, None, None, 7, 'albedo', 1.0)
        return normal

    def forward(self, x, d, l=None, ratio=1, shading='albedo'):   # :140-170
        if shading != 'albedo' and l is None:
            raise L.Mi3dError("light direction `l` is required for lit shading")
        sigma, color, normal, _, _ = self._eval(x, L.f32c(d).view(-1, 3) if d is not None else None,
                                                L.f32c(l) if l is not None else None, 7, shading, ratio)
        return sigma, color, normal

    def density(self, x):                                     # :173-180
        sigma, albedo = self.common_forward(x)
        return {'sigma': sigma, 'albedo': albedo}

    def get_params(self, lr):                                 # :195-206
        return [{'params': self.encoder.parameters(), 'lr': lr * 10},
                {'params': self.sigma_net.parameters(), 'lr': lr}]
