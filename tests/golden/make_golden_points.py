"""tests/golden/make_golden_points.py -- golden vectors of the refine stage's point renderer and z-buffer from the REFERENCE's own
nerf/refine_utils.py, imported unmodified (needs a checkout of the reference; runs on CPU):
    MI3D_REFERENCE_DIR=<checkout> python tests/golden/make_golden_points.py

What is real reference code: `z_buffer` (and the `project` it calls), and `render_point`'s glue around the two pytorch3d calls:
the torch.matmul projection, the NDC sign flips, the alpha formula and the permutes.  What is substituted, because pytorch3d is not
installed: `Pointclouds`, `rasterize_points` and `compositing.alpha_composite` are stubs over oracle/points_ref.py's primitives;
cv2 / imageio / tqdm are import-only MagicMocks.  The projected cloud the glue hands to `rasterize_points` is recorded too.
"""
import os
import sys
import types
from unittest.mock import MagicMock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import points_ref as pr      # noqa: E402

STATE = {}


def install_stubs():
    for name in ("cv2", "imageio", "tqdm"):
        sys.modules.setdefault(name, MagicMock())

    class Pointclouds:
        def __init__(self, points, features):
            self.points, self.features = points[0], features[0]

        def features_packed(self):
            return self.features

    def rasterize_points(pts, image_size, radius, ppp):
        p = pts.points.detach()
        STATE["ndc"] = p.clone()
        idx, zb, d2 = pr.rasterize_ndc(p[:, 0], p[:, 1], p[:, 2], int(image_size[0]), radius, ppp)
        return idx[None], zb[None], d2[None]

    def alpha_composite(idx, alphas, features):          # idx / alphas [1,K,H,W], features [C,P]; pytorch3d's front-to-back order
        out = torch.zeros(features.shape[0], idx.shape[2], idx.shape[3], dtype=torch.float32)
        T = torch.ones(idx.shape[2], idx.shape[3], dtype=torch.float32)
        for k in range(idx.shape[1]):
            i, a = idx[0, k], alphas[0, k]
            v = i >= 0
            w = T * a
            out = torch.where(v[None], out + w[None] * features[:, i.clamp(min=0)], out)
            T = torch.where(v, T * (1.0 - a), T)
        return out[None]

    p3d = types.ModuleType("pytorch3d")
    structures, renderer, points, compositing = (types.ModuleType(n) for n in
                                                 ("pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.points",
                                                  "pytorch3d.renderer.compositing"))
    structures.Pointclouds = Pointclouds
    points.rasterize_points = rasterize_points
    compositing.alpha_composite = alpha_composite
    renderer.compositing = compositing
    renderer.AlphaCompositor = MagicMock()
    renderer.points = points
    for name, mod in (("pytorch3d", p3d), ("pytorch3d.structures", structures), ("pytorch3d.renderer", renderer),
                      ("pytorch3d.renderer.points", points), ("pytorch3d.renderer.compositing", compositing)):
        sys.modules[name] = mod
    sys.path.insert(0, os.path.join(os.environ["MI3D_REFERENCE_DIR"], "nerf"))
    import refine_utils      # noqa: E402  (REFERENCE module)
    return refine_utils


# render cases: (name, S, views of the surface cloud, its depth-map size, C, radius in pixels, extra behind-camera / off-image points)
RENDER_CASES = [("a", 96, 6, 32, 3, 2.0, 200), ("b", 40, 4, 16, 19, 1.0, 50)]


def render_inputs(S, views, dsize, C, extra, seed):
    rng = np.random.default_rng(seed)
    cloud = pr.surface_cloud(views, dsize, seed=seed)
    wild = (rng.standard_normal((extra, 3)) * 1.5).astype(np.float32)       # many land behind the camera or off the image
    pts = np.concatenate([cloud, wild])
    pts = pts[rng.permutation(pts.shape[0])]
    feats_u8 = rng.integers(0, 256, (pts.shape[0], C), dtype=np.uint8)      # stored as 8-bit codes, see pr.golden_case
    c2w = pr.lookat_c2w(1.2, 70.0, 30.0)
    return pts, feats_u8, pr.intrinsics(S), np.linalg.inv(c2w)


def main():
    ru = install_stubs()
    out = {}
    for n, (name, S, views, dsize, C, rpx, extra) in enumerate(RENDER_CASES):
        pts, feats_u8, K, w2c = render_inputs(S, views, dsize, C, extra, seed=10 + n)
        radius = rpx / S * 2.0
        img = ru.render_point(torch.from_numpy(pts), torch.from_numpy(pr.decode_feats(feats_u8)), S, S, torch.from_numpy(K).float(),
                              torch.from_numpy(w2c).float(), [S, S], radius, 8)
        out.update({f"{name}_points": pts, f"{name}_feats_u8": feats_u8, f"{name}_K": K, f"{name}_w2c": w2c, f"{name}_S": np.int32(S),
                    f"{name}_radius": np.float64(radius), f"{name}_image": img.numpy(), f"{name}_ndc": STATE["ndc"].numpy()})
        print(f"render {name}: {pts.shape[0]} points, {S}x{S}, C={C}, covered pixels {(img.abs().sum(1) > 0).float().mean():.3f}")
    # z_buffer: a depth-map cloud (as depth2point builds it) and random clouds with many points per pixel and off-image points
    S = 48
    K = pr.intrinsics(S)
    c2w = pr.lookat_c2w(1.3, 80.0, 10.0)
    D, m = pr.sphere_depth(c2w, K, S)
    # clouds are stored as float32 values (held in float64, as z_buffer receives them) to keep the fixture small
    cases = {"depth": (pr.depth_cloud(D, m, c2w, K).astype(np.float32).astype(np.float64), np.linalg.inv(c2w), S)}
    rng = np.random.default_rng(3)
    for i, (n, S2) in enumerate(((3000, 24), (5000, 32))):
        c2w2 = pr.lookat_c2w(1.0 + 0.3 * i, 60.0 + 20 * i, 100.0 * i)
        cases[f"rand{i}"] = ((rng.standard_normal((n, 3)) * 0.4).astype(np.float32).astype(np.float64), np.linalg.inv(c2w2), S2)
    for name, (v, w2c, S2) in cases.items():
        K2 = pr.intrinsics(S2)
        mask = ru.z_buffer(v, w2c, S2, S2, K2)
        out.update({f"zb_{name}_v": v.astype(np.float32), f"zb_{name}_w2c": w2c, f"zb_{name}_K": K2, f"zb_{name}_S": np.int32(S2), f"zb_{name}_mask": mask})
        print(f"z_buffer {name}: {v.shape[0]} points, {S2}x{S2}, visible {mask.sum()}")
    np.savez_compressed(os.path.join(HERE, "points_ref.npz"), **out)


if __name__ == "__main__":
    main()
