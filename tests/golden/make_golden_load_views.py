"""tests/golden/make_golden_load_views.py -- golden vectors of the refine stage's point-cloud construction from the REFERENCE's own
nerf/refine_utils.py (load_views, depth2point, multidepth2point_mask), imported unmodified and run on CPU with the real cv2 (needs a
checkout of the reference):
    MI3D_REFERENCE_DIR=<checkout> python tests/golden/make_golden_load_views.py

Substituted: pytorch3d is stubbed over oracle/points_ref.py's primitives exactly as tests/golden/make_golden_points.py does; imageio
is a cv2-backed shim that reads and writes RGB order; tqdm.tqdm is an identity wrapper.  cv2 is wrapped only to record what erode,
Canny and dilate return, in call order.

Recorded per case (5 views at 64^2 and 9 views at 96^2, synthetic folders written by oracle/views_ref.make_mvimg):
- inputs: the decoded uint16 depths, uint8 masks and RGB images, float32 poses, K, gt_rgb as uint8 codes (gt_rgb = code / 255.);
- intermediates: the canonical mask, each other view's eroded mask, Canny and dilated edges, the canonical-cloud mask PNG (channel 0)
  read back by multidepth2point_mask and its final mask;
- the four outputs of load_views, and multidepth2point_mask with npoint = half its output under np.random.seed(7);
- cv2 erode / dilate / Canny of extra random images.
"""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import cv2                                      # noqa: E402
import make_golden_points as mgp                # noqa: E402
from oracle import views_ref as vr              # noqa: E402

CALLS = []
WRITES = {}


def install():
    rec = types.ModuleType("cv2")
    rec.__dict__.update({k: getattr(cv2, k) for k in dir(cv2) if not k.startswith("__")})

    def recorded(name):
        fn = getattr(cv2, name)

        def call(*a, **kw):
            out = fn(*a, **kw)
            CALLS.append((name, out.copy()))
            return out
        return call
    for name in ("erode", "dilate", "Canny"):
        setattr(rec, name, recorded(name))
    sys.modules["cv2"] = rec

    iio = types.ModuleType("imageio")

    def imread(path):
        im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        return im[..., ::-1] if im.ndim == 3 else im

    def imwrite(path, im):
        WRITES[os.path.basename(path)] = np.array(im)
        cv2.imwrite(path, im[..., ::-1] if im.ndim == 3 else im)
    iio.imread, iio.imwrite = imread, imwrite
    sys.modules["imageio"] = iio
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, *a, **kw: it
    sys.modules["tqdm"] = tq
    return mgp.install_stubs()


def run_case(ru, name, n_views, S, seed, out):
    with tempfile.TemporaryDirectory() as tmp:
        mv = os.path.join(tmp, "mvimg")
        gt, rgb_f, depth_f, mask_f, poses, K = vr.make_mvimg(mv, n_views, S, seed)
        outdir = os.path.join(tmp, "refine")
        os.makedirs(outdir)
        seen = {}
        orig = ru.multidepth2point_mask

        def spy(*a, **kw):
            seen["args"] = a
            return orig(*a, **kw)
        ru.multidepth2point_mask = spy
        CALLS.clear()
        WRITES.clear()
        vc, cc, vn, cn = ru.load_views(gt, rgb_f, depth_f, mask_f, poses, S, S, K, 2, 8, outdir, "cpu")
        ru.multidepth2point_mask = orig
        assert os.listdir(outdir) == []
        ind = (n_views - 1) // 2
        names = [c[0] for c in CALLS]
        # order: canonical erode / Canny / dilate, then (erode, Canny, dilate) per other view, then one 15x15 erode per other view
        assert names[:3] == ["erode", "Canny", "dilate"] and len(names) == 3 + 4 * (n_views - 1), names
        views = CALLS[3:3 + 3 * (n_views - 1)]
        a = seen["args"]
        np.random.seed(7)
        npoint = max(1, len(vn) // 2)
        vs, cs = orig(*a, npoint=npoint)
        # the final per-view mask is not returned by the reference; recompute it from the recorded intermediates as lines 84-85 do
        masks = []
        for j in range(n_views - 1):
            e15 = CALLS[3 + 3 * (n_views - 1) + j][1]
            cov = np.logical_or(np.logical_or(e15[:, :, 0] > 0.9, e15[:, :, 1] > 0.9), e15[:, :, 2] > 0.9)
            masks.append(np.logical_and(a[1][j], ~cov))
        dec = lambda f, fl: cv2.imread(f, fl)
        out.update({
            f"{name}_depth": np.stack([dec(f, cv2.IMREAD_UNCHANGED) for f in depth_f]),
            f"{name}_mask": np.stack([dec(f, cv2.IMREAD_UNCHANGED) for f in mask_f]),
            f"{name}_rgb": np.stack([dec(f, cv2.IMREAD_UNCHANGED)[..., ::-1] for f in rgb_f]),
            f"{name}_poses": poses, f"{name}_K": K, f"{name}_gt_u8": np.round(gt * 255).astype(np.uint8),
            f"{name}_cano_mask": CALLS[0][1] == 1,
            f"{name}_eroded": np.stack([views[3 * j][1] == 1 for j in range(n_views - 1)]),
            f"{name}_canny": np.stack([views[3 * j + 1][1] for j in range(n_views - 1)]),
            f"{name}_dilated": np.stack([views[3 * j + 2][1] for j in range(n_views - 1)]),
            f"{name}_quant": np.stack([WRITES[f"render_{j}_mask.png"][..., 0] for j in range(n_views - 1)]),
            f"{name}_final_mask": np.stack(masks),
            f"{name}_v_cano": vc, f"{name}_c_cano": cc, f"{name}_v_novel": vn, f"{name}_c_novel": cn,
            f"{name}_sub_npoint": np.int64(npoint), f"{name}_sub_v": vs, f"{name}_sub_c": cs,
        })
        assert np.array_equal(out[f"{name}_gt_u8"] / 255., gt)
        print(f"{name}: {n_views} views at {S}^2: cano {len(vc)} points, novel {len(vn)}, "
              f"canny px {int((out[f'{name}_canny'] > 0).sum())}")


def main():
    ru = install()
    out = {}
    for name, n, S, seed in (("a", 5, 64, 1), ("b", 9, 96, 2)):
        run_case(ru, name, n, S, seed, out)
    # erode / dilate / Canny of random blob images against the real cv2
    rng = np.random.default_rng(5)
    imgs = []
    for h, w in ((40, 56), (64, 64), (33, 47)):
        im = rng.integers(0, 256, (h // 4 + 1, w // 4 + 1)).astype(np.uint8)
        im = cv2.resize(im, (w, h), interpolation=cv2.INTER_LINEAR)
        im[rng.random((h, w)) < 0.05] = rng.integers(0, 256)
        imgs.append(im)
    for j, im in enumerate(imgs):
        out[f"rand{j}_img"] = im
        for k in (3, 11, 15):
            out[f"rand{j}_erode{k}"] = cv2.erode(im, np.ones((k, k), np.uint8))
            out[f"rand{j}_dilate{k}"] = cv2.dilate(im, np.ones((k, k), np.uint8))
        out[f"rand{j}_erode11x2"] = cv2.erode(im, np.ones((11, 11), np.uint8), iterations=2)
        for t in (10, 30):
            out[f"rand{j}_canny{t}"] = cv2.Canny(im, t, t)
    np.savez_compressed(os.path.join(HERE, "load_views_ref.npz"), **out)


if __name__ == "__main__":
    main()
