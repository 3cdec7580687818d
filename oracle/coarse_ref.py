"""fp64 restatement of the coarse loop's losses (nerf/utils.py:491-493, :519-533, :551-556) that csrc/coarse.cu fuses: the
align_corners=True bilinear upsample to 512^2 and its adjoint, the gt composite, the L1 term, torchmetrics' Pearson coefficient on
nan_to_num(up(depth)) over a mask, and the opacity / entropy regularisers, with their gradients.  numpy only;
tests/test_coarse_oracle_cpu.py holds it against torch CPU autograd, tests/test_coarse_gpu.py holds the kernels against it."""
import numpy as np

OUT = 512


def taps(n, dtype=np.float32, out=OUT):
    """torch's upsample_bilinear2d (align_corners=True) taps of every output index for an input of size n, with the source index
    computed in `dtype` as torch does: (i0, i1, l0, l1), the weights as fp64"""
    dt = np.dtype(dtype).type
    scale = dt(n - 1) / dt(out - 1)
    src = (scale * np.arange(out).astype(dt)).astype(dt)
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n - 1)
    l1 = (src - i0.astype(dt)).astype(dt)
    l0 = (dt(1) - l1).astype(dt)
    return i0, i1, l0.astype(np.float64), l1.astype(np.float64)


def upsample(x, dtype=None):
    """[..., h, w] -> [..., 512, 512] in fp64 (a non-finite input poisons every output whose stencil holds it, as in torch)"""
    x = np.asarray(x)
    dtype = dtype or (x.dtype if x.dtype in (np.float32, np.float64) else np.float32)
    y0, y1, a0, a1 = taps(x.shape[-2], dtype)
    x0, x1, b0, b1 = taps(x.shape[-1], dtype)
    x = x.astype(np.float64)
    r0, r1 = x[..., y0, :], x[..., y1, :]
    top = b0 * r0[..., x0] + b1 * r0[..., x1]
    bot = b0 * r1[..., x0] + b1 * r1[..., x1]
    return a0[:, None] * top + a1[:, None] * bot


def _matrix(n, dtype):
    i0, i1, l0, l1 = taps(n, dtype)
    m = np.zeros((OUT, n))
    np.add.at(m, (np.arange(OUT), i0), l0)
    np.add.at(m, (np.arange(OUT), i1), l1)
    return m


def upsample_adjoint(g, h, w, dtype=np.float32):
    """the adjoint of `upsample`: [..., 512, 512] -> [..., h, w]"""
    return _matrix(h, dtype).T @ np.asarray(g, np.float64) @ _matrix(w, dtype)


def gt_composite(ref, bg):
    """ref[:3] alpha + bg (1 - alpha) in fp32 (utils.py:491-493): ref [1,4,512,512], bg [3] -> [1,3,512,512]"""
    ref, bg = np.asarray(ref, np.float32), np.asarray(bg, np.float32)
    a = ref[:, 3:]
    return ref[:, :3] * a + bg.reshape(1, 3, 1, 1) * (np.float32(1) - a)


def nan_to_num(x, dtype=np.float32):
    """torch.nan_to_num in `dtype`: NaN -> 0, +-inf -> +-the largest finite value"""
    big = float(np.finfo(dtype).max)
    x = np.asarray(x, np.float64)
    return np.where(np.isnan(x), 0.0, np.where(np.isposinf(x), big, np.where(np.isneginf(x), -big, x)))


def l1(pred, gt):
    """mean |pred - gt| and its gradient"""
    d = np.asarray(pred, np.float64) - np.asarray(gt, np.float64)
    return float(np.abs(d).mean()), np.sign(d) / d.size


def pearson(x, y, mask):
    """torchmetrics' PearsonCorrCoef on x[mask], y[mask] (two-pass, fp64): clamp(cov / sqrt(var_x var_y), -1, 1) and its gradient
    w.r.t. x.  Fewer than 2 pixels give NaN, and a coefficient outside [-1, 1] (or NaN) passes no gradient (clamp backward)."""
    x, y, m = np.asarray(x, np.float64).ravel(), np.asarray(y, np.float64).ravel(), np.asarray(mask).ravel() != 0
    xs, ys = x[m], y[m]
    n = float(xs.size)
    with np.errstate(invalid="ignore", divide="ignore"):
        mx, my = xs.sum() / n, ys.sum() / n
        dx, dy = xs - mx, ys - my
        sxx, syy, sxy = (dx * dx).sum(), (dy * dy).sum(), (dx * dy).sum()
        r = (sxy / (n - 1)) / np.sqrt((sxx / (n - 1)) * (syy / (n - 1)))
    grad = np.zeros_like(x)
    if -1.0 <= r <= 1.0:
        grad[m] = dy / np.sqrt(sxx * syy) - r * dx / sxx
    rc = r if np.isnan(r) else min(max(r, -1.0), 1.0)
    return float(rc), grad


def opacity(ws):
    """mean(ws^2) and its gradient"""
    ws = np.asarray(ws, np.float64)
    return float((ws * ws).mean()), 2.0 * ws / ws.size


def entropy(ws, dtype=np.float32):
    """mean(-a log2 a - (1-a) log2(1-a)), a = clamp(ws, 1e-5, 1 - 1e-5) with the bounds in `dtype`, and its gradient (inclusive
    at the bounds)"""
    lo, hi = float(np.asarray(1e-5, dtype)), float(np.asarray(1 - 1e-5, dtype))
    ws = np.asarray(ws, np.float64)
    a = np.clip(ws, lo, hi)
    e = -a * np.log2(a) - (1 - a) * np.log2(1 - a)
    inside = (ws >= lo) & (ws <= hi)
    return float(e.mean()), np.where(inside, np.log2(1 - a) - np.log2(a), 0.0) / ws.size


def forward(image, depth, ws, h, w, ref, bg, prior, mask, front, dtype=np.float32):
    """terms (opacity, entropy, l1, pearson), pred512, gt512 of csrc/coarse.cu for image [h*w,3], depth / ws [h*w]"""
    img = np.asarray(image).reshape(h, w, 3).transpose(2, 0, 1)[None]
    pred = upsample(img, dtype)
    gt = gt_composite(ref, bg).astype(np.float64)
    op, _ = opacity(ws)
    en, _ = entropy(ws, dtype)
    terms = [op, en, 0.0, 0.0]
    if front:
        terms[2] = l1(pred, gt)[0]
        x = nan_to_num(upsample(np.asarray(depth).reshape(h, w), dtype), dtype)
        terms[3] = pearson(x, prior, mask)[0]
    return np.array(terms), pred, gt


def backward(image, depth, ws, h, w, ref, bg, prior, mask, front, g_terms, g_pred512=None, dtype=np.float32):
    """(d image [h*w,3], d depth [h*w], d ws [h*w]) of g_terms . terms + <g_pred512, pred512>"""
    g_terms = np.asarray(g_terms, np.float64)
    _, pred, gt = forward(image, depth, ws, h, w, ref, bg, prior, mask, False, dtype)
    gp = np.zeros((1, 3, OUT, OUT)) if g_pred512 is None else np.asarray(g_pred512, np.float64).reshape(1, 3, OUT, OUT).copy()
    gd = np.zeros((h, w))
    if front:
        gp += g_terms[2] * l1(pred, gt)[1]
        raw = upsample(np.asarray(depth).reshape(h, w), dtype)
        _, gx = pearson(nan_to_num(raw, dtype), prior, mask)
        gx = np.where(np.isfinite(raw.ravel()), gx, 0.0).reshape(OUT, OUT)
        gd = upsample_adjoint(g_terms[3] * gx, h, w, dtype)
    gi = upsample_adjoint(gp[0], h, w, dtype)
    g_ws = g_terms[0] * opacity(ws)[1] + g_terms[1] * entropy(ws, dtype)[1]
    return gi.transpose(1, 2, 0).reshape(h * w, 3), gd.reshape(h * w), np.asarray(g_ws).reshape(h * w)
