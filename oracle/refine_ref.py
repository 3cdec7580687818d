"""fp64 restatement of the refine loop's glue (nerf/utils.py:865-894) that csrc/refine.cu fuses: the unit-colour coverage, its 5x5 max
dilation, the background loss, the front iteration's masked L1, the colour regularisers and torch.optim.Adam's update.  numpy only;
tests/test_refine_oracle_cpu.py holds it against torch's own CPU modules, tests/test_refine_gpu.py holds the kernels against it."""
import numpy as np


def coverage(weights):
    """[S,S,ppp] composite weights -> [S,S]: the image render_point makes with unit colours"""
    return np.asarray(weights, np.float64).sum(-1)


def dilate(cov, k=5):
    """MaxPool2d(k, stride 1, padding k // 2) of [S,S] (padding never wins: -inf)"""
    cov = np.asarray(cov, np.float64)
    p = k // 2
    pad = np.full((cov.shape[0] + 2 * p, cov.shape[1] + 2 * p), -np.inf)
    pad[p:-p, p:-p] = cov
    out = np.full(cov.shape, -np.inf)
    for dy in range(k):
        for dx in range(k):
            out = np.maximum(out, pad[dy:dy + cov.shape[0], dx:dx + cov.shape[1]])
    return out


def bg_loss(pred, dil):
    """1e-3 * sum(1 - pred * (1 - dilate)) over [1,3,S,S] and its gradient"""
    pred = np.asarray(pred, np.float64)
    keep = 1.0 - np.asarray(dil, np.float64)[None, None]
    return 1e-3 * float((1.0 - pred * keep).sum()), np.broadcast_to(-1e-3 * keep, pred.shape).copy()


def masked_l1(pred, gt, mask):
    """1000 * L1Loss()(pred * m, gt * m) (mean over [1,3,S,S]) and its gradient w.r.t. pred"""
    pred, gt, mask = (np.asarray(a, np.float64) for a in (pred, gt, mask))
    d = pred * mask - gt * mask
    n = d.size
    return 1000.0 * float(np.abs(d).sum()) / n, 1000.0 / n * np.sign(d) * mask


def regulariser(colour_cano, origin_cano, colour_novel, origin_novel, w_cano=1e5, w_novel=1e3):
    """w_novel MSE(colour_novel, origin_novel) + w_cano MSE(colour_cano, origin_cano) and the two gradients"""
    dc = np.asarray(colour_cano, np.float64) - np.asarray(origin_cano, np.float64)
    dn = np.asarray(colour_novel, np.float64) - np.asarray(origin_novel, np.float64)
    val = w_novel * float((dn * dn).mean()) + w_cano * float((dc * dc).mean())
    return val, 2.0 * w_cano * dc / dc.size, 2.0 * w_novel * dn / dn.size


def adam_step(param, grad, exp_avg, exp_avg_sq, step, lr=1e-3, betas=(0.9, 0.99), eps=1e-15):
    """one torch.optim.Adam update (no weight decay, no amsgrad); step counts from 1.  Returns (param, exp_avg, exp_avg_sq)."""
    b1, b2 = betas
    g = np.asarray(grad, np.float64)
    m = np.asarray(exp_avg, np.float64) + (1.0 - b1) * (g - exp_avg)
    v = np.asarray(exp_avg_sq, np.float64) * b2 + (1.0 - b2) * g * g
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    denom = np.sqrt(v) / np.sqrt(bc2) + eps
    return np.asarray(param, np.float64) - (lr / bc1) * m / denom, m, v
