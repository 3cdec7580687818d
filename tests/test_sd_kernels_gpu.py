"""GPU: the kernels the SD engine adds on top of the op layer (sd_kernels.cuh, Builder::conv3_s2 / conv_small_cin / conv_small_cout and
the per-view latent kernels of sd_engine.cu), one at a time with the launch geometry the engine plans (mi3d_op_* entry points), against
torch float64 computed from exactly the fp16 / fp32 values the kernel reads.

As in test_op_layer_gpu.py: every comparison is element-wise, |got - ref| <= bound, with the bound derived per element from the
kernel's arithmetic (u = 2^-24 per fp32 rounding, one fp16 output rounding); the worst err / bound of every case is printed; every
output lies in a sentinel-filled buffer whose remainder must stay untouched.
"""
import ctypes as C
import importlib
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_op_layer_gpu import U32, Canvas, acc_bound, check, conv_ref, f16_round, ln_lane_terms, rnd  # noqa: E402

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
EXP_ULP = 2.0 ** -21          # __expf (ex2.approx): ~2^-22 relative, + the rounding of its argument (added per use)
FLT_MAX = 3.4028234663852886e38


@pytest.fixture(scope="module")
def L():
    return importlib.import_module("make-it-3d_b200._lib")


def sync_check(L, code, what):
    L.check(code, what)
    torch.cuda.synchronize()


def silu(x):
    return x * torch.sigmoid(x)


def silu_grad(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def silu_ulps(v):
    """x / (1 + __expf(-x)): the exp's relative error (and that of its argument) moves s by (1 - s) of it; three fp32 roundings"""
    return silu(v).abs() * (EXP_ULP + 2 * U32 * v.abs() + 3 * U32)


# ------------------------------------------------------------------------------------------------------------------------------
# GroupNorm (+ SiLU): sdk::k_gn_stats / k_gn_apply / k_gn_bwd_stats / k_gn_bwd_apply
# ------------------------------------------------------------------------------------------------------------------------------
GN_ADVERSARIAL = 12           # the first groups of image 0


def gn_input(g, N, HW, C, G):
    """x [N][HW][C] fp16.  Image 0's first GN_ADVERSARIAL groups as test_op_layer_gpu.ln_rows builds its rows: constant groups (var = 0)
    and groups with |mean| / std about 10, 100 and 1000 at means 1, -16 and 1000; every other group random."""
    x = torch.randn(N, HW, C, device="cuda", generator=g) * 2 + 0.5
    cpg = C // G
    k = 0
    for val in (0.0, 3.140625, -1000.0):
        x[0, :, k * cpg:(k + 1) * cpg] = val; k += 1
    for ratio in (10, 100, 1000):
        for mu in (1.0, -16.0, 1000.0):
            x[0, :, k * cpg:(k + 1) * cpg] = mu + (abs(mu) / ratio) * torch.randn(HW, cpg, device="cuda", generator=g); k += 1
    assert k == GN_ADVERSARIAL
    return x.half()


def gn_stats(x, G, eps, geom):
    """fp64 group statistics of x [N][HW][C] and the bounds of the kernel's, for the planned geometry (chunks, ppc, PL):
    each thread sums n = ceil(ppc / PL) terms d = x - k of one channel in fp32 (k: the channel's value at pixel 0), sum d with
    (n + 1) u sum|d| error, sum d^2 (fmaf) with (n + 3) u sum d^2; the fp64 rebuild and the fold over channels, lanes and CTAs
    add (cpg + PL + chunks + 8) 2^-53 of the magnitudes.  var = E[x^2] - mean^2 in fp64: an error delta_c of channel c's sum d
    moves it by 2 (k_c - mean) delta_c / cnt (the shift cancels to first order), the sum of d^2 by its own error / cnt.
    Returns mean, var, r = 1/sqrt(var + eps), the sums, their bounds, and the kernel's mean error e_mu (fp32 mean) and relative rstd
    error rho (half the relative var error, + the fp32 rounding of var + eps and rsqrtf's 2 ulp)."""
    N, HW, Cc = x.shape
    cpg = Cc // G
    chunks, ppc, PL = geom
    n = (ppc + PL - 1) // PL
    X = x.double().view(N, HW, G, cpg)
    cnt = HW * cpg
    s1 = X.sum((1, 3))
    s2 = (X * X).sum((1, 3))
    mu = s1 / cnt
    var = ((X - mu[:, None, :, None]) ** 2).sum((1, 3)) / cnt
    k = X[:, :1]
    d = X - k
    e1c = (n + 1) * U32 * d.abs().sum(1)                                    # [N, G, cpg]
    fold = (cpg + PL + chunks + 8) * U64
    e_s1 = e1c.sum(-1) + fold * X.abs().sum((1, 3))
    e_s2 = (n + 3) * U32 * (d * d).sum((1, 3)) + 2 * (k[:, 0].abs() * e1c).sum(-1) + fold * s2
    e_m = e_s1 / cnt
    e_var = ((n + 3) * U32 * (d * d).sum((1, 3)) + 2 * ((k[:, 0] - mu[..., None]).abs() * e1c).sum(-1)) / cnt + e_m ** 2 \
        + 2 * fold * s2 / cnt
    r = 1.0 / torch.sqrt(var + eps)
    e_mu = e_m + U32 * mu.abs()
    rho = 0.51 * e_var / (var + eps) + 2.0 ** -21
    return mu, var, r, (s1, s2), (e_s1, e_s2), e_mu, rho


def run_gn(L, x, G, eps, do_silu, g):
    N, HW, Cc = x.shape
    gamma = torch.rand(Cc, device="cuda", generator=g) + 0.5
    beta = torch.rand(Cc, device="cuda", generator=g) * 0.6 - 0.3
    stats = torch.zeros(N, G, 2, dtype=torch.float64, device="cuda")
    cv = Canvas(N * HW * Cc)
    y = cv.view((N, HW, Cc), (HW * Cc, Cc, 1))
    geom = (C.c_int * 3)()
    sync_check(L, L.lib().mi3d_op_groupnorm(L.ptr(x), L.ptr(y), L.ptr(stats), L.ptr(gamma), L.ptr(beta), N, HW, Cc, G, C.c_float(eps),
                                            int(do_silu), geom, L.stream()), "op_groupnorm")
    return gamma, beta, stats, cv, y, (geom[0], geom[1], geom[2])


def gn_expand(t, HW, cpg):
    """[N][G] -> [N][HW][C]"""
    return t[:, None, :].repeat_interleave(cpg, -1).expand(-1, HW, -1)


# (C, HW, eps, N): the GroupNorms the SD-2 / SD-1.5 U-Net plans at 64^2 latents (N = 2 per view pair, 16 at eight views), the VAE
# encoder and decoder at 512^2 (one image per encode), and the tiny configs of the engine tests (cpg 2 and 4).  cpg = C / 32: 10, 20,
# 30 (an 8-channel vector straddles two groups), 40, 60, 80, 4, 8, 16; C = 2560, 1920: VPP > 256 (PL = 1); C = 320: PL = 6 (256 % VPP
# != 0); HW = 64 and 256 are not multiples of PL * 8 chunks at C = 320 / 960, 512^2 splits into uneven chunks.
GN_CASES = [
    (320, 4096, 1e-5, 2), (320, 4096, 1e-6, 16), (640, 4096, 1e-5, 2), (960, 4096, 1e-5, 2), (960, 4096, 1e-5, 16),
    (320, 1024, 1e-5, 2), (640, 1024, 1e-6, 2), (960, 1024, 1e-5, 2), (1280, 1024, 1e-5, 2), (1920, 1024, 1e-5, 16),
    (640, 256, 1e-5, 2), (1280, 256, 1e-6, 2), (1920, 256, 1e-5, 2), (2560, 256, 1e-5, 2), (2560, 256, 1e-5, 16),
    (1280, 64, 1e-5, 2), (1280, 64, 1e-6, 16), (2560, 64, 1e-5, 2),
    (128, 512 * 512, 1e-6, 1), (128, 256 * 256, 1e-6, 1), (256, 256 * 256, 1e-6, 1), (256, 128 * 128, 1e-6, 1),
    (512, 128 * 128, 1e-6, 1), (512, 64 * 64, 1e-6, 1), (512, 64 * 64, 1e-6, 8), (512, 256 * 256, 1e-6, 1), (256, 512 * 512, 1e-6, 1),
    (64, 1024, 1e-5, 2), (128, 256, 1e-6, 6), (64, 256 * 256, 1e-6, 1), (128, 32 * 32, 1e-6, 3),
]


@pytest.mark.parametrize("Cc,HW,eps,N", GN_CASES)
@pytest.mark.parametrize("do_silu", [False, True])
def test_groupnorm_forward_matches_fp64(L, Cc, HW, eps, N, do_silu):
    """mi3d_op_groupnorm (G = 32) with the engine's geometry.  The stats buffer against the fp64 sums (bounds of gn_stats).
    y: v = x a + b with a = r gamma and b = beta - mean a in fp32: |gamma| r (e_mu + |x - mean| (rho + 2u)) + 3 u (|beta| + |mean gamma r|
    + |x gamma r|); SiLU carries it by max|silu'| = 1.1 and adds its __expf ulps; + one fp16 rounding.  The adversarial groups are held
    to the same bound, that of a two-pass variance (rho scales with the group's spread, not with its mean)."""
    G = 32
    g = torch.Generator(device="cuda").manual_seed(Cc * 7 + HW + N + int(do_silu))
    x = gn_input(g, N, HW, Cc, G)
    gamma, beta, stats, cv, y, geom = run_gn(L, x, G, eps, do_silu, g)
    print(f"geometry (chunks, ppc, PL) = {geom}")
    mu, var, r, sums, e_sums, e_mu, rho = gn_stats(x, G, eps, geom)
    what = f"groupnorm C{Cc} HW{HW} N{N} eps{eps} silu{int(do_silu)}"
    check(what + " stats sum", stats[..., 0], sums[0], e_sums[0] + 1e-300)
    check(what + " stats sum of squares", stats[..., 1], sums[1], e_sums[1] + 1e-300)
    cpg = Cc // G
    X = x.double()
    M, R, EM, RHO = (gn_expand(t, HW, cpg) for t in (mu, r, e_mu, rho))
    Gm, Bt = gamma.double(), beta.double()
    core = (X - M) * R * Gm
    pre = core + Bt
    e = 1.01 * Gm.abs() * R * (EM + (X - M).abs() * (RHO + 2 * U32)) + 3 * U32 * (Bt.abs() + (M * Gm * R).abs() + (X * Gm * R).abs())
    if do_silu:
        ref, e = silu(pre), 1.1 * e + silu_ulps(pre)
    else:
        ref = pre
    bound = f16_round(ref, e)
    check(what + " adversarial groups", y[0, :, :GN_ADVERSARIAL * cpg], ref[0, :, :GN_ADVERSARIAL * cpg], bound[0, :, :GN_ADVERSARIAL * cpg])
    check(what, y, ref, bound)
    cv.check_untouched("groupnorm")


GN_BWD_CASES = [c for i, c in enumerate(GN_CASES) if i % 2 == 0 or c[0] in (128, 256, 512)]


@pytest.mark.parametrize("Cc,HW,eps,N", GN_BWD_CASES)
@pytest.mark.parametrize("do_silu,add", [(True, False), (True, True), (False, True), (False, False)])
def test_groupnorm_backward_matches_fp64(L, Cc, HW, eps, N, do_silu, add):
    """mi3d_op_groupnorm_bwd after the forward (its stats): dg = dy silu'(z) gamma (z = xhat gamma + beta; dg = dy gamma without SiLU),
    dx = r (dg - mean(dg) - xhat mean(dg xhat)) (+ add).  Bound: the forward's xhat error e_xh = r e_mu + |xhat| (rho + 2u) carried
    through silu' (|silu''| <= 0.5, and its __expf ulps), the fp32 group means of dg and dg xhat ((n + 8) u of their magnitudes, n
    the per-thread terms), 3 u of the formula's terms, rho of r, u |add| and one fp16 rounding.  The bstats buffer against fp64."""
    G = 32
    g = torch.Generator(device="cuda").manual_seed(Cc * 5 + HW + N + 2 * int(do_silu) + int(add))
    x = gn_input(g, N, HW, Cc, G)
    gamma, beta, stats, _, _, geom = run_gn(L, x, G, eps, do_silu, g)
    dy = rnd(g, N, HW, Cc)
    ad = rnd(g, N, HW, Cc) if add else None
    bstats = torch.zeros(N, G, 2, dtype=torch.float64, device="cuda")
    cv = Canvas(N * HW * Cc)
    dx = cv.view((N, HW, Cc), (HW * Cc, Cc, 1))
    geom2 = (C.c_int * 3)()
    sync_check(L, L.lib().mi3d_op_groupnorm_bwd(L.ptr(x), L.ptr(dy), L.ptr(stats), L.ptr(bstats), L.ptr(gamma), L.ptr(beta), L.ptr(ad),
                                                L.ptr(dx), N, HW, Cc, G, C.c_float(eps), int(do_silu), geom2, L.stream()), "op_groupnorm_bwd")
    assert tuple(geom2) == geom
    mu, var, r, _, _, e_mu, rho = gn_stats(x, G, eps, geom)
    n = (geom[1] + geom[2] - 1) // geom[2]
    cpg = Cc // G
    cnt = HW * cpg
    X = x.double()
    M, R, EM, RHO = (gn_expand(t, HW, cpg) for t in (mu, r, e_mu, rho))
    Gm, Bt = gamma.double(), beta.double()
    xh = (X - M) * R
    e_xh = R * EM + xh.abs() * (RHO + 2 * U32)
    D = dy.double()
    if do_silu:
        z = xh * Gm + Bt
        sg = silu_grad(z)
        dg = D * sg * Gm
        e_sg = 0.5 * Gm.abs() * e_xh + sg.abs() * (EXP_ULP + 2 * U32 * z.abs()) + (1 + z.abs()) * (EXP_ULP + 2 * U32 * z.abs()) * 0.25 \
            + 6 * U32 * (1 + z.abs())
        e_dg = (D * Gm).abs() * e_sg + 2 * U32 * dg.abs()
    else:
        dg = D * Gm
        e_dg = U32 * dg.abs()

    def gsum(t):                                          # [N][HW][C] -> per-group sums, expanded back
        return gn_expand(t.view(N, HW, G, cpg).sum((1, 3)), HW, cpg)
    m1, m2 = gsum(dg) / cnt, gsum(dg * xh) / cnt
    e_m1 = gsum(e_dg) / cnt + (n + 8) * U32 * gsum(dg.abs()) / cnt
    e_m2 = gsum(e_dg * xh.abs() + dg.abs() * e_xh) / cnt + (n + 8) * U32 * gsum((dg * xh).abs()) / cnt
    h = dg - m1 - xh * m2
    e_h = e_dg + e_m1 + xh.abs() * e_m2 + m2.abs() * e_xh + 3 * U32 * (dg.abs() + m1.abs() + (xh * m2).abs())
    ref = R * h + (ad.double() if add else 0.0)
    err = 1.01 * ((R * h).abs() * RHO + R * e_h) + U32 * ((R * h).abs() + (ad.double().abs() if add else 0.0))
    bound = f16_round(ref, err)
    what = f"groupnorm_bwd C{Cc} HW{HW} N{N} silu{int(do_silu)} add{int(add)}"
    b1 = (m1 * cnt)[:, 0, ::cpg]
    b2 = (m2 * cnt)[:, 0, ::cpg]
    check(what + " bstats sum dg", bstats[..., 0], b1, (e_m1 * cnt)[:, 0, ::cpg] + 1e-300)
    check(what + " bstats sum dg xhat", bstats[..., 1], b2, (e_m2 * cnt)[:, 0, ::cpg] + 1e-300)
    check(what + " adversarial groups", dx[0, :, :GN_ADVERSARIAL * cpg], ref[0, :, :GN_ADVERSARIAL * cpg], bound[0, :, :GN_ADVERSARIAL * cpg])
    check(what, dx, ref, bound)
    cv.check_untouched("groupnorm_bwd")


# ------------------------------------------------------------------------------------------------------------------------------
# Builder::conv3_s2 (k_im2col_s2 + tile GEMM) and its input gradient's k_col2im_s2
# ------------------------------------------------------------------------------------------------------------------------------
def conv_s2_ref(x, w, pad_lo):
    """fp64 3x3 stride-2 conv of NHWC x: pad_lo 1 = padding 1 on every side, 0 = padding (0, 1, 0, 1); and of |x|, |w|"""
    X, W = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    pad = (1, 1, 1, 1) if pad_lo else (0, 1, 0, 1)
    f = torch.nn.functional

    def conv(a, b):
        return f.conv2d(f.pad(a, pad), b, stride=2).permute(0, 2, 3, 1)
    return conv(X, W), conv(X.abs(), W.abs())


# (N, H, W, C, pad_lo): the U-Net downsamplers at 64^2 latents (pad 1; N = 2 and 16), the VAE encoder's at 512^2 (pad (0,1,0,1)),
# DPT's ResNet stride-2 convs (pad (0,1,0,1)) and its reassemble level-4 conv (pad 1), the tiny configs
CONV_S2_CASES = [(2, 64, 64, 320, 1), (16, 64, 64, 320, 1), (2, 32, 32, 640, 1), (2, 16, 16, 1280, 1), (16, 16, 16, 1280, 1),
                 (1, 512, 512, 128, 0), (1, 256, 256, 256, 0), (1, 128, 128, 512, 0), (4, 128, 128, 512, 0),
                 (1, 96, 96, 128, 0), (1, 48, 48, 256, 0), (1, 24, 24, 768, 1),
                 (2, 32, 32, 64, 1), (6, 16, 16, 128, 1), (1, 256, 256, 64, 0), (3, 64, 64, 128, 0)]


@pytest.mark.parametrize("N,H,W,Cc,pad_lo", CONV_S2_CASES)
def test_conv3_s2_matches_fp64(L, N, H, W, Cc, pad_lo):
    """mi3d_op_conv3_s2 (Cout = C, bias, a split-K workspace as the SD engine passes one).  Bound as test_conv3_sd_shapes_match_fp64:
    2 K u conv(|x|, |w|) + epilogue ulps + one fp16 rounding, K = 9 C.  The im2col matrix left in col is checked bit for bit."""
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + H + Cc + pad_lo)
    Ho, Wo = H // 2, W // 2
    x = rnd(g, N, H, W, Cc)
    w = rnd(g, Cc, 3, 3, Cc, scale=(9 * Cc) ** -0.5)
    bias = torch.randn(Cc, device="cuda", generator=g)
    cv = Canvas(N * Ho * Wo * Cc)
    y = cv.view((N, Ho, Wo, Cc), (Ho * Wo * Cc, Wo * Cc, Cc, 1))
    col = torch.empty(N * Ho * Wo * 9 * Cc, dtype=torch.float16, device="cuda")
    ws = torch.full((2048 * 2560,), float("nan"), device="cuda")
    plan = (C.c_int * 2)(0, 0)
    sync_check(L, L.lib().mi3d_op_conv3_s2(L.ptr(x), L.ptr(w), L.ptr(y), N, H, W, Cc, Ho, Wo, Cc, L.ptr(bias), pad_lo, L.ptr(col),
                                           C.c_size_t(col.numel() * 2), L.ptr(ws), C.c_size_t(ws.numel() * 4), plan, L.stream()), "op_conv3_s2")
    print(f"planned block_n {plan[0]}, splits {plan[1]}")
    acc, absacc = conv_s2_ref(x, w, pad_lo)
    ref = acc + bias.double()
    e = acc_bound(9 * Cc, absacc, 1.0, bias.double().expand_as(acc))
    check(f"conv3_s2 {N}x{H}x{W}x{Cc} pad_lo{pad_lo}", y, ref, f16_round(ref, e))
    cv.check_untouched("conv3_s2")
    pad = (0, 0, 1, 1, 1, 1) if pad_lo else (0, 0, 0, 1, 0, 1)
    xp = torch.nn.functional.pad(x, pad)
    taps = torch.stack([xp[:, ky:ky + 2 * Ho:2, kx:kx + 2 * Wo:2] for ky in range(3) for kx in range(3)], 3)    # [N][Ho][Wo][9][C]
    assert torch.equal(col.view(N, Ho, Wo, 9, Cc).view(torch.int16), taps.contiguous().view(torch.int16)), "im2col"


# the VAE encoder's input gradient through its downsamplers (512^2: C 128 / 256 / 512), DPT-sized, the tiny VAE, and an odd size
COL2IM_CASES = [(1, 512, 512, 128, 0), (1, 256, 256, 256, 0), (1, 128, 128, 512, 0), (4, 128, 128, 512, 0), (8, 64, 64, 64, 0),
                (1, 64, 64, 128, 0), (2, 24, 24, 768, 1), (1, 33, 47, 64, 1), (2, 33, 47, 64, 0)]


@pytest.mark.parametrize("N,H,W,Cc,pad_lo", COL2IM_CASES)
def test_col2im_s2_matches_fp64_scatter(L, N, H, W, Cc, pad_lo):
    """mi3d_op_col2im_s2: dx[n,h,w,c] = sum of dcol over the (output pixel, tap) pairs that read (h, w), against an fp64 scatter-add of the
    same dcol (the adjoint of the stride-2 im2col, Ho = H // 2).  At most 4 terms: 4 fp32 roundings + one fp16 rounding."""
    g = torch.Generator(device="cuda").manual_seed(N * 100 + H + W + Cc + pad_lo)
    Ho, Wo = H // 2, W // 2
    dcol = rnd(g, N, Ho, Wo, 9, Cc)
    cv = Canvas(N * H * W * Cc)
    dx = cv.view((N, H, W, Cc), (H * W * Cc, W * Cc, Cc, 1))
    sync_check(L, L.lib().mi3d_op_col2im_s2(L.ptr(dcol), L.ptr(dx), N, H, W, Cc, Ho, Wo, pad_lo, L.stream()), "op_col2im_s2")
    ref = torch.zeros(N, H + 2, W + 2, Cc, dtype=torch.float64, device="cuda")         # padded frame: index h + 1 - pad_lo... below
    absr = torch.zeros_like(ref)
    off = 1 - pad_lo
    D = dcol.double()
    for ky in range(3):
        for kx in range(3):
            t = ky * 3 + kx
            ref[:, off + ky:off + ky + 2 * Ho:2, off + kx:off + kx + 2 * Wo:2] += D[:, :, :, t]
            absr[:, off + ky:off + ky + 2 * Ho:2, off + kx:off + kx + 2 * Wo:2] += D[:, :, :, t].abs()
    ref, absr = ref[:, 1:H + 1, 1:W + 1], absr[:, 1:H + 1, 1:W + 1]
    check(f"col2im_s2 {N}x{H}x{W}x{Cc} pad_lo{pad_lo}", dx, ref, f16_round(ref, 4 * U32 * absr))
    cv.check_untouched("col2im_s2")


# ------------------------------------------------------------------------------------------------------------------------------
# Builder::conv_small_cin / conv_small_cout
# ------------------------------------------------------------------------------------------------------------------------------
# (N, H, W, Cin, Cout, bias): U-Net conv_in (4 -> 320 at 64^2, N 2 / 16), VAE encoder conv_in (4 -> 128 at 512^2), the decoder's conv_in
# (4 -> 512 at 64^2), the VAE input gradient through conv_out (8 -> 512 at 64^2, the largest weight staging: 144 KiB), VGG conv1_1
# (4 -> 64), the tiny configs, an odd pixel count
CIN_CASES = [(2, 64, 64, 4, 320, True), (16, 64, 64, 4, 320, True), (1, 512, 512, 4, 128, True), (1, 64, 64, 4, 512, True),
             (1, 64, 64, 8, 512, False), (8, 64, 64, 8, 512, False), (1, 224, 224, 4, 64, True), (2, 32, 32, 4, 64, True),
             (1, 32, 32, 8, 128, False), (3, 33, 47, 4, 64, False), (1, 33, 47, 8, 72, True)]


@pytest.mark.parametrize("N,H,W,Cin,Cout,with_bias", CIN_CASES)
def test_conv_small_cin_matches_fp64(L, N, H, W, Cin, Cout, with_bias):
    """mi3d_op_conv_small_cin: fp32 weights, fp32 FMA chain of 9 Cin terms from the bias.  Bound: 2 K u conv(|x|, |w|) + 4u |bias|
    + one fp16 rounding, K = 9 Cin."""
    g = torch.Generator(device="cuda").manual_seed(N * 10 + H + Cin * 100 + Cout)
    x = rnd(g, N, H, W, Cin)
    w = torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) * (9 * Cin) ** -0.5
    bias = torch.randn(Cout, device="cuda", generator=g) if with_bias else None
    cv = Canvas(N * H * W * Cout)
    y = cv.view((N, H, W, Cout), (H * W * Cout, W * Cout, Cout, 1))
    sync_check(L, L.lib().mi3d_op_conv_small_cin(L.ptr(x), L.ptr(w), L.ptr(bias), L.ptr(y), N, H, W, Cin, Cout, L.stream()), "op_conv_small_cin")
    acc, absacc = conv_ref(x, w)
    extra = [bias.double().expand_as(acc)] if with_bias else []
    ref = acc + (bias.double() if with_bias else 0.0)
    check(f"conv_small_cin {N}x{H}x{W} {Cin}->{Cout} bias{int(with_bias)}", y, ref, f16_round(ref, acc_bound(9 * Cin, absacc, 1.0, *extra)))
    cv.check_untouched("conv_small_cin")


# (N, H, W, Cin, Cout, bias): U-Net conv_out (320 -> 4 at 64^2, N 2 / 16: 32-lane groups), the VAE encoder's conv_out (512 -> 8 at 64^2,
# N 1 / 8), the decoder's conv_out (128 -> 4 at 512^2: 16-lane groups), the VAE image gradient through conv_in (128 -> 4 at 512^2, no
# bias), VGG's (64 -> 4), the tiny configs, odd pixel counts (the last warp's second pixel idle at Cin <= 128)
COUT_CASES = [(2, 64, 64, 320, 4, True), (16, 64, 64, 320, 4, True), (1, 64, 64, 512, 8, True), (8, 64, 64, 512, 8, True),
              (1, 512, 512, 128, 4, True), (1, 512, 512, 128, 4, False), (1, 224, 224, 64, 4, False), (2, 32, 32, 64, 4, True),
              (1, 32, 32, 128, 8, True), (1, 33, 47, 64, 4, False), (3, 33, 47, 136, 8, True), (1, 7, 9, 128, 8, False)]


@pytest.mark.parametrize("N,H,W,Cin,Cout,with_bias", COUT_CASES)
def test_conv_small_cout_matches_fp64(L, N, H, W, Cin, Cout, with_bias):
    """mi3d_op_conv_small_cout: fp16 weights, per-lane fp32 FMA chains, a shuffle tree over the lane group, the bias added last, fp32 out.
    Bound: 2 K u conv(|x|, |w|) + 4u |bias| + u |y|, K = 9 Cin."""
    g = torch.Generator(device="cuda").manual_seed(N * 10 + H + Cin * 100 + Cout + 1)
    x = rnd(g, N, H, W, Cin)
    w = rnd(g, Cout, 3, 3, Cin, scale=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout, device="cuda", generator=g) if with_bias else None
    cv = Canvas(N * H * W * Cout, torch.float32)
    y = cv.view((N, H, W, Cout), (H * W * Cout, W * Cout, Cout, 1))
    sync_check(L, L.lib().mi3d_op_conv_small_cout(L.ptr(x), L.ptr(w), L.ptr(bias), L.ptr(y), N, H, W, Cin, Cout, L.stream()), "op_conv_small_cout")
    acc, absacc = conv_ref(x, w)
    extra = [bias.double().expand_as(acc)] if with_bias else []
    ref = acc + (bias.double() if with_bias else 0.0)
    check(f"conv_small_cout {N}x{H}x{W} {Cin}->{Cout} bias{int(with_bias)}", y, ref, acc_bound(9 * Cin, absacc, 1.0, *extra) + U32 * ref.abs() + 1e-30)
    cv.check_untouched("conv_small_cout")


# ------------------------------------------------------------------------------------------------------------------------------
# k_linear_small / k_linear_small_grouped (the time embedding and the per-ResBlock projections)
# ------------------------------------------------------------------------------------------------------------------------------
ROWS = [1, 2, 8, 10, 16]          # the U-Net batch 2G for G = 1, 4, 5 and 8 views; rows 8.. are a second block of the kernel


def run_linear_small(L, x, ws, biases, B, K, silu_in, silu_out, grouped):
    """ws / biases: one entry per layer; returns the canvases and the y views [B][N_i]"""
    layers = len(ws)
    Ns = [w.shape[0] for w in ws]
    cvs = [Canvas(B * n + 97, torch.float32) for n in Ns]
    ys = [cv.view((B, n), (n, 1)) for cv, n in zip(cvs, Ns)]
    Wp = (C.c_void_p * layers)(*[w.data_ptr() for w in ws])
    Bp = (C.c_void_p * layers)(*[b.data_ptr() if b is not None else None for b in biases])
    Yp = (C.c_void_p * layers)(*[y.data_ptr() for y in ys])
    Np = (C.c_int * layers)(*Ns)
    sync_check(L, L.lib().mi3d_op_linear_small(L.ptr(x), Wp, Bp, Yp, Np, layers, B, K, int(silu_in), int(silu_out), int(grouped), L.stream()),
               "op_linear_small")
    return cvs, ys


def linear_small_ref(x, w, bias, silu_in, silu_out, K):
    """fp64 y = act(bias + act(x) W^T).  Bound: each lane's fp32 FMA chain (ln_lane_terms(K) terms), the 5-level warp tree and the bias
    add: (n + 8) u (|act(x)| |W|^T + |bias|); SiLU on x adds its __expf ulps times |W|; SiLU on y carries the bound by 1.1 + its ulps."""
    X, Wd = x.double(), w.double()
    ax = silu(X) if silu_in else X
    y = ax @ Wd.t()
    n = ln_lane_terms(K)
    e = (n + 8) * U32 * (ax.abs() @ Wd.abs().t())
    if silu_in:
        e = e + silu_ulps(X) @ Wd.abs().t()
    if bias is not None:
        y = y + bias.double()
        e = e + (n + 8) * U32 * bias.double().abs()
    if silu_out:
        return silu(y), 1.1 * e + silu_ulps(y)
    return y, e + U32 * y.abs()


@pytest.mark.parametrize("B", ROWS, ids=[f"B{b}" for b in ROWS])
@pytest.mark.parametrize("K,N", [(320, 1280), (1280, 1280), (64, 256), (256, 1001)])
@pytest.mark.parametrize("silu_in,silu_out", [(False, True), (False, False), (True, False), (True, True)])
def test_linear_small_matches_fp64(L, B, K, N, silu_in, silu_out):
    """k_linear_small for every U-Net batch B = 2G the engine plans (G <= 8), a distinct input row per b: linear_1 (K = 320 =
    SD's c0, not a multiple of 256; 64 the tiny config's) with SiLU on its output, linear_2 (K = 1280), SiLU on the input.
    N = 1001 leaves the last CTA's warps partly without an output."""
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + K + N + 2 * silu_in + silu_out)
    x = torch.randn(B, K, device="cuda", generator=g) * 2
    w = rnd(g, N, K, scale=K ** -0.5)
    bias = torch.randn(N, device="cuda", generator=g)
    cvs, ys = run_linear_small(L, x, [w], [bias], B, K, silu_in, silu_out, False)
    ref, e = linear_small_ref(x, w, bias, silu_in, silu_out, K)
    check(f"linear_small B{B} K{K} N{N} silu_in{int(silu_in)} silu_out{int(silu_out)}", ys[0], ref, e + 1e-30)
    cvs[0].check_untouched("linear_small")


@pytest.mark.parametrize("B", ROWS, ids=[f"B{b}" for b in ROWS])
@pytest.mark.parametrize("K", [1280, 256, 320])
def test_linear_small_grouped_matches_fp64(L, B, K):
    """k_linear_small_grouped as the U-Net's per-ResBlock time-embedding projections: one launch over layers of different widths
    (320, 640, 1280 and a 1001-wide one, the grid sized by the widest), SiLU on the shared input, bias on all but one layer.  Bound as
    linear_small_ref."""
    g = torch.Generator(device="cuda").manual_seed(B * 100 + K)
    x = torch.randn(B, K, device="cuda", generator=g) * 2
    Ns = [320, 640, 1280, 1001, 1280]
    ws = [rnd(g, n, K, scale=K ** -0.5) for n in Ns]
    biases = [torch.randn(n, device="cuda", generator=g) if i != 3 else None for i, n in enumerate(Ns)]
    cvs, ys = run_linear_small(L, x, ws, biases, B, K, True, False, True)
    for i, (w, b, y, cv) in enumerate(zip(ws, biases, ys, cvs)):
        ref, e = linear_small_ref(x, w, b, True, False, K)
        check(f"linear_small_grouped B{B} K{K} layer {i} N{w.shape[0]}", y, ref, e + 1e-30)
        cv.check_untouched(f"linear_small_grouped layer {i}")


# ------------------------------------------------------------------------------------------------------------------------------
# per-view latent kernels (mi3d_sd_encode / _backward, mi3d_sd_unet_sds)
# ------------------------------------------------------------------------------------------------------------------------------
VIEWS = [3, 5, 8]


@pytest.mark.parametrize("G", VIEWS)
@pytest.mark.parametrize("H,W,S", [(64, 64, 256), (128, 128, 256), (256, 256, 512), (128, 128, 512), (96, 128, 256)])
def test_interp_in_and_backward_match_fp64(L, G, H, W, S):
    """k_interp_in: bilinear (F.interpolate, align_corners=False) of each view's [3][H][W] to S x S, 2 v - 1, NHWC fp16 with a zero 4th
    channel; the source coordinates are exact at these ratios, so the bound is the fp32 lerps (6 u max|p|) and the 2 v - 1 (2 u) plus one
    fp16 rounding.  k_interp_bwd: the adjoint, 2 interp^T(g) over channels 0..2 of g [S*S][4], against fp64 autograd of the same
    interpolation (every output pixel's gradient reaches its source pixels, whatever the kernel's footprint window); bound: (n + 4) u of
    the adjoint of |g| with n = the footprint's terms."""
    gen = torch.Generator(device="cuda").manual_seed(G * 1000 + H + W + S)
    rgb = torch.rand(G, 3, H, W, device="cuda", generator=gen)
    cv = Canvas(G * S * S * 4)
    out = cv.view((G, S, S, 4), (S * S * 4, S * 4, 4, 1))
    sync_check(L, L.lib().mi3d_op_interp_in(L.ptr(rgb), H, W, L.ptr(out), S, G, L.stream()), "op_interp_in")
    f = torch.nn.functional
    R = rgb.double().requires_grad_()
    up = f.interpolate(R, size=(S, S), mode="bilinear", align_corners=False)
    ref = (2 * up - 1).permute(0, 2, 3, 1)
    e = 8 * U32 * (2 * rgb.double().abs().amax((1, 2, 3)).view(G, 1, 1, 1) + 1)
    check(f"interp_in G{G} {H}x{W}->{S}", out[..., :3], ref.detach(), f16_round(ref.detach(), e.expand(G, S, S, 3)))
    assert (out[..., 3].view(torch.int16) == 0).all(), "the 4th channel is +0"
    cv.check_untouched("interp_in")

    g = torch.randn(G, S * S, 4, device="cuda", generator=gen)
    gcv = Canvas(G * 3 * H * W, torch.float32)
    grad = gcv.view((G, 3, H, W), (3 * H * W, H * W, W, 1))
    sync_check(L, L.lib().mi3d_op_interp_bwd(L.ptr(g), S, L.ptr(grad), H, W, G, L.stream()), "op_interp_bwd")
    gimg = g[..., :3].double().reshape(G, S, S, 3).permute(0, 3, 1, 2)
    (ref_g,) = torch.autograd.grad(up, R, gimg)
    Ra = rgb.double().requires_grad_()
    upa = f.interpolate(Ra, size=(S, S), mode="bilinear", align_corners=False)
    (abs_g,) = torch.autograd.grad(upa, Ra, gimg.abs())
    n = (2 * S // min(H, W) + 2) ** 2
    check(f"interp_bwd G{G} {S}->{H}x{W}", grad, 2 * ref_g, 2 * (n + 4) * U32 * abs_g + 1e-30)
    gcv.check_untouched("interp_bwd")


def posterior_case(gen, G, pix, identity):
    """conv_out [G][pix][8], quant_conv (qw, qb), eps [G][4][pix].  identity: qw = I, qb = 0 and logvar values at -30 and 20 exactly and one
    fp32 ulp either side of each (plus far outside), so the clamp and its gradient mask are pinned"""
    co = torch.randn(G, pix, 8, device="cuda", generator=gen) * 2
    if identity:
        qw, qb = torch.eye(8, device="cuda"), torch.zeros(8, device="cuda")
        edge = torch.tensor([-30.0, 20.0], dtype=torch.float32)
        vals = torch.cat([edge, torch.nextafter(edge, edge - 1), torch.nextafter(edge, edge + 1), torch.tensor([-45.0, 33.0])]).cuda()
        lv = co[..., 4:]
        idx = torch.randint(0, vals.numel() + 2, lv.shape, device="cuda", generator=gen)
        lv[idx < vals.numel()] = vals[idx[idx < vals.numel()]]
    else:
        qw = torch.randn(8, 8, device="cuda", generator=gen) * 0.5
        qb = torch.randn(8, device="cuda", generator=gen)
    eps = torch.randn(G, 4, pix, device="cuda", generator=gen)
    return co, qw, qb, eps


@pytest.mark.parametrize("G", VIEWS)
@pytest.mark.parametrize("pix", [64 * 64, 32 * 32, 1000])
@pytest.mark.parametrize("identity", [False, True])
def test_sample_latents_and_backward_match_fp64(L, G, pix, identity):
    """k_sample_latents: m = qb + qw conv_out (8 fp32 FMAs), lat = (m[c] + exp(0.5 clamp(m[4+c], -30, 20)) eps) 0.18215; and its gradient
    d conv_out = qw^T dm with dm[c] = 0.18215 g, dm[4+c] = 0.18215 g eps 0.5 exp(0.5 lv) where -30 <= lv <= 20 (both ends inclusive),
    else 0.  Bound: e_m = 10 u (|qb| + |qw| |co|); the exp moves by 0.5 e_m and its 2 ulp; a few u per product; the transposed product
    10 u |qw|^T |dm| + |qw|^T e_dm."""
    gen = torch.Generator(device="cuda").manual_seed(G * 100 + pix + int(identity))
    co, qw, qb, eps = posterior_case(gen, G, pix, identity)
    cv = Canvas(G * 4 * pix, torch.float32)
    lat = cv.view((G, 4, pix), (4 * pix, pix, 1))
    sync_check(L, L.lib().mi3d_op_sample_latents(L.ptr(co), L.ptr(qw), L.ptr(qb), L.ptr(eps), L.ptr(lat), pix, G, L.stream()), "op_sample_latents")
    CO, QW, QB, EPS = co.double(), qw.double(), qb.double(), eps.double()
    m = CO @ QW.t() + QB                                          # [G][pix][8]
    e_m = 10 * U32 * (CO.abs() @ QW.abs().t() + QB.abs())
    mean, lv = m[..., :4].permute(0, 2, 1), m[..., 4:].permute(0, 2, 1)
    em_mean, em_lv = e_m[..., :4].permute(0, 2, 1), e_m[..., 4:].permute(0, 2, 1)
    inside = (lv >= -30) & (lv <= 20)
    std = torch.exp(0.5 * lv.clamp(-30, 20))
    ref = (mean + std * EPS) * 0.18215
    e_std = std * (0.5 * em_lv + 4 * U32)
    err = 0.18215 * (em_mean + e_std * EPS.abs() + 3 * U32 * (mean.abs() + (std * EPS).abs())) + U32 * ref.abs()
    check(f"sample_latents G{G} pix{pix} identity{int(identity)}", lat, ref, err + 1e-30)
    cv.check_untouched("sample_latents")
    if identity:
        # the clamp is pinned: every m[4+c] is exact, so std is exp(0.5 * clamp) to expf's accuracy even at the edges
        assert torch.equal(lv, co[..., 4:].double().permute(0, 2, 1))

    g_lat = torch.randn(G, 4, pix, device="cuda", generator=gen)
    gcv = Canvas(G * pix * 8, torch.float32)
    gco = gcv.view((G, pix, 8), (pix * 8, 8, 1))
    sync_check(L, L.lib().mi3d_op_sample_latents_bwd(L.ptr(co), L.ptr(qw), L.ptr(qb), L.ptr(eps), L.ptr(g_lat), L.ptr(gco), pix, G, L.stream()),
               "op_sample_latents_bwd")
    GL = g_lat.double() * 0.18215
    dm_lv = GL * EPS * 0.5 * torch.exp(0.5 * lv) * inside
    dm = torch.cat([GL, dm_lv], 1).permute(0, 2, 1)               # [G][pix][8]
    e_dm = torch.cat([U32 * GL.abs(), dm_lv.abs() * (0.5 * em_lv + 6 * U32)], 1).permute(0, 2, 1)
    ref_g = dm @ QW
    err_g = 10 * U32 * (dm.abs() @ QW.abs()) + e_dm @ QW.abs()
    if not identity:
        # a random logvar within its error of a clamp edge could take either side of the mask; none may be that close
        assert (((lv + 30).abs() > em_lv) & ((lv - 20).abs() > em_lv)).all()
    check(f"sample_latents_bwd G{G} pix{pix} identity{int(identity)}", gco, ref_g, err_g + 1e-30)
    gcv.check_untouched("sample_latents_bwd")


@pytest.mark.parametrize("G", VIEWS)
@pytest.mark.parametrize("pix", [64 * 64, 1000])
def test_add_noise_duplicates_each_view_into_its_two_rows(L, G, pix):
    """k_add_noise: rows v (uncond) and G + v (text) of the U-Net input both hold fp16(sqrt(a_t) z_v + sqrt(1 - a_t) eps_v) in NHWC, bit
    for bit the same; nothing else is written (the canvas holds one more row).  Bound: 4 u of the terms + one fp16 rounding."""
    gen = torch.Generator(device="cuda").manual_seed(G * 10 + pix)
    lat = torch.randn(G, 4, pix, device="cuda", generator=gen)
    noise = torch.randn(G, 4, pix, device="cuda", generator=gen)
    alphas = torch.rand(1000, device="cuda", generator=gen) * 0.98 + 0.01
    t = torch.tensor([637], dtype=torch.long, device="cuda")
    cv = Canvas((2 * G + 1) * pix * 4)
    xin = cv.view((2 * G, pix, 4), (pix * 4, 4, 1))
    sync_check(L, L.lib().mi3d_op_add_noise(L.ptr(lat), L.ptr(noise), L.ptr(alphas), L.ptr(t), L.ptr(xin), pix, G, L.stream()), "op_add_noise")
    a = alphas[637].double()
    sa, sb = torch.sqrt(a), torch.sqrt(1 - a)
    ref = (sa * lat.double() + sb * noise.double()).permute(0, 2, 1)
    e = 4 * U32 * ((sa * lat.double()).abs() + (sb * noise.double()).abs()).permute(0, 2, 1)
    check(f"add_noise G{G} pix{pix} uncond rows", xin[:G], ref, f16_round(ref, e))
    assert torch.equal(xin[:G].view(torch.int16), xin[G:].view(torch.int16)), "rows v and G + v differ"
    cv.check_untouched("add_noise")


@pytest.mark.parametrize("G", VIEWS)
@pytest.mark.parametrize("case", ["random", "nonfinite", "overflow"])
def test_cfg_sds_pairs_views_and_sanitises_like_nan_to_num(L, G, case):
    """k_cfg_sds: view v takes U-Net rows v (uncond) and G + v (text): noise_pred = text + gs (text - uncond) and grad =
    nan_to_num((1 - a_t) (noise_pred - noise)) (NaN -> 0, +-inf -> +-FLT_MAX), NHWC in, NCHW out; every view's data distinct.  'nonfinite'
    plants NaN and +-inf in the U-Net output, 'overflow' takes a guidance scale that overflows fp32.  Finite results: 2 u of the CFG terms
    and u of the difference and the product; non-finite and overflowing ones exactly as torch.nan_to_num makes them."""
    gen = torch.Generator(device="cuda").manual_seed(G * 7 + len(case))
    pix = 32 * 32
    un = torch.randn(2 * G, pix, 4, device="cuda", generator=gen)
    noise = torch.randn(G, 4, pix, device="cuda", generator=gen)
    alphas = torch.rand(1000, device="cuda", generator=gen) * 0.98 + 0.01
    t = torch.tensor([421], dtype=torch.long, device="cuda")
    gs = 7.5
    if case == "nonfinite":
        pick = torch.randint(0, 12, un.shape, device="cuda", generator=gen)
        un[pick == 0] = float("nan"); un[pick == 1] = float("inf"); un[pick == 2] = -float("inf")
    elif case == "overflow":
        gs = 1e30
        un = un * 1e9
    cvp, cvg = Canvas(G * 4 * pix, torch.float32), Canvas(G * 4 * pix, torch.float32)
    npred, grad = cvp.view((G, 4, pix), (4 * pix, pix, 1)), cvg.view((G, 4, pix), (4 * pix, pix, 1))
    sync_check(L, L.lib().mi3d_op_cfg_sds(L.ptr(un), L.ptr(noise), L.ptr(alphas), L.ptr(t), C.c_float(gs), L.ptr(npred), L.ptr(grad), pix, G,
                                          L.stream()), "op_cfg_sds")
    U = un.double()
    unc, txt = U[:G].permute(0, 2, 1), U[G:].permute(0, 2, 1)
    w = 1 - alphas[421].double()
    diff = txt - unc
    npd = txt + gs * diff
    gd = w * (npd - noise.double())
    e_np = 2 * U32 * (txt.abs() + (gs * diff).abs()) + U32 * (gs * diff).abs()
    e_g = w * (e_np + U32 * (npd - noise.double()).abs()) + 2 * U32 * gd.abs()
    what = f"cfg_sds G{G} {case}"
    # where the fp64 value is finite and clear of FLT_MAX, the kernel's is held to the bound; elsewhere to its IEEE / nan_to_num value
    ok_np = torch.isfinite(npd) & (npd.abs() < FLT_MAX * (1 - 1e-5))
    far_np = torch.isnan(npd) | (npd.abs() > FLT_MAX * (1 + 1e-5))
    # an fp32 noise_pred that overflowed makes the gradient +-inf even where (1 - a_t) would bring it back below FLT_MAX
    ok_g = torch.isfinite(gd) & (gd.abs() < FLT_MAX * (1 - 1e-5)) & ok_np
    far_g = (torch.isnan(gd) | (gd.abs() > FLT_MAX * (1 + 1e-5)) | far_np) & (ok_np | far_np)
    if case == "random":
        assert ok_np.all() and ok_g.all()
    else:
        assert far_g.any(), "the case must reach the sanitising branch"
    check(what + " noise_pred", npred, npd.nan_to_num(0.0), e_np + 1e-30, mask=ok_np)
    check(what + " grad", grad, gd.nan_to_num(0.0), e_g + 1e-30, mask=ok_g)
    want_np = npd[far_np].float()                                  # NaN, or +-inf past FLT_MAX
    got_np = npred[far_np]
    assert torch.equal(torch.isnan(got_np), torch.isnan(want_np)) and torch.equal(got_np[~torch.isnan(got_np)], want_np[~torch.isnan(want_np)])
    want_g = torch.nan_to_num(torch.where(far_np, w * npd.float().double(), gd)[far_g].float())      # 0, or +-FLT_MAX
    assert torch.equal(grad[far_g], want_g), "grad is not nan_to_num of the fp32 value"
    assert torch.isfinite(grad).all()
    cvp.check_untouched("cfg_sds noise_pred")
    cvg.check_untouched("cfg_sds grad")
