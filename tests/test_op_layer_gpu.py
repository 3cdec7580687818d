"""GPU: the op layer every planned engine is built on (plan::Builder / plan::TowerBuilder: the tile GEMM with each epilogue, batched
per-head products, split-K, both implicit convs, both attention paths, the row kernels), one op at a time through the builder methods
the engines call (mi3d_op_* in csrc/tc_test.cu), against torch float64 computed from exactly the fp16 / fp32 values the kernel reads.

Every comparison is element-wise, |got - ref| <= bound, with the bound derived per element from the kernel's arithmetic:
  u = 2^-24 (one fp32 rounding), one fp16 output rounding = 2^-11 |ref| + 2^-25 (the absolute part covers fp16 subnormals);
  a K-term fp32 dot product of exact fp16 products: 2 K u (|A| |B|^T) (2 u per add: the tensor-core adder may truncate);
  epilogue arithmetic: a few u of the magnitudes involved; activations carry the pre-activation bound through max |act'|.
The worst err / bound ratio of every case is printed.  Every output buffer is larger than the op's output (rows past M, ldc > N where
the op allows it, a guard region after the end) and filled with a sentinel; what lies outside the output must be unchanged bit for bit.
"""
import ctypes as C
import importlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
U16 = 2.0 ** -11
SUB16 = 2.0 ** -25
GUARD = 4096
QG_D = 1.0999          # max |d/dy y sigmoid(1.702 y)|
GELU_D = 1.1290        # max |d/dy 0.5 y (1 + erf(y / sqrt 2))|
EPI = {"plain": 0, "geglu": 1, "transposed": 2, "quickgelu": 3, "quickgelu_bwd": 4, "relu": 5, "relu_bwd": 6, "gelu": 7}


@pytest.fixture(scope="module")
def L():
    return importlib.import_module("make-it-3d_b200._lib")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Canvas:
    """A sentinel-filled flat buffer; views taken with .view() are the op's output, everything else must stay untouched."""

    def __init__(self, n, dtype=torch.float16):
        it = torch.int16 if dtype == torch.float16 else torch.int32
        self.sent = 0x7D3F if it == torch.int16 else 0x7FC0BEEF          # NaN bit patterns no kernel produces
        self.raw = torch.full((n + GUARD,), self.sent, dtype=it, device="cuda")
        self.t = self.raw.view(dtype)
        self.written = torch.zeros(n + GUARD, dtype=torch.bool, device="cuda")

    def view(self, shape, strides, offset=0):
        self.written.as_strided(shape, strides, offset).fill_(True)
        return self.t.as_strided(shape, strides, offset)

    def check_untouched(self, what):
        bad = int((self.raw[~self.written] != self.sent).sum())
        assert bad == 0, f"{what}: {bad} elements outside the output were written"


def check(what, got, ref, bound, mask=None):
    """element-wise |got - ref| <= bound (over mask); prints the worst ratio"""
    ratio = (got.double() - ref).abs() / bound
    if mask is not None:
        ratio = ratio[mask]
    worst = ratio.max().item() if ratio.numel() else 0.0
    print(f"{what}: worst err/bound {worst:.3g}")
    assert worst <= 1.0, f"{what}: err/bound {worst:.3g}"          # NaN fails here too


def f16_round(ref, e):
    """bound after one fp16 output rounding of a value within e of ref"""
    return e + U16 * (ref.abs() + e) + SUB16


def rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).half()


def sync_check(L, code, what):
    L.check(code, what)
    torch.cuda.synchronize()


def qg_ulps(y):
    """__expf (ex2.approx: ~2^-22 relative, plus the rounding of arg * log2 e) inside y * sigmoid(1.702 y), and its three roundings"""
    d = 2.0 ** -21 + 2.0 ** -23 * 1.702 * y.abs()
    return y.abs() * (0.25 * d + 4 * U32)


def qg_grad(x):
    s = torch.sigmoid(1.702 * x)
    return s * (1 + 1.702 * x * (1 - s))


def gelu(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def gelu_ulps(y):
    """erff (2 ulp of a value <= 1), the rounding of its argument, and three fp32 roundings"""
    return 0.5 * y.abs() * (2.0 ** -22 + y.abs() * U32) + 3 * U32 * y.abs()


# ------------------------------------------------------------------------------------------------------------------------------
# Builder::gemm
# ------------------------------------------------------------------------------------------------------------------------------
def run_gemm(L, a, b, N, out16=None, out32=None, ldc=0, bias=None, row_bias=None, rpg=1, residual=None, ld_res=0, mode=0, alpha=1.0,
             aux=None, batch=1, b_batched=0, ws=None, out_z1=1, s_lo=0, s_hi=0):
    """a, b: dicts with the fields of Builder::Mat (p, ld, rows, z1, sz1, z2, sz2); K from a's tensor layout"""
    g = L.OpGemmArgs()
    for pre, m in (("a", a), ("b", b)):
        setattr(g, pre, m["p"].data_ptr())
        setattr(g, "ld" + pre, m["ld"]); setattr(g, pre + "_rows", m["rows"])
        setattr(g, pre + "_z1", m.get("z1", 1)); setattr(g, pre + "_sz1", m.get("sz1", 0))
        setattr(g, pre + "_z2", m.get("z2", 1)); setattr(g, pre + "_sz2", m.get("sz2", 0))
    g.K = a["K"]; g.N = N; g.batch = batch; g.b_batched = b_batched
    g.out16 = out16.data_ptr() if out16 is not None else None
    g.out32 = out32.data_ptr() if out32 is not None else None
    g.ldc = ldc; g.out_z1 = out_z1; g.out_s_lo = s_lo; g.out_s_hi = s_hi
    g.bias = bias.data_ptr() if bias is not None else None
    g.row_bias = row_bias.data_ptr() if row_bias is not None else None
    g.rows_per_group = rpg
    g.residual = residual.data_ptr() if residual is not None else None
    g.ld_res = ld_res; g.mode = mode; g.alpha = alpha
    g.aux = aux.data_ptr() if aux is not None else None
    plan = (C.c_int * 2)(0, 0)
    wsp, wsb = (C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel() * 4)) if ws is not None else (C.c_void_p(0), C.c_size_t(0))
    sync_check(L, L.lib().mi3d_op_gemm(C.byref(g), wsp, wsb, plan, L.stream()), "op_gemm")
    return plan[0], plan[1]


def acc_bound(K, absacc, alpha, *extra):
    """fp32 accumulation of K exact fp16 products, then alpha * acc + bias + row_bias + residual in fp32"""
    e = 2 * K * U32 * abs(alpha) * absacc + 4 * U32 * abs(alpha) * absacc
    for t in extra:
        e = e + 4 * U32 * t.abs()
    return e


# (mode, M, N, K, features, block-N the planner picks on a 132-SM H100)
#   features: a alpha = 0.5, b bias, r1 / rg row_bias with rows_per_group 1 / 64, s residual, f fp32 out, w ldc > N, x aux
GEMM_CASES = [
    ("plain", 1, 64, 768, "abw", 64),
    ("plain", 33, 128, 1024, "bs", 64),
    ("plain", 77, 1024, 1024, "bsw", 64),
    ("plain", 128, 256, 4096, "f", 64),
    ("plain", 197, 2304, 768, "b", 64),
    ("plain", 257, 960, 512, "br1w", 64),
    ("plain", 577, 4096, 1024, "brgs", 128),
    ("plain", 8192, 768, 320, "ab", 256),
    ("plain", 8192, 384, 640, "sw", 128),
    ("plain", 8192, 320, 640, "brgs", 160),
    ("plain", 1408, 960, 256, "bfw", 160),
    ("plain", 4096, 640, 192, "absf", 128),
    ("plain", 5000, 1024, 320, "bf", 256),
    ("geglu", 197, 512, 256, "b", 64),
    ("geglu", 8192, 1280, 320, "b", 256),
    ("geglu", 8192, 320, 128, "b", 160),
    ("transposed", 197, 256, 128, "b", 64),
    ("transposed", 8192, 320, 64, "ab", 160),
    ("quickgelu", 77, 3072, 768, "bx", 64),
    ("quickgelu", 197, 1024, 256, "b", 64),
    ("quickgelu", 8192, 3072, 768, "bx", 256),
    ("quickgelu", 8192, 320, 128, "bx", 64),
    ("quickgelu", 1408, 960, 128, "b", 64),
    ("gelu", 77, 4096, 1024, "b", 64),
    ("gelu", 8192, 320, 256, "ab", 64),
    ("gelu", 1408, 960, 64, "b", 64),
]


@pytest.mark.parametrize("mode,M,N,K,feat,want_bn", GEMM_CASES)
def test_gemm_epilogues_match_fp64(L, sms, mode, M, N, K, feat, want_bn):
    """Builder::gemm with one epilogue, ragged M, ldc > N.  y = alpha acc + bias + row_bias (+ residual) has the error
    acc_bound(); PLAIN / TRANSPOSED store y (fp16: + one rounding; fp32: + u |y|); GEGLU stores v gelu(g) (error e_v |gelu(g)| +
    |v| (1.129 e_g + erff ulps)); QUICKGELU stores q(y) (1.1 e_y + __expf ulps) and y itself to aux; GELU 1.129 e_y + erff ulps."""
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K + EPI[mode])
    alpha = 0.5 if "a" in feat else 1.0
    a = rnd(g, M, K)
    b = rnd(g, N, K, scale=K ** -0.5)
    bias = torch.randn(N, device="cuda", generator=g) if "b" in feat else None
    rpg = 64 if "rg" in feat else 1
    rb = torch.randn((M + rpg - 1) // rpg, N, device="cuda", generator=g) if ("r1" in feat or "rg" in feat) else None
    ld_res = N + 64 if "w" in feat else N
    res = rnd(g, M, ld_res) if "s" in feat else None
    f32 = "f" in feat
    N_out = N // 2 if mode == "geglu" else N
    extra = 64 if "w" in feat else 0
    if mode == "transposed":
        ldc = M + 5 + extra                           # scalar stores: any ldc
        cv = Canvas((N + 3) * ldc)
        out = cv.view((N, M), (ldc, 1))
    else:
        ldc = N_out + extra
        cv = Canvas((M + 37) * ldc, torch.float32 if f32 else torch.float16)
        out = cv.view((M, N_out), (ldc, 1))
    aux_cv = Canvas((M + 37) * ldc) if "x" in feat else None
    aux = aux_cv.view((M, N), (ldc, 1)) if aux_cv is not None else None
    bn, splits = run_gemm(L, {"p": a, "ld": K, "rows": M, "K": K}, {"p": b, "ld": K, "rows": N}, N,
                          out16=None if f32 else out, out32=out if f32 else None, ldc=ldc, bias=bias, row_bias=rb, rpg=rpg,
                          residual=res, ld_res=ld_res, mode=EPI[mode], alpha=alpha, aux=aux)
    print(f"planned block_n {bn}, splits {splits}")
    if sms == 132:
        assert (bn, splits) == (want_bn, 1)

    A, B = a.double(), b.double()
    acc, absacc = A @ B.t(), A.abs() @ B.abs().t()
    y = alpha * acc
    terms = []
    if bias is not None:
        y = y + bias.double(); terms.append(bias.double().expand(M, N))
    if rb is not None:
        rbr = rb.double().repeat_interleave(rpg, 0)[:M]
        y = y + rbr; terms.append(rbr)
    if mode == "plain" and res is not None:
        r = res[:, :N].double()
        y = y + r; terms.append(r)
    e = acc_bound(K, absacc, alpha, *terms)
    if mode == "plain":
        bound = e + U32 * y.abs() if f32 else f16_round(y, e)
        check(f"{mode} M{M} N{N} K{K}", out, y, bound)
    elif mode == "transposed":
        check(f"{mode} M{M} N{N} K{K}", out, y.t(), f16_round(y, e).t())
    elif mode == "geglu":
        v, gt, ev, eg = y[:, 0::2], y[:, 1::2], e[:, 0::2], e[:, 1::2]
        ref = v * gelu(gt)
        err = ev * gelu(gt).abs() + (v.abs() + ev) * (GELU_D * eg + gelu_ulps(gt)) + 2 * U32 * ref.abs()
        check(f"{mode} M{M} N{N} K{K}", out, ref, f16_round(ref, err))
    elif mode == "quickgelu":
        ref = y * torch.sigmoid(1.702 * y)
        check(f"{mode} M{M} N{N} K{K}", out, ref, f16_round(ref, QG_D * e + qg_ulps(y)))
        if aux is not None:
            check(f"{mode} aux M{M} N{N} K{K}", aux, y, f16_round(y, e))
    elif mode == "gelu":
        ref = gelu(y)
        check(f"{mode} M{M} N{N} K{K}", out, ref, f16_round(ref, GELU_D * e + gelu_ulps(y)))
    cv.check_untouched(mode)
    if aux_cv is not None:
        aux_cv.check_untouched(mode + " aux")


@pytest.mark.parametrize("M,N,K,want_bn", [(77, 3072, 768, 64), (197, 1024, 4096, 64), (8192, 320, 256, 64), (1408, 960, 128, 64)])
def test_gemm_quickgelu_backward_reads_the_stored_aux(L, sms, M, N, K, want_bn):
    """The CLIP MLP pair: a QUICKGELU forward stores the pre-activation to aux (fp16); the input-gradient GEMM's QUICKGELU_BWD
    epilogue reads that aux: out = y q'(aux).  Bound: e_y |q'(aux)| + |y| (1 + 1.702 |aux|) (__expf ulps of sigmoid) + one fp16
    rounding, with q' evaluated in fp64 at exactly the stored fp16 aux."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K + 4)
    a, b = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5)
    ldc = N + 64
    fwd_out = torch.empty(M, ldc, dtype=torch.float16, device="cuda")
    aux = torch.empty(M, ldc, dtype=torch.float16, device="cuda")
    run_gemm(L, {"p": a, "ld": K, "rows": M, "K": K}, {"p": b, "ld": K, "rows": N}, N, out16=fwd_out, ldc=ldc, mode=EPI["quickgelu"], aux=aux)
    K2 = 512
    dy, w = rnd(g, M, K2), rnd(g, N, K2, scale=K2 ** -0.5)
    cv = Canvas((M + 37) * ldc)
    out = cv.view((M, N), (ldc, 1))
    bn, splits = run_gemm(L, {"p": dy, "ld": K2, "rows": M, "K": K2}, {"p": w, "ld": K2, "rows": N}, N, out16=out, ldc=ldc,
                          mode=EPI["quickgelu_bwd"], aux=aux)
    print(f"planned block_n {bn}, splits {splits}")
    if sms == 132:
        assert (bn, splits) == (want_bn, 1)
    A, B = dy.double(), w.double()
    y, e = A @ B.t(), acc_bound(K2, A.abs() @ B.abs().t(), 1.0)
    x = aux[:, :N].double()
    qd = qg_grad(x)
    ref = y * qd
    err = e * qd.abs() + (y.abs() + e) * (1 + 1.702 * x.abs()) * (0.25 * (2.0 ** -21 + 2.0 ** -23 * 1.702 * x.abs()) + 6 * U32)
    check(f"quickgelu_bwd M{M} N{N}", out, ref, f16_round(ref, err))
    cv.check_untouched("quickgelu_bwd")


# block-N on a 132-SM H100: 128 for the first four, then 64 and 160.  160-wide tiles are split only when they number exactly half the
# SMs (66 at M = 4224), so on other SM counts the last case may run unsplit.
@pytest.mark.parametrize("M,N,K,rpg", [(128, 1280, 11520, 1), (256, 640, 5760, 64), (384, 1280, 4096, 128), (512, 1280, 5760, 1),
                                       (256, 320, 4096, 64), (4224, 320, 3072, 64)])
def test_gemm_split_k_planned_with_row_bias(L, sms, M, N, K, rpg):
    """Builder::gemm with a split-K workspace: batch 1, few M tiles, deep K -> the planner splits K; k_splitk_finish applies alpha,
    bias, row_bias and the residual.  Same bound as the unsplit GEMM (the K-ranges meet by fp32 adds: still 2 K u |A||B|^T)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a, b = rnd(g, M, K), rnd(g, N, K, scale=K ** -0.5)
    bias = torch.randn(N, device="cuda", generator=g)
    rb = torch.randn(M // rpg, N, device="cuda", generator=g)
    res = rnd(g, M, N)
    ldc = N + 64
    cv = Canvas((M + 37) * ldc)
    out = cv.view((M, N), (ldc, 1))
    ws = torch.full((2048 * 2560,), float("nan"), device="cuda")
    bn, splits = run_gemm(L, {"p": a, "ld": K, "rows": M, "K": K}, {"p": b, "ld": K, "rows": N}, N, out16=out, ldc=ldc, bias=bias,
                          row_bias=rb, rpg=rpg, residual=res, ld_res=N, alpha=0.75, ws=ws)
    print(f"planned block_n {bn}, splits {splits}")
    if sms == 132 or bn != 160:
        assert splits > 1
    A, B = a.double(), b.double()
    rbr = rb.double().repeat_interleave(rpg, 0)
    y = 0.75 * (A @ B.t()) + bias.double() + rbr + res.double()
    e = acc_bound(K, A.abs() @ B.abs().t(), 0.75, bias.double().expand(M, N), rbr, res.double())
    check(f"split-K M{M} N{N} K{K}", out, y, f16_round(y, e))
    cv.check_untouched("split-K")


# the batched per-head operands of TowerBuilder (transformer_plan.cuh), mirrored field for field
def heads_rows(p, ld, Tpad, heads, B):
    return {"p": p, "ld": ld, "rows": Tpad, "K": 64, "z1": heads, "sz1": 64, "z2": B, "sz2": Tpad * ld}


def heads_cols(p, ldT, Tpad, heads, B):
    return {"p": p, "ld": Tpad, "rows": 64, "K": Tpad, "z1": heads, "sz1": 64 * Tpad, "z2": B, "sz2": ldT * Tpad}


def scores(p, Tpad, heads, B):
    return {"p": p, "ld": Tpad, "rows": Tpad, "K": Tpad, "z1": heads, "sz1": Tpad * Tpad, "z2": B, "sz2": heads * Tpad * Tpad}


@pytest.mark.parametrize("B,heads,Tpad", [(1, 1, 64), (2, 12, 128), (2, 1, 320), (1, 12, 640), (2, 12, 320)])
@pytest.mark.parametrize("kind", ["scores", "pv"])
def test_batched_head_gemms_match_fp64(L, B, heads, Tpad, kind):
    """TowerBuilder::bgemm as attention_materialised builds it: S = Q K^T per (batch, head) out of the packed qkv [B*Tpad][3C]
    (heads_rows), and O = P V^T with P [B*heads][Tpad][Tpad] (scores) and V from the transposed qkvT (heads_cols), written as column
    slices of a [B*Tpad][ldc] matrix with ldc > C.  Distinct random data per (batch, head).  Bound: 2 K u |A||B|^T + one fp16 rounding."""
    g = torch.Generator(device="cuda").manual_seed(B * 100 + heads * 10 + Tpad)
    Cm = 64 * heads
    if kind == "scores":
        qkv = rnd(g, B * Tpad, 3 * Cm)
        a = heads_rows(qkv, 3 * Cm, Tpad, heads, B)
        bm = heads_rows(qkv.view(-1)[Cm:], 3 * Cm, Tpad, heads, B)
        N, K = Tpad, 64
        cv = Canvas((B * heads + 1) * Tpad * Tpad)
        out = cv.view((B * heads, Tpad, Tpad), (Tpad * Tpad, Tpad, 1))
        run_gemm(L, a, bm, N, out16=cv.t, ldc=Tpad, batch=B * heads, b_batched=1, out_z1=1, s_lo=0, s_hi=Tpad * Tpad)
        q = qkv.double().view(B, Tpad, 3, heads, 64)
        Q, Kk = q[:, :, 0].permute(0, 2, 1, 3), q[:, :, 1].permute(0, 2, 1, 3)
        ref = (Q @ Kk.transpose(-1, -2)).reshape(B * heads, Tpad, Tpad)
        absacc = (Q.abs() @ Kk.abs().transpose(-1, -2)).reshape(B * heads, Tpad, Tpad)
    else:
        P = (torch.rand(B * heads, Tpad, Tpad, device="cuda", generator=g) * (4.0 / Tpad)).half()
        qkvT = rnd(g, B, 3 * Cm, Tpad)
        a = scores(P, Tpad, heads, B)
        bm = heads_cols(qkvT.view(-1)[2 * Cm * Tpad:], 3 * Cm, Tpad, heads, B)
        N, K = 64, Tpad
        ldc = Cm + 64
        cv = Canvas((B * Tpad + 9) * ldc)
        out = cv.view((B, Tpad, heads, 64), (Tpad * ldc, ldc, 64, 1))
        run_gemm(L, a, bm, N, out16=cv.t, ldc=ldc, batch=B * heads, b_batched=1, out_z1=heads, s_lo=64, s_hi=Tpad * ldc)
        V = qkvT.double()[:, 2 * Cm:].view(B, heads, 64, Tpad)                 # [b][h][d][token]
        Pd = P.double().view(B, heads, Tpad, Tpad)
        ref = (Pd @ V.transpose(-1, -2)).permute(0, 2, 1, 3)                     # [b][token][h][d]
        absacc = (Pd.abs() @ V.abs().transpose(-1, -2)).permute(0, 2, 1, 3)
    check(f"bgemm {kind} B{B} heads{heads} Tpad{Tpad}", out, ref, f16_round(ref, acc_bound(K, absacc, 1.0)))
    cv.check_untouched(f"bgemm {kind}")


# ------------------------------------------------------------------------------------------------------------------------------
# Builder::conv3 / Builder::conv3_block
# ------------------------------------------------------------------------------------------------------------------------------
def conv_ref(x, w, pad=1):
    """fp64 3x3 conv of NHWC x with [Cout][3][3][Cin] w, and the same of |x|, |w|"""
    X, W = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    f = torch.nn.functional.conv2d
    return f(X, W, padding=pad).permute(0, 2, 3, 1), f(X.abs(), W.abs(), padding=pad).permute(0, 2, 3, 1)


# (Nimg, H, W, Cin, Cout, a split-K workspace is passed, (block-N, splits) the planner picks on a 132-SM H100)
CONV_CASES = [(2, 64, 64, 320, 320, True, (160, 1)), (2, 32, 32, 640, 640, True, (64, 1)), (2, 16, 16, 1280, 1280, True, (128, 3)),
              (2, 8, 8, 1280, 1280, True, (128, 8)), (2, 8, 8, 2560, 1280, True, (128, 8)), (2, 16, 16, 640, 320, False, (64, 1)),
              (2, 32, 32, 320, 640, False, (64, 1)), (2, 8, 8, 64, 64, False, (64, 1)), (2, 16, 16, 128, 128, False, (64, 1)),
              (1, 128, 128, 128, 256, False, (128, 1)), (2, 32, 32, 640, 1280, False, (128, 1)), (1, 256, 256, 64, 64, False, (64, 1))]


@pytest.mark.parametrize("Nimg,H,W,Cin,Cout,splitk,want", CONV_CASES)
def test_conv3_sd_shapes_match_fp64(L, sms, Nimg, H, W, Cin, Cout, splitk, want):
    """Builder::conv3 as the SD U-Net and VAE call it: bias, the time embedding as row_bias with rows_per_group = H W (one row per
    image), residual, and (with a workspace) the split-K the planner chooses at the deep levels.  Bound: 2 K u conv(|x|, |w|)
    + epilogue ulps + one fp16 rounding, K = 9 Cin."""
    g = torch.Generator(device="cuda").manual_seed(H * 10 + Cin + Cout)
    x = rnd(g, Nimg, H, W, Cin)
    w = rnd(g, Cout, 3, 3, Cin, scale=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    rb = torch.randn(Nimg, Cout, device="cuda", generator=g)
    res = rnd(g, Nimg, H, W, Cout)
    cv = Canvas(Nimg * H * W * Cout)
    y = cv.view((Nimg, H, W, Cout), (H * W * Cout, W * Cout, Cout, 1))
    ws = torch.full((2048 * 2560,), float("nan"), device="cuda") if splitk else None
    plan = (C.c_int * 2)(0, 0)
    wsp, wsb = (C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel() * 4)) if splitk else (C.c_void_p(0), C.c_size_t(0))
    sync_check(L, L.lib().mi3d_op_conv3(L.ptr(x), L.ptr(w), L.ptr(y), Nimg, H, W, Cin, Cout, L.ptr(bias), L.ptr(rb), L.ptr(res), wsp, wsb,
                                        plan, L.stream()), "op_conv3")
    print(f"planned block_n {plan[0]}, splits {plan[1]}")
    if sms == 132:
        assert (plan[0], plan[1]) == want
    if splitk and H == 8:
        assert plan[1] > 1, "the deepest SD level must reach k_splitk_finish (bias, per-image row_bias, residual)"
    acc, absacc = conv_ref(x, w)
    rbr = rb.double()[:, None, None, :]
    ref = acc + bias.double() + rbr + res.double()
    e = acc_bound(9 * Cin, absacc, 1.0, bias.double().expand_as(acc), rbr.expand_as(acc), res.double())
    check(f"conv3 {Nimg}x{H}x{W}x{Cin}->{Cout}", y, ref, f16_round(ref, e))
    cv.check_untouched("conv3")


CONV_BLOCK_CASES = [
    (1, 1, 1, 64, 64, "plain"), (2, 1, 1, 256, 128, "relu_bwd"), (1, 7, 9, 64, 128, "relu"), (2, 7, 9, 256, 64, "plain"),
    (2, 12, 12, 64, 256, "relu_bwd"), (1, 12, 12, 256, 256, "relu"), (2, 24, 24, 64, 64, "relu"), (1, 24, 24, 256, 128, "relu_bwd"),
    (1, 33, 47, 64, 256, "plain"), (2, 33, 47, 256, 128, "relu"), (2, 50, 50, 64, 128, "relu_bwd"), (1, 50, 50, 256, 64, "plain"),
    (1, 100, 75, 256, 256, "relu_bwd"), (2, 100, 75, 64, 64, "plain"), (2, 100, 75, 64, 256, "relu"), (2, 100, 75, 64, 320, "relu"),
]


@pytest.mark.parametrize("Nimg,H,W,Cin,Cout,mode", CONV_BLOCK_CASES)
def test_conv3_block_matches_fp64(L, Nimg, H, W, Cin, Cout, mode):
    """Builder::conv3_block (VGG / DPT): any H x W, tiles overhang the right and bottom edges and store only in-image pixels.
    PLAIN + bias + residual, RELU, and RELU_BWD whose aux (the mask source, torch's x > 0) holds exact zeros, -0.0 and negatives.
    Bound: 2 K u conv(|x|, |w|) + epilogue ulps + one fp16 rounding (ReLU is 1-Lipschitz, the mask exact)."""
    g = torch.Generator(device="cuda").manual_seed(H * W + Cin + Cout + len(mode))
    x = rnd(g, Nimg, H, W, Cin)
    w = rnd(g, Cout, 3, 3, Cin, scale=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout, device="cuda", generator=g) if mode != "relu_bwd" else None
    res = rnd(g, Nimg, H, W, Cout) if mode == "plain" else None
    aux = None
    if mode == "relu_bwd":
        aux = rnd(g, Nimg, H, W, Cout)
        pick = torch.randint(0, 4, aux.shape, device="cuda", generator=g)
        aux[pick == 0] = 0.0
        aux[pick == 1] = -0.0
    cv = Canvas(Nimg * H * W * Cout)
    y = cv.view((Nimg, H, W, Cout), (H * W * Cout, W * Cout, Cout, 1))
    plan = (C.c_int * 2)(0, 0)
    sync_check(L, L.lib().mi3d_op_conv3_block(L.ptr(x), L.ptr(w), L.ptr(y), Nimg, H, W, Cin, Cout, L.ptr(bias), EPI[mode], L.ptr(aux),
                                              L.ptr(res), plan, L.stream()), "op_conv3_block")
    print(f"planned block_n {plan[0]}")
    acc, absacc = conv_ref(x, w)
    terms = []
    if bias is not None:
        acc = acc + bias.double(); terms.append(bias.double().expand_as(acc))
    if res is not None:
        acc = acc + res.double(); terms.append(res.double())
    e = acc_bound(9 * Cin, absacc, 1.0, *terms)
    if mode == "relu":
        ref = acc.clamp_min(0)
    elif mode == "relu_bwd":
        m = (aux > 0).double()
        ref, e = acc * m, e * m
    else:
        ref = acc
    check(f"conv3_block {mode} {Nimg}x{H}x{W}x{Cin}->{Cout}", y, ref, f16_round(ref, e))
    cv.check_untouched("conv3_block")


# ------------------------------------------------------------------------------------------------------------------------------
# attention on the packed qkv of a transformer block
# ------------------------------------------------------------------------------------------------------------------------------
def run_attention(L, qkv, B, T, Tpad, heads, mode):
    Cm = 64 * heads
    cv = Canvas(B * Tpad * Cm)
    o = cv.view((B * Tpad, Cm), (Cm, 1))
    qkvT = torch.empty(B, 3 * Cm, Tpad, dtype=torch.float16, device="cuda")
    S = torch.empty(B * heads, Tpad, Tpad, dtype=torch.float16, device="cuda")
    sync_check(L, L.lib().mi3d_op_attention(L.ptr(qkv), L.ptr(qkvT), L.ptr(S), L.ptr(o), B, T, Tpad, heads, mode, L.stream()), "op_attention")
    cv.check_untouched(f"attention mode {mode}")
    return o, S


@pytest.mark.parametrize("B,heads", [(1, 1), (2, 12)])
@pytest.mark.parametrize("T,Tpad", [(77, 128), (197, 256), (257, 320), (577, 640)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_attention_on_packed_qkv_matches_fp64(L, mode, T, Tpad, B, heads):
    """Attention of a transformer block on qkv [B*Tpad][3C] (q, k, v at column offsets 0, C, 2C, ld = 3C), keys < T (and j <= q when
    causal): mode 0 the fused kernel (attention_core as block_fwd calls it), 1 / 2 attention_materialised (causal for 2), which also
    leaves P.  Reference: fp64 softmax(q k^T / 8) over the valid keys, times v, for every query row.
    Bound per key term: a logit error sigma (fp32 dot of 64 products; in modes 1, 2 also the fp16 store of S) moves p_j by
    p_j (sigma_j + sum_i p_i sigma_i); plus __expf / ex2 ulps and the fp32 row sums; P is rounded to fp16 before the PV product
    (2^-11 p_j + 2^-25 per term), the PV product accumulates Tpad terms in fp32, and O is rounded to fp16 once.
    Padded-row contract: rows T..Tpad-1 of qkv overwritten with +-60000 must leave rows < T of O (and of P) bit-identical."""
    g = torch.Generator(device="cuda").manual_seed(T * 3 + B + heads + mode)
    Cm = 64 * heads
    qkv = rnd(g, B * Tpad, 3 * Cm)
    o, S = run_attention(L, qkv, B, T, Tpad, heads, mode)

    q = qkv.double().view(B, Tpad, 3, heads, 64).permute(2, 0, 3, 1, 4)       # [3][b][h][token][d]
    Q, K, V = q[0], q[1], q[2]
    s = Q @ K.transpose(-1, -2)
    z = s / 8.0
    valid = torch.zeros(Tpad, Tpad, dtype=torch.bool, device="cuda")
    valid[:, :T] = True
    if mode == 2:
        valid &= torch.ones(Tpad, Tpad, dtype=torch.bool, device="cuda").tril()
    P = torch.softmax(z.masked_fill(~valid, -math.inf), dim=-1)
    ref_o = P @ V
    zmax = z.masked_fill(~valid, -math.inf).amax(-1, keepdim=True)
    dot = 2 * 64 * U32 * (Q.abs() @ K.abs().transpose(-1, -2)) / 8.0
    ulp = 2.0 ** -20 + 2 * U32 * (z.abs() + zmax.abs())                          # exp / ex2 and the rounding of its argument
    sigma = dot + ulp
    if mode:
        sigma = sigma + (s.abs() * U16 + SUB16) / 8.0                             # S stored as fp16
    sigma = sigma.masked_fill(~valid, 0.0)
    ebar = (P * sigma).sum(-1, keepdim=True)
    rho = 1.01 * (sigma + ebar + ulp.masked_fill(~valid, 0).amax(-1, keepdim=True) + (Tpad / 4 + 16) * U32)
    p_err = P * rho                                                             # before P's fp16 rounding
    if mode:
        p_bound = f16_round(P, p_err).masked_fill(~valid, 0.0)
        Pk = S.view(B, heads, Tpad, Tpad).double()
        check(f"attention P mode {mode} T{T} B{B} h{heads}", Pk, P, p_bound.masked_fill(~valid, 1.0))
        assert (Pk[~valid.expand_as(Pk)] == 0).all(), "masked P entries must be exactly 0"
    else:
        p_bound = p_err + U16 * P + SUB16 * valid
    e = p_bound @ V.abs() + 2 * Tpad * U32 * (P @ V.abs())
    ref = ref_o.permute(0, 2, 1, 3).reshape(B * Tpad, Cm)
    bound = f16_round(ref, e.permute(0, 2, 1, 3).reshape(B * Tpad, Cm))
    check(f"attention O mode {mode} T{T} Tpad{Tpad} B{B} h{heads}", o, ref, bound)

    bad = qkv.clone().view(B, Tpad, 3 * Cm)
    sign = torch.randint(0, 2, bad[:, T:].shape, device="cuda", generator=g).half() * 2 - 1
    bad[:, T:] = sign * 60000.0
    o2, S2 = run_attention(L, bad.view(B * Tpad, 3 * Cm), B, T, Tpad, heads, mode)
    rows = (torch.arange(B * Tpad, device="cuda") % Tpad) < T
    assert torch.equal(o2[rows].view(torch.int16), o[rows].view(torch.int16)), "padded rows reached a valid row of O"
    if mode:
        assert torch.equal(S2[:, :T].view(torch.int16), S[:, :T].view(torch.int16)), "padded rows reached a valid row of P"


def run_attention_core(L, q, k, v, o, B, T, Tk, valid, heads):
    """Builder::attention_core at head_dim 64 as the SD engine calls it; every row stride is its tensor's width"""
    sync_check(L, L.lib().mi3d_op_attention_core(L.ptr(q), C.c_longlong(q.shape[1]), L.ptr(k), C.c_longlong(k.shape[1]), L.ptr(v),
                                                 C.c_longlong(v.shape[1]), L.ptr(o), C.c_longlong(o.shape[1]), B, T, Tk, valid, heads, 64,
                                                 L.stream()), "op_attention_core")


@pytest.mark.parametrize("B,T,Tk,valid,heads", [(2, 4096, 4096, 4096, 5), (2, 1024, 1024, 1024, 10), (2, 256, 128, 77, 20), (2, 64, 64, 64, 20),
                                                (1, 16, 16, 16, 1), (1, 384, 300, 300, 2)])
def test_flash_attention_matches_fp32_reference(L, B, T, Tk, valid, heads):
    """Builder::attention_core at head_dim 64: the fused attention (S, P and O in registers) vs torch fp32 softmax(q k^T / 8) v on
    the same fp16 inputs.  Bound: P is rounded to fp16 before the second product (2^-11 relative per term) + one fp16 rounding of the output."""
    g = torch.Generator(device="cuda").manual_seed(B * T + heads)
    C_ = heads * 64
    q = torch.randn(B * T, C_, device="cuda", generator=g).half()
    k = torch.randn(B * Tk, C_, device="cuda", generator=g).half()
    v = torch.randn(B * Tk, C_, device="cuda", generator=g).half()
    o = torch.zeros(B * T, C_, dtype=torch.float16, device="cuda")
    run_attention_core(L, q, k, v, o, B, T, Tk, valid, heads)
    qf = q.float().view(B, T, heads, 64).permute(0, 2, 1, 3)
    kf = k.float().view(B, Tk, heads, 64).permute(0, 2, 1, 3)[:, :, :valid]
    vf = v.float().view(B, Tk, heads, 64).permute(0, 2, 1, 3)[:, :, :valid]
    ref = torch.softmax(qf @ kf.transpose(-1, -2) / 8.0, dim=-1) @ vf
    ref = ref.permute(0, 2, 1, 3).reshape(B * T, C_)
    err = (o.float() - ref).abs().max().item()
    assert err < 3e-3 * max(1.0, ref.abs().max().item()), err


def test_flash_attention_lazy_rescale(L):
    """Logits that keep growing along the key axis force the online rescale (O rows in registers multiplied by alpha) in every block;
    logits that shrink never trigger it.  Both must match the fp32 reference."""
    B, T, heads, C_ = 1, 256, 2, 128
    g = torch.Generator(device="cuda").manual_seed(3)
    for sign in (+1.0, -1.0):
        q = torch.zeros(B * T, C_, device="cuda")
        q[:, 0] = 8.0; q[:, 64] = 8.0                      # every query: logit = ramp(key) (1/8 scale folded in)
        k = torch.randn(B * 1024, C_, device="cuda", generator=g) * 0.05
        ramp = sign * torch.linspace(0.0, 60.0, 1024, device="cuda")
        k[:, 0] = ramp; k[:, 64] = ramp
        v = torch.randn(B * 1024, C_, device="cuda", generator=g)
        qh, kh, vh = q.half(), k.half(), v.half()
        o = torch.zeros(B * T, C_, dtype=torch.float16, device="cuda")
        run_attention_core(L, qh, kh, vh, o, B, T, 1024, 1024, heads)
        qf = qh.float().view(B, T, heads, 64).permute(0, 2, 1, 3)
        kf = kh.float().view(B, 1024, heads, 64).permute(0, 2, 1, 3)
        vf = vh.float().view(B, 1024, heads, 64).permute(0, 2, 1, 3)
        ref = (torch.softmax(qf @ kf.transpose(-1, -2) / 8.0, dim=-1) @ vf).permute(0, 2, 1, 3).reshape(B * T, C_)
        assert torch.isfinite(o).all()
        err = (o.float() - ref).abs().max().item()
        assert err < 3e-3 * max(1.0, ref.abs().max().item()), (sign, err)


# ------------------------------------------------------------------------------------------------------------------------------
# row kernels
# ------------------------------------------------------------------------------------------------------------------------------
LN_ADVERSARIAL = 12     # the first rows of ln_rows


def ln_rows(g, rows, width):
    """LN_ADVERSARIAL adversarial rows, then random ones.  Adversarial: constant rows (var = 0) and rows with a large common offset
    relative to their spread (|mean| / std about 10, 100 and 1000); every value exactly representable in fp16 (the kernel reads fp16)"""
    x = torch.randn(rows, width, device="cuda", generator=g) * 2 + 0.5
    k = 0
    for val in (0.0, 3.140625, -1000.0):
        x[k] = val; k += 1
    for ratio in (10, 100, 1000):
        for mu in (1.0, -16.0, 1000.0):
            x[k] = mu + (abs(mu) / ratio) * torch.randn(width, device="cuda", generator=g); k += 1
    assert k == LN_ADVERSARIAL
    return x.half()


def ln_lane_terms(width):
    return 8 * ((width + 255) // 256)     # one lane's serial terms (8 per 16-byte load), then a 5-level shuffle tree


def ln_stats(x, width, eps):
    """fp64 mean, deviation, rstd, and per row the bounds on the kernel's mean error (e_mu) and relative rstd error (rho), for the
    branch sdk::row_stats takes on that row (n = ln_lane_terms):
      mean: the fp32 row sum and the division, e_mu = (n + 6) u mean|x|;
      one pass (mean^2 <= E[x^2] / 4): var = E[x^2] - mean^2, error (n + 8) u E[x^2] + 2 |mean| e_mu + e_mu^2;
      two pass (every other row): var = (sum d^2 - (sum d)^2 / C) / C over the deviations d = x - mean, error
        (n + 10) u (var + e_mu^2) + 2 (n + 6) u e_mu std + e_mu^2 (the (sum d)^2 term removes the mean's error to first order);
      a row within 0.1 % of the threshold may take either branch and gets the larger bound;
      rstd: half the relative var error, + (var + eps) rounding and rsqrtf's 2 ulp."""
    n = ln_lane_terms(width)
    X = x.double()
    mu = X.mean(-1, keepdim=True)
    d = X - mu
    var = (d * d).mean(-1, keepdim=True)
    ex2 = (X * X).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    e_mu = (n + 6) * U32 * X.abs().mean(-1, keepdim=True)
    e_one = (n + 8) * U32 * ex2 + 2 * mu.abs() * e_mu + e_mu ** 2
    e_two = (n + 10) * U32 * (var + e_mu ** 2) + 2 * (n + 6) * U32 * e_mu * var.sqrt() + e_mu ** 2
    q = (mu * mu) / ex2.clamp_min(1e-300)
    e_var = torch.where(q < 0.25 * (1 - 1e-3), e_one, torch.where(q > 0.25 * (1 + 1e-3), e_two, torch.maximum(e_one, e_two)))
    rho = 0.51 * e_var / (var + eps) + 2.0 ** -21
    return d, r, e_mu, rho


@pytest.mark.parametrize("width", [64, 768, 1024, 1408, 2560])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_layernorm_forward_matches_fp64(L, width, eps):
    """Builder::layernorm (sdk::k_layernorm, one warp per row), 77 rows with the adversarial rows of ln_rows.
    Bound: |gamma| r (e_mu + |x - mean| (rho + 3 u)) + u |y| (fp32 arithmetic) + one fp16 rounding; see ln_stats."""
    g = torch.Generator(device="cuda").manual_seed(width + int(eps * 1e7))
    rows = 77
    x = ln_rows(g, rows, width)
    gamma = torch.randn(width, device="cuda", generator=g)
    beta = torch.randn(width, device="cuda", generator=g)
    cv = Canvas((rows + 5) * width)
    y = cv.view((rows, width), (width, 1))
    sync_check(L, L.lib().mi3d_op_layernorm(L.ptr(x), L.ptr(y), L.ptr(gamma), L.ptr(beta), rows, width, C.c_float(eps), L.stream()), "op_layernorm")
    d, r, e_mu, rho = ln_stats(x, width, eps)
    G, Bt = gamma.double(), beta.double()
    core = d * r * G
    ref = core + Bt
    err = 1.01 * G.abs() * r * (e_mu + d.abs() * (rho + 3 * U32)) + U32 * (core.abs() + Bt.abs())
    bound = f16_round(ref, err)
    check(f"layernorm width{width} eps{eps} adversarial rows", y[:LN_ADVERSARIAL], ref[:LN_ADVERSARIAL], bound[:LN_ADVERSARIAL])
    check(f"layernorm width{width} eps{eps}", y, ref, bound)
    cv.check_untouched("layernorm")


@pytest.mark.parametrize("width", [64, 768, 1024, 1408, 2560])
@pytest.mark.parametrize("add", [False, True])
def test_layernorm_backward_matches_fp64(L, width, add):
    """clipk::k_layernorm_bwd: dx = r (g - mean(g) - xhat mean(g xhat)) (+ add), g = dy gamma, statistics recomputed from x, on the
    rows of ln_rows.  Bound: the kernel's r (rho), xhat (r e_mu + |xhat| (rho + 2u)) and fp32 row means ((n + 8) u of their
    magnitudes) carried through the formula, + u |add| + one fp16 rounding."""
    g = torch.Generator(device="cuda").manual_seed(width + 2 * add)
    rows, eps = 93, 1e-5
    x = ln_rows(g, rows, width)
    dy = rnd(g, rows, width)
    gamma = torch.randn(width, device="cuda", generator=g)
    ad = rnd(g, rows, width) if add else None
    cv = Canvas((rows + 5) * width)
    dx = cv.view((rows, width), (width, 1))
    sync_check(L, L.lib().mi3d_op_layernorm_bwd(L.ptr(x), L.ptr(dy), L.ptr(gamma), L.ptr(ad), L.ptr(dx), rows, width, C.c_float(eps), L.stream()),
               "op_layernorm_bwd")
    n = ln_lane_terms(width)
    d, r, e_mu, rho = ln_stats(x, width, eps)
    xh = d * r
    gg = dy.double() * gamma.double()
    g1 = gg.mean(-1, keepdim=True)
    g2 = (gg * xh).mean(-1, keepdim=True)
    h = gg - g1 - xh * g2
    ref = r * h + (ad.double() if add else 0.0)
    e_xh = r * e_mu + xh.abs() * (rho + 2 * U32)
    e_g1 = (n + 6) * U32 * gg.abs().mean(-1, keepdim=True)
    e_g2 = (gg.abs() * e_xh).mean(-1, keepdim=True) + (n + 8) * U32 * (gg * xh).abs().mean(-1, keepdim=True)
    e_h = U32 * gg.abs() + e_g1 + xh.abs() * e_g2 + g2.abs() * e_xh + 3 * U32 * (gg.abs() + g1.abs() + (xh * g2).abs())
    err = 1.01 * ((r * h).abs() * rho + r * e_h) + U32 * ((r * h).abs() + (ad.double().abs() if add else 0.0))
    bound = f16_round(ref, err)
    check(f"layernorm_bwd width{width} add{add} adversarial rows", dx[:LN_ADVERSARIAL], ref[:LN_ADVERSARIAL], bound[:LN_ADVERSARIAL])
    check(f"layernorm_bwd width{width} add{add}", dx, ref, bound)
    cv.check_untouched("layernorm_bwd")


@pytest.mark.parametrize("cols,valid", [(64, 50), (128, 77), (320, 257), (640, 577), (640, 640)])
@pytest.mark.parametrize("causal", [False, True])
def test_softmax_matches_fp64(L, cols, valid, causal):
    """Builder::softmax (in place, columns >= valid written as 0) and clipk::k_softmax_causal (row r keeps keys j <= r % tq and
    j < valid) over [3][tq = cols][cols] scores.  Bound: p (2 max|exp ulps| + (n + 8) u) + one fp16 rounding, exp ulps =
    2^-21 + 2u |argument|; masked entries exactly 0."""
    g = torch.Generator(device="cuda").manual_seed(cols + valid + causal)
    Z, scale = 3, 0.125
    rows = Z * cols
    x = rnd(g, rows, cols, scale=6.0)
    cv = Canvas((rows + 3) * cols)
    s = cv.view((rows, cols), (cols, 1))
    s.copy_(x)
    sync_check(L, L.lib().mi3d_op_softmax(L.ptr(s), C.c_size_t(rows), cols, valid, cols if causal else 0, C.c_float(scale), L.stream()), "op_softmax")
    keep = torch.zeros(rows, cols, dtype=torch.bool, device="cuda")
    keep[:, :valid] = True
    if causal:
        q = (torch.arange(rows, device="cuda") % cols)[:, None]
        keep &= torch.arange(cols, device="cuda")[None, :] <= q
    zz = (x.double() * scale).masked_fill(~keep, -math.inf)
    ref = torch.softmax(zz, -1)
    zm = zz.amax(-1, keepdim=True)
    ulp = 2.0 ** -21 + 2 * U32 * ((x.double() * scale).abs() + zm.abs())
    n = ln_lane_terms(cols)
    err = ref * (ulp + ulp.masked_fill(~keep, 0).amax(-1, keepdim=True) + (n + 8) * U32)
    check(f"softmax cols{cols} valid{valid} causal{causal}", s, ref, f16_round(ref, err).masked_fill(~keep, 1.0))
    assert (s[~keep] == 0).all(), "masked entries must be exactly 0"
    cv.check_untouched("softmax")


@pytest.mark.parametrize("rows,cols", [(77, 128), (1000, 320), (13, 640), (300, 64)])
def test_softmax_backward_matches_fp64(L, rows, cols):
    """sdk::k_softmax_bwd in place: ds = scale p (dp - sum(p dp)).  The products p dp are exact in fp32; the row sum has
    (n + 6) u sum|p dp|.  Bound: |scale p| (e_dot + 3 u |dp - dot|) + one fp16 rounding."""
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    p = torch.softmax(torch.randn(rows, cols, device="cuda", generator=g) * 3, -1).half()
    dp0 = rnd(g, rows, cols)
    cv = Canvas((rows + 3) * cols)
    dp = cv.view((rows, cols), (cols, 1))
    dp.copy_(dp0)
    scale = 0.125
    sync_check(L, L.lib().mi3d_op_softmax_bwd(L.ptr(p), L.ptr(dp), C.c_size_t(rows), cols, C.c_float(scale), L.stream()), "op_softmax_bwd")
    Pd, D = p.double(), dp0.double()
    dot = (Pd * D).sum(-1, keepdim=True)
    ref = scale * Pd * (D - dot)
    e_dot = (ln_lane_terms(cols) + 6) * U32 * (Pd * D).abs().sum(-1, keepdim=True)
    err = 1.01 * scale * Pd * (e_dot + 3 * U32 * (D - dot).abs())
    check(f"softmax_bwd rows{rows} cols{cols}", dp, ref, f16_round(ref, err))
    cv.check_untouched("softmax_bwd")


@pytest.mark.parametrize("R", [1, 31, 33, 77, 320])
@pytest.mark.parametrize("Ccols", [1, 31, 33, 77, 320])
def test_transpose_is_exact(L, R, Ccols):
    """Builder::transpose [Z][R][C] -> [Z][C][R] with 32 x 32 tiles: bit-exact, nothing stored past the output."""
    g = torch.Generator(device="cuda").manual_seed(R * 1000 + Ccols)
    Z = 3
    x = rnd(g, Z, R, Ccols)
    cv = Canvas(Z * R * Ccols)
    out = cv.view((Z, Ccols, R), (Ccols * R, R, 1))
    sync_check(L, L.lib().mi3d_op_transpose(L.ptr(x), L.ptr(out), Z, R, Ccols, L.stream()), "op_transpose")
    assert torch.equal(out.view(torch.int16), x.transpose(1, 2).contiguous().view(torch.int16))
    cv.check_untouched("transpose")
