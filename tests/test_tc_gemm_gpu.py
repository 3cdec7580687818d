"""GPU: the wgmma/TMA tile kernel vs a plain PyTorch fp32 reference of the same op (floating-point kernel:
torch fp32 is the stated checker).  Inputs are fp16; products are exact in fp32, accumulation order differs -> the
bound is K * eps_fp32 * |a||b| plus one fp16 rounding of the output (2^-11 relative)."""
import ctypes as C
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    return importlib.import_module("make-it-3d_b200._lib")


def _gemm(L, a, b, out_f32=False, block_n=0, alpha=1.0, bias=None, residual=None, epi=0):
    M, K = a.shape
    N = b.shape[0]
    shape = (M, N // 2) if epi == 1 else ((N, M) if epi == 2 else (M, N))
    out = torch.empty(shape, dtype=torch.float32 if out_f32 else torch.float16, device="cuda")
    L.check(L.lib().mi3d_gemm_f16(L.ptr(a), L.ptr(b), L.ptr(out), C.c_int(int(out_f32)), C.c_int(M), C.c_int(N), C.c_int(K), C.c_int(block_n),
                                  C.c_float(alpha), L.ptr(bias), L.ptr(residual), C.c_int(epi), L.stream()), "gemm_f16")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("M,N,K,bn", [(128, 64, 64, 64), (128, 128, 128, 128), (256, 256, 512, 256), (1024, 320, 320, 64),
                                      (8192, 640, 1280, 128), (512, 1280, 11520, 256), (128, 2560, 64, 0), (384, 192, 4096, 64)])
def test_gemm_matches_fp32_reference(L, M, N, K, bn):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g)).half()
    b = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
    ref = a.float() @ b.float().t()
    out = _gemm(L, a, b, out_f32=True, block_n=bn)
    err = (out - ref).abs().max().item()
    assert err < 1e-3 * max(1.0, ref.abs().max().item()), err     # fp32 accumulate: observed ~1e-5
    out16 = _gemm(L, a, b, block_n=bn)
    assert (out16.float() - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,N,K,bn,splits", [(128, 1280, 11520, 128, 8), (512, 1280, 5760, 128, 3), (256, 320, 2880, 160, 5),
                                             (1024, 640, 1280, 64, 2)])
def test_gemm_split_k(L, M, N, K, bn, splits):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    b = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).half()
    ref = 0.5 * (a.float() @ b.float().t()) + bias + res.float()
    out = torch.empty(M, N, dtype=torch.float16, device="cuda")
    ws = torch.empty(M, N, dtype=torch.float32, device="cuda")
    L.check(L.lib().mi3d_gemm_f16_splitk(L.ptr(a), L.ptr(b), L.ptr(out), C.c_int(M), C.c_int(N), C.c_int(K), C.c_int(bn), C.c_int(splits),
                                         C.c_float(0.5), L.ptr(bias), L.ptr(res), L.ptr(ws), L.stream()), "gemm_f16_splitk")
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())


def test_gemm_block_n_160(L):
    g = torch.Generator(device="cuda").manual_seed(160)
    a = torch.randn(2048, 640, device="cuda", generator=g).half()
    b = (torch.randn(320, 640, device="cuda", generator=g) / 640 ** 0.5).half()
    ref = a.float() @ b.float().t()
    out = _gemm(L, a, b, out_f32=True, block_n=160)
    assert (out - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())


def test_gemm_epilogues(L):
    g = torch.Generator(device="cuda").manual_seed(5)
    M, N, K = 256, 256, 192
    a = torch.randn(M, K, device="cuda", generator=g).half()
    b = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).half()
    ref = 0.5 * (a.float() @ b.float().t()) + bias + res.float()
    out = _gemm(L, a, b, out_f32=True, alpha=0.5, bias=bias, residual=res, block_n=128)
    assert (out - ref).abs().max().item() < 1e-3
    # GEGLU: B rows interleaved (value, gate) -> out[:, j] = value_j * gelu(gate_j)
    full = a.float() @ b.float().t() + bias
    val, gate = full[:, 0::2], full[:, 1::2]
    ref_g = val * torch.nn.functional.gelu(gate)
    out_g = _gemm(L, a, b, bias=bias, epi=1, block_n=64)
    assert (out_g.float() - ref_g).abs().max().item() < 4e-3
    # transposed store
    out_t = _gemm(L, a, b, epi=2, block_n=64)
    assert (out_t.float() - (a.float() @ b.float().t()).t()).abs().max().item() < 4e-3


@pytest.mark.parametrize("Nimg,H,W,Cin,Cout", [(2, 8, 8, 64, 64), (2, 16, 16, 128, 128), (2, 64, 64, 320, 320), (1, 128, 128, 128, 256),
                                               (2, 32, 32, 640, 1280), (1, 256, 256, 64, 64)])
def test_implicit_conv3x3_matches_fp32_reference(L, Nimg, H, W, Cin, Cout):
    g = torch.Generator(device="cuda").manual_seed(H + Cin)
    x = torch.randn(Nimg, H, W, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / (9 * Cin) ** 0.5).half()
    bias = torch.randn(Cout, device="cuda", generator=g)
    y = torch.empty(Nimg, H, W, Cout, dtype=torch.float16, device="cuda")
    L.check(L.lib().mi3d_conv3x3_f16(L.ptr(x), L.ptr(w), L.ptr(y), C.c_int(Nimg), C.c_int(H), C.c_int(W), C.c_int(Cin), C.c_int(Cout),
                                     C.c_int(0), L.ptr(bias), C.c_void_p(0), L.stream()), "conv3x3_f16")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    err = (y.float() - ref).abs().max().item()
    assert err < 4e-3 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("N,K", [(64, 32), (64, 64), (32, 64), (16, 64), (64, 128), (32, 128)])
def test_tf32_split_tiles(L, N, K):
    """Hand-written wgmma tf32 tiles of the field FORWARD kernel (K-major operands): the 3-term split must be fp32-class.
    (tf32 wgmma reads K-major operands only, which is why the backward uses bf16 tiles.)"""
    g = torch.Generator(device="cuda").manual_seed(N + K)
    a = torch.randn(128, K, device="cuda", generator=g); b = torch.randn(N, K, device="cuda", generator=g); ref = a.double() @ b.double().t()
    d = torch.empty(128, N, device="cuda")
    L.check(L.lib().mi3d_tf32_tile_test(L.ptr(a), L.ptr(b), L.ptr(d), C.c_int(N), C.c_int(K), C.c_int(0), L.stream()), "tf32_tile_test")
    torch.cuda.synchronize()
    err = (d.double() - ref).abs().max().item()
    assert err < 2e-5 * max(1.0, ref.abs().max().item()), (N, K, err)     # plain tf32 would be ~1e-2


@pytest.mark.parametrize("M,N,K,bn", [(128, 64, 64, 64), (128, 64, 256, 64), (256, 128, 128, 128), (128, 256, 64, 256), (1024, 64, 512, 64)])
def test_gemm_mn_major_b_operand(L, M, N, K, bn):
    """16-bit MN-major B operand (B given as [K][N]): the descriptor form the field backward relies on for dgrad / wgrad."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    bt = (torch.randn(K, N, device="cuda", generator=g) / K ** 0.5).half()
    out = torch.zeros(M, N, device="cuda")
    L.check(L.lib().mi3d_gemm_f16_bt(L.ptr(a), L.ptr(bt), L.ptr(out), C.c_int(M), C.c_int(N), C.c_int(K), C.c_int(bn), L.stream()), "gemm_f16_bt")
    torch.cuda.synchronize()
    ref = a.float() @ bt.float()
    assert (out - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("B,T,Tk,valid,heads", [(2, 4096, 4096, 4096, 5), (2, 1024, 1024, 1024, 10), (2, 256, 128, 77, 20), (2, 64, 64, 64, 20),
                                                (1, 16, 16, 16, 1), (1, 384, 300, 300, 2)])
def test_flash_attention_matches_fp32_reference(L, B, T, Tk, valid, heads):
    """Fused attention (S, P and O in registers) vs torch fp32 softmax(q k^T / 8) v on the same fp16 inputs.
    Bound: P is rounded to fp16 before the second product (2^-11 relative per term) + one fp16 rounding of the output."""
    g = torch.Generator(device="cuda").manual_seed(B * T + heads)
    C_ = heads * 64
    q = torch.randn(B * T, C_, device="cuda", generator=g).half()
    k = torch.randn(B * Tk, C_, device="cuda", generator=g).half()
    v = torch.randn(B * Tk, C_, device="cuda", generator=g).half()
    o = torch.zeros(B * T, C_, dtype=torch.float16, device="cuda")
    L.check(L.lib().mi3d_flash_attn_f16(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(o), C.c_int(B), C.c_int(T), C.c_int(Tk), C.c_int(valid), C.c_int(heads),
                                        C.c_int(C_), C.c_int(C_), C.c_int(C_), C.c_int(C_), L.stream()), "flash_attn")
    torch.cuda.synchronize()
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
        L.check(L.lib().mi3d_flash_attn_f16(L.ptr(qh), L.ptr(kh), L.ptr(vh), L.ptr(o), C.c_int(B), C.c_int(T), C.c_int(1024), C.c_int(1024), C.c_int(heads),
                                            C.c_int(C_), C.c_int(C_), C.c_int(C_), C.c_int(C_), L.stream()), "flash_attn")
        torch.cuda.synchronize()
        qf = qh.float().view(B, T, heads, 64).permute(0, 2, 1, 3)
        kf = kh.float().view(B, 1024, heads, 64).permute(0, 2, 1, 3)
        vf = vh.float().view(B, 1024, heads, 64).permute(0, 2, 1, 3)
        ref = (torch.softmax(qf @ kf.transpose(-1, -2) / 8.0, dim=-1) @ vf).permute(0, 2, 1, 3).reshape(B * T, C_)
        assert torch.isfinite(o).all()
        err = (o.float() - ref).abs().max().item()
        assert err < 3e-3 * max(1.0, ref.abs().max().item()), (sign, err)
