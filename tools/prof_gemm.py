"""Stand-alone launches of the tensor-core tile kernel / fused attention at SD-2.0-base shapes, through the op layer (mi3d_op_gemm /
mi3d_op_attention_core: planned by the same builder methods as the SD engine, with a split-K workspace of the engine's size), for
profiler captures and quick timing.  Prints the planned (block_n, splits) and the GPU time per call (torch.profiler: every kernel
of the call, so a split GEMM includes its workspace clear and finish pass).
Usage (GPU box): python tools/prof_gemm.py [iters]"""
import ctypes as C
import importlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [  # (M, N, K, what)
    (8192, 320, 320, "level-0 attention projection"),
    (2048, 640, 640, "level-1 attention projection"),
    (8192, 2560, 320, "level-0 GEGLU up-projection (plain epilogue here)"),
    (65536, 256, 2304, "VAE 256x256 conv as GEMM"),
]
SPLITK_ELEMS = 2048 * 2560      # the SD engine's split-K workspace (sd_engine.cu)


def gpu_us(call, iters):
    """GPU time per call: the summed device time of every kernel / memset the calls launched"""
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / iters


def main():
    L = importlib.import_module("make-it-3d_b200._lib")
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    g = torch.Generator(device="cuda").manual_seed(0)
    ws = torch.empty(SPLITK_ELEMS, device="cuda")
    for M, N, K, what in SHAPES:
        a = torch.randn(M, K, device="cuda", generator=g).half()
        b = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        args = L.OpGemmArgs(a=a.data_ptr(), lda=K, a_rows=M, K=K, a_z1=1, a_z2=1, b=b.data_ptr(), ldb=K, b_rows=N, b_z1=1, b_z2=1, N=N,
                            batch=1, out16=out.data_ptr(), ldc=N, out_z1=1, rows_per_group=1, alpha=1.0)
        plan = (C.c_int * 2)(0, 0)
        call = lambda: L.check(L.lib().mi3d_op_gemm(C.byref(args), L.ptr(ws), C.c_size_t(ws.numel() * 4), plan, L.stream()), "op_gemm")
        us = gpu_us(call, iters)
        print(f"gemm {M}x{N}x{K} ({what}): block_n {plan[0]}, splits {plan[1]}: {us:.1f} us/call, "
              f"{2.0 * M * N * K / us / 1e6:.1f} TFLOP/s")
    # fused attention, level 0: B=2, T=4096, heads=5, q | k | v packed side by side as the SD engine lays them out
    B, T, H = 2, 4096, 5
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda", generator=g).half()
    o = torch.empty(B * T, H * 64, dtype=torch.float16, device="cuda")
    ld = 3 * H * 64
    col = lambda c: C.c_void_p(qkv.data_ptr() + 2 * c)
    call = lambda: L.check(L.lib().mi3d_op_attention_core(col(0), C.c_longlong(ld), col(H * 64), C.c_longlong(ld), col(2 * H * 64), C.c_longlong(ld),
                                                          L.ptr(o), C.c_longlong(H * 64), B, T, T, T, H, 64, L.stream()), "op_attention_core")
    us = gpu_us(call, iters)
    print(f"flash attention B={B} T={T} heads={H}: {us:.1f} us/call, {4.0 * B * H * T * T * 64 / us / 1e6:.1f} TFLOP/s")


if __name__ == "__main__":
    main()
