// warp_reduce.cuh -- warp-level reductions shared by the row kernels of the op layer (plan.cu) and the engines' own kernels.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ float warp_sum(float v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// LayerNorm statistics of one fp16 row of C (C % 8 == 0), one warp.  One pass gives the mean and var = E[x^2] - mean^2, which is
// accurate while mean^2 <= E[x^2] / 4 (then var >= 3/4 E[x^2]).  A row with a larger common offset would lose its variance to the
// cancellation: its variance is recomputed from the deviations d = x - mean over a second (L1-resident) read of the row, as
// (sum d^2 - (sum d)^2 / C) / C (the second term removes the rounding error of the mean).
__device__ __forceinline__ void row_stats(const __half* xr, int C, float eps, int lane, float& mean, float& rstd) {
    float s = 0.f, ss = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) { const float v = __half2float(h[k]); s += v; ss += v * v; }
    }
    s = warp_sum(s); ss = warp_sum(ss);
    mean = s / C;
    if (mean * mean <= 0.25f * (ss / C)) {               // warp-uniform: the sums are the warp's
        rstd = rsqrtf(fmaxf(ss / C - mean * mean, 0.f) + eps);
        return;
    }
    float sd = 0.f;
    ss = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) { const float d = __half2float(h[k]) - mean; sd += d; ss = fmaf(d, d, ss); }
    }
    sd = warp_sum(sd); ss = warp_sum(ss);
    rstd = rsqrtf(fmaxf(ss - sd * sd / C, 0.f) / C + eps);
}
