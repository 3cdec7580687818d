// clip_kernels.cuh -- the memory-bound kernels of the CLIP engine (clip_engine.cu) that the op layer (plan.cu) does not provide:
// image preprocessing (resize / normalise / patchify) and its input gradient, the feature-gradient scaling, the class / positional
// embedding of the image tower and the EOT-row select of the text tower.  Activations are token rows of fp16 ("tokens x C"),
// reductions are fp32, and every output element is written by exactly one thread (no atomics: run-to-run deterministic).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "warp_reduce.cuh"

namespace clipk {
namespace {

// openai CLIP's Normalize constants
__device__ __forceinline__ float norm_mean(int c) { return c == 0 ? 0.48145466f : (c == 1 ? 0.4578275f : 0.40821073f); }
__device__ __forceinline__ float norm_inv_std(int c) { return c == 0 ? 1.f / 0.26862954f : (c == 1 ? 1.f / 0.26130258f : 1.f / 0.27577711f); }

// Source coordinate of a bilinear resize, F.interpolate(mode='bilinear', align_corners=False, antialias=False)
struct Tap { int i0, i1; float l; };
__device__ __forceinline__ Tap bilinear_tap(int o, float scale, int in) {
    const float f = fmaxf((o + 0.5f) * scale - 0.5f, 0.f);
    Tap t; t.i0 = min((int)f, in - 1); t.i1 = min(t.i0 + 1, in - 1); t.l = f - t.i0;
    return t;
}

// img fp32 [B,3,H,W] -> patch rows fp16 [B * G*G][3*P*P], column (c, ky, kx), row (b, py, px), G = R / P.
// aug != 0: bilinear resize H x W -> R x R, then (x - mean) / std.  aug == 0: the image is already R x R and augmented.
// One thread per 8 consecutive kx of one (row, c, ky).
__global__ void k_preprocess(const float* __restrict__ img, int B, int H, int W, int R, int P, int aug, __half* __restrict__ out) {
    const int G = R / P, KP = 3 * P * P, vec = P / 8;
    const size_t total = (size_t)B * G * G * 3 * P * vec;
    const float sy = (float)H / R, sx = (float)W / R;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vec); size_t r = i / vec;
        const int ky = (int)(r % P); r /= P;
        const int c = (int)(r % 3); const size_t row = r / 3;
        const int px = (int)(row % G), py = (int)((row / G) % G), b = (int)(row / ((size_t)G * G));
        const int oy = py * P + ky;
        const float* ch = img + ((size_t)b * 3 + c) * H * W;
        __align__(16) __half o[8];
        if (aug) {
            const Tap ty = bilinear_tap(oy, sy, H);
            #pragma unroll
            for (int k = 0; k < 8; k++) {
                const Tap tx = bilinear_tap(px * P + v * 8 + k, sx, W);
                const float val = (1.f - ty.l) * ((1.f - tx.l) * ch[(size_t)ty.i0 * W + tx.i0] + tx.l * ch[(size_t)ty.i0 * W + tx.i1]) +
                                  ty.l * ((1.f - tx.l) * ch[(size_t)ty.i1 * W + tx.i0] + tx.l * ch[(size_t)ty.i1 * W + tx.i1]);
                o[k] = __float2half_rn((val - norm_mean(c)) * norm_inv_std(c));
            }
        } else {
            #pragma unroll
            for (int k = 0; k < 8; k++) o[k] = __float2half_rn(ch[(size_t)oy * W + px * P + v * 8 + k]);
        }
        *reinterpret_cast<uint4*>(out + row * KP + ((size_t)c * P + ky) * P + v * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// Input gradient of k_preprocess, as a gather: grad[b,c,y,x] = sum over the output pixels whose bilinear taps touch (y, x) of
// tap weight * dpatch / std, divided by the gradient scale s of k_grad_in.  dpatch fp16 [n * G*G][3*P*P]; grad fp32 [n,3,H,W] (overwritten).
__global__ void k_preprocess_bwd(const __half* __restrict__ dpatch, int n, int H, int W, int R, int P, int aug, const float* __restrict__ scale,
                                 float* __restrict__ grad) {
    const int G = R / P, KP = 3 * P * P;
    const float inv_s = 1.f / *scale;
    const size_t total = (size_t)n * 3 * H * W;
    const float sy = (float)H / R, sx = (float)W / R;
    auto at = [&](int b, int c, int oy, int ox) {
        const size_t row = ((size_t)b * G + oy / P) * G + ox / P;
        return __half2float(dpatch[row * KP + ((size_t)c * P + oy % P) * P + ox % P]);
    };
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H), c = (int)((i / ((size_t)W * H)) % 3), b = (int)(i / ((size_t)3 * W * H));
        if (!aug) { grad[i] = at(b, c, y, x) * inv_s; continue; }
        // output pixels whose source footprint can touch (x, y): source coordinate within (x - 1, x + 1)
        const int ox_lo = max(0, (int)floorf((x - 1 + 0.5f) / sx - 0.5f)), ox_hi = min(R - 1, (int)ceilf((x + 1 + 0.5f) / sx - 0.5f));
        const int oy_lo = max(0, (int)floorf((y - 1 + 0.5f) / sy - 0.5f)), oy_hi = min(R - 1, (int)ceilf((y + 1 + 0.5f) / sy - 0.5f));
        float acc = 0.f;
        for (int oy = oy_lo; oy <= oy_hi; oy++) {
            const Tap ty = bilinear_tap(oy, sy, H);
            float wy = 0.f; if (ty.i0 == y) wy += 1.f - ty.l; if (ty.i1 == y) wy += ty.l;
            if (wy == 0.f) continue;
            for (int ox = ox_lo; ox <= ox_hi; ox++) {
                const Tap tx = bilinear_tap(ox, sx, W);
                float wx = 0.f; if (tx.i0 == x) wx += 1.f - tx.l; if (tx.i1 == x) wx += tx.l;
                if (wx == 0.f) continue;
                acc += wy * wx * at(b, c, oy, ox);
            }
        }
        grad[i] = acc * norm_inv_std(c) * inv_s;
    }
}

// Feature gradient fp32 [n] -> fp16, scaled by the power of two s that brings max |g| into [128, 256); s is stored for k_preprocess_bwd.
// The input-gradient pass runs in fp16 and is linear in g: without the scale, the per-token gradients (about 1e-3 of the feature
// gradient after the attention spreads it over the tokens) fall into fp16's subnormal range.  One block.
__global__ void k_grad_in(const float* __restrict__ g, int n, __half* __restrict__ out, float* __restrict__ scale) {
    __shared__ float s_max[32];
    float m = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(g[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = threadIdx.x < (blockDim.x >> 5) ? s_max[threadIdx.x] : 0.f;
        m = warp_max(m);
        if (threadIdx.x == 0) {
            int e = 0;
            if (m > 0.f && isfinite(m)) frexpf(m, &e);
            s_max[0] = m > 0.f && isfinite(m) ? ldexpf(1.f, min(max(8 - e, -100), 100)) : 1.f;
        }
    }
    __syncthreads();
    const float s = s_max[0];
    for (int i = threadIdx.x; i < n; i += blockDim.x) out[i] = __float2half_rn(g[i] * s);
    if (threadIdx.x == 0) *scale = s;
}

// x[b*Tpad + t] = (t == 0 ? cls : patch[b*np + t - 1]) + pos[t] for t <= np; rows np+1 .. Tpad-1 are zero.  8 channels per thread.
__global__ void k_image_embed(const __half* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, __half* __restrict__ x,
                              int B, int np, int Tpad, int C) {
    const int vc = C / 8;
    const size_t total = (size_t)B * Tpad * vc;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); const size_t r = i / vc;
        const int t = (int)(r % Tpad), b = (int)(r / Tpad);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = v * 8 + k;
            float val = 0.f;
            if (t <= np) val = (t == 0 ? cls[c] : __half2float(patch[((size_t)b * np + t - 1) * C + c])) + pos[(size_t)t * C + c];
            o[k] = __float2half_rn(val);
        }
        *reinterpret_cast<uint4*>(x + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// out[b] = x[b*Tpad + argmax_t tokens[b, t]] (the first maximum, like torch.argmax): the EOT token's row.  One block per b.
__global__ void k_text_eot_rows(const long long* __restrict__ tokens, const __half* __restrict__ x, __half* __restrict__ out, int L, int Tpad, int C) {
    const int b = blockIdx.x;
    __shared__ int s_arg;
    if (threadIdx.x == 0) {
        long long best = tokens[(size_t)b * L]; int arg = 0;
        for (int t = 1; t < L; t++) { const long long v = tokens[(size_t)b * L + t]; if (v > best) { best = v; arg = t; } }
        s_arg = arg;
    }
    __syncthreads();
    const __half* src = x + ((size_t)b * Tpad + s_arg) * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) out[(size_t)b * C + c] = src[c];
}

}  // namespace
}  // namespace clipk
