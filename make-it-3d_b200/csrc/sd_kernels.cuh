// sd_kernels.cuh -- the memory-bound kernels around the tensor-core tiles of the SD guidance path: normalisations,
// softmax, small direct convolutions, layout movers, latent arithmetic.  All activations are NHWC fp16 ("tokens x C"),
// statistics and reductions are fp32 (fp64 for the GroupNorm group sums).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace sdk {
namespace {   // internal linkage: every engine's translation unit includes these kernels

__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }
__device__ __forceinline__ float silu_grad(float x) { const float s = 1.f / (1.f + __expf(-x)); return s * (1.f + x * (1.f - s)); }

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

// ------------------------------------------------------------------------------------------------------------
// parameter conversion (run once at load time)
// ------------------------------------------------------------------------------------------------------------
__global__ void k_f32_to_f16(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = __float2half_rn(src[i]);
}
// conv weight OIHW fp32 -> [O][ky][kx][I] fp16 ; if flip: dgrad layout [I][2-ky][2-kx][O]
__global__ void k_conv_w(const float* __restrict__ src, __half* __restrict__ dst, int O, int I, int flip) {
    const size_t n = (size_t)O * I * 9;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int kx = i % 3, ky = (i / 3) % 3, ci = (i / 9) % I, co = i / (9 * (size_t)I);
        const float v = src[i];
        if (!flip) dst[(((size_t)co * 3 + ky) * 3 + kx) * I + ci] = __float2half_rn(v);
        else dst[(((size_t)ci * 3 + (2 - ky)) * 3 + (2 - kx)) * O + co] = __float2half_rn(v);
    }
}
// linear [O][I] fp32 -> transposed [I][O] fp16
__global__ void k_transpose_w(const float* __restrict__ src, __half* __restrict__ dst, int O, int I) {
    const size_t n = (size_t)O * I;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = i % I, co = i / I;
        dst[(size_t)ci * O + co] = __float2half_rn(src[i]);
    }
}
// GEGLU proj [2*inner][I]: rows (value_j | gate_j) -> interleaved rows 2j, 2j+1 ; bias likewise (fp32)
__global__ void k_geglu_w(const float* __restrict__ w, const float* __restrict__ b, __half* __restrict__ wd, float* __restrict__ bd, int inner, int I) {
    const size_t n = (size_t)2 * inner * I;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = i % I; const int r = i / I;
        const int j = r < inner ? r : r - inner, dst_r = 2 * j + (r < inner ? 0 : 1);
        wd[(size_t)dst_r * I + ci] = __float2half_rn(w[i]);
        if (ci == 0) bd[dst_r] = b[r];
    }
}

// ------------------------------------------------------------------------------------------------------------
// GroupNorm (+ SiLU) over NHWC fp16.
// Thread mapping shared by all four kernels: blockDim = PL * VPP with VPP = C/8 channel vectors and PL pixel lanes;
// thread (pl, cv) walks pixels p0+pl, p0+pl+PL, ... of image n = blockIdx.y and always sees the SAME 8 channels, so
// per-channel partial sums live in registers; one shared-memory pass per CTA folds lanes -> channels -> groups and a
// handful of fp64 atomics per CTA fold CTAs -> stats[n][g] = (sum, sum of squares).
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void gn_group_consts(const double* __restrict__ stats, int n, int G, double cnt, float eps, float* sm_mean, float* sm_rstd) {
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        const double m = stats[((size_t)n * G + g) * 2] / cnt;
        const double var = stats[((size_t)n * G + g) * 2 + 1] / cnt - m * m;
        sm_mean[g] = (float)m;
        sm_rstd[g] = rsqrtf((float)(var > 0 ? var : 0) + eps);
    }
}

// Fold the per-thread partial sums sm[PL][C][2] of one CTA into its (group) totals and add them to out[G][2], in a FIXED order (run-to-run
// deterministic): thread (g, q) first sums the group's channels of pixel lane q, then thread g sums the PL lanes (one thread per group
// walking all cpg x PL slots serially would be a long dependent chain of double-precision adds).
// Dynamic shared memory: 2 * PL * C floats + 2 * G * PL doubles (gn_smem_bytes).
__device__ __forceinline__ void gn_fold(const float* sm, int C, int G, int cpg, int PL, double* __restrict__ out) {
    double* part = reinterpret_cast<double*>(const_cast<float*>(sm) + (((size_t)2 * PL * C + 1) & ~(size_t)1));
    for (int t = threadIdx.x; t < G * PL; t += blockDim.x) {
        const int g = t / PL, q = t - g * PL;
        double a = 0, b = 0;
        for (int c = g * cpg; c < (g + 1) * cpg; c++) { a += sm[2 * (q * C + c)]; b += sm[2 * (q * C + c) + 1]; }
        part[2 * t] = a; part[2 * t + 1] = b;
    }
    __syncthreads();
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        double a = 0, b = 0;
        for (int q = 0; q < PL; q++) { a += part[2 * (g * PL + q)]; b += part[2 * (g * PL + q) + 1]; }
        atomicAdd(&out[2 * g], a); atomicAdd(&out[2 * g + 1], b);
    }
}
inline size_t gn_smem_bytes(int PL, int C, int G) { return ((((size_t)2 * PL * C + 1) & ~(size_t)1) * sizeof(float)) + (size_t)2 * G * PL * sizeof(double); }

__global__ void k_gn_stats(const __half* __restrict__ x, int HW, int C, int G, int pix_per_cta, double* __restrict__ stats /*[N][G][2]*/) {
    extern __shared__ float sm[];                 // [PL][C][2]: one slot per thread, folded in a FIXED order (run-to-run deterministic)
    const int n = blockIdx.y, cpg = C / G, VPP = C / 8, PL = blockDim.x / VPP;
    const int pl = threadIdx.x / VPP, cv = threadIdx.x % VPP;
    const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
    float s[8], ss[8];
    #pragma unroll
    for (int k = 0; k < 8; k++) { s[k] = 0.f; ss[k] = 0.f; }
    if (pl < PL) {
        const __half* base = x + ((size_t)n * HW) * C + (size_t)cv * 8;
        // 4 independent 16-byte loads in flight per thread: with 2 CTAs x 8 warps per SM a single load per iteration leaves the
        // kernel latency-bound (Little's law); the pixel order of the sums is unchanged (still deterministic)
        int p = p0 + pl;
        for (; p + 3 * PL < p1; p += 4 * PL) {
            uint4 raw[4];
            #pragma unroll
            for (int u = 0; u < 4; u++) raw[u] = __ldg(reinterpret_cast<const uint4*>(base + (size_t)(p + u * PL) * C));
            #pragma unroll
            for (int u = 0; u < 4; u++) {
                const __half* h = reinterpret_cast<const __half*>(&raw[u]);
                #pragma unroll
                for (int k = 0; k < 8; k++) { const float v = __half2float(h[k]); s[k] += v; ss[k] = fmaf(v, v, ss[k]); }
            }
        }
        for (; p < p1; p += PL) {
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(base + (size_t)p * C));
            const __half* h = reinterpret_cast<const __half*>(&raw);
            #pragma unroll
            for (int k = 0; k < 8; k++) { const float v = __half2float(h[k]); s[k] += v; ss[k] = fmaf(v, v, ss[k]); }
        }
        #pragma unroll
        for (int k = 0; k < 8; k++) { sm[2 * (pl * C + cv * 8 + k)] = s[k]; sm[2 * (pl * C + cv * 8 + k) + 1] = ss[k]; }
    }
    __syncthreads();
    gn_fold(sm, C, G, cpg, PL, stats + (size_t)n * G * 2);
}

// y = act((x - mean) * rstd * gamma + beta); same (chunks, N) grid and thread mapping as k_gn_stats
__global__ void k_gn_apply(const __half* __restrict__ x, __half* __restrict__ y, const double* __restrict__ stats, const float* __restrict__ gamma,
                           const float* __restrict__ beta, int HW, int C, int G, float eps, int do_silu, int pix_per_cta) {
    __shared__ float sm_mean[64], sm_rstd[64];
    const int n = blockIdx.y, cpg = C / G, VPP = C / 8, PL = blockDim.x / VPP;
    gn_group_consts(stats, n, G, (double)HW * cpg, eps, sm_mean, sm_rstd);
    __syncthreads();
    const int pl = threadIdx.x / VPP, cv = threadIdx.x % VPP;
    if (pl >= PL) return;
    float a[8], b[8];
    #pragma unroll
    for (int k = 0; k < 8; k++) {
        const int c = cv * 8 + k, g = c / cpg;
        a[k] = sm_rstd[g] * gamma[c]; b[k] = beta[c] - sm_mean[g] * a[k];
    }
    const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
    const size_t base = ((size_t)n * HW) * C + (size_t)cv * 8;
    auto one = [&](const uint4& raw, int p) {
        const __half* h = reinterpret_cast<const __half*>(&raw);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            float v = fmaf(__half2float(h[k]), a[k], b[k]);
            if (do_silu) v = silu(v);
            o[k] = __float2half_rn(v);
        }
        *reinterpret_cast<uint4*>(y + base + (size_t)p * C) = *reinterpret_cast<const uint4*>(o);
    };
    int p = p0 + pl;
    for (; p + 3 * PL < p1; p += 4 * PL) {                 // 4 loads in flight per thread (see k_gn_stats)
        uint4 raw[4];
        #pragma unroll
        for (int u = 0; u < 4; u++) raw[u] = __ldg(reinterpret_cast<const uint4*>(x + base + (size_t)(p + u * PL) * C));
        #pragma unroll
        for (int u = 0; u < 4; u++) one(raw[u], p + u * PL);
    }
    for (; p < p1; p += PL) one(__ldg(reinterpret_cast<const uint4*>(x + base + (size_t)p * C)), p);
}

// GroupNorm(+SiLU) backward, pass 1: per-(n,group) sums of dg = dz*gamma and dg*xhat (dz = dy * silu'(z) when do_silu)
__global__ void k_gn_bwd_stats(const __half* __restrict__ x, const __half* __restrict__ dy, const double* __restrict__ stats,
                               const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C, int G, float eps, int do_silu,
                               int pix_per_cta, double* __restrict__ bstats /*[N][G][2]*/) {
    extern __shared__ float sm[];                 // [PL][C][2], folded in a fixed order
    __shared__ float sm_mean[64], sm_rstd[64];
    const int n = blockIdx.y, cpg = C / G, VPP = C / 8, PL = blockDim.x / VPP;
    gn_group_consts(stats, n, G, (double)HW * cpg, eps, sm_mean, sm_rstd);
    __syncthreads();
    const int pl = threadIdx.x / VPP, cv = threadIdx.x % VPP;
    if (pl < PL) {
        float mu[8], rs[8], ga[8], be[8], s1[8], s2[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = cv * 8 + k, g = c / cpg;
            mu[k] = sm_mean[g]; rs[k] = sm_rstd[g]; ga[k] = gamma[c]; be[k] = beta[c]; s1[k] = 0.f; s2[k] = 0.f;
        }
        const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
        const size_t base = ((size_t)n * HW) * C + (size_t)cv * 8;
        auto one = [&](const uint4& rx, const uint4& rd) {
            const __half* hx = reinterpret_cast<const __half*>(&rx); const __half* hd = reinterpret_cast<const __half*>(&rd);
            #pragma unroll
            for (int k = 0; k < 8; k++) {
                const float xh = (__half2float(hx[k]) - mu[k]) * rs[k];
                float d = __half2float(hd[k]);
                if (do_silu) d *= silu_grad(fmaf(xh, ga[k], be[k]));
                const float dg = d * ga[k];
                s1[k] += dg; s2[k] = fmaf(dg, xh, s2[k]);
            }
        };
        int p = p0 + pl;
        for (; p + PL < p1; p += 2 * PL) {                 // 4 loads in flight per thread
            const uint4 rx0 = __ldg(reinterpret_cast<const uint4*>(x + base + (size_t)p * C)), rd0 = __ldg(reinterpret_cast<const uint4*>(dy + base + (size_t)p * C));
            const uint4 rx1 = __ldg(reinterpret_cast<const uint4*>(x + base + (size_t)(p + PL) * C)), rd1 = __ldg(reinterpret_cast<const uint4*>(dy + base + (size_t)(p + PL) * C));
            one(rx0, rd0); one(rx1, rd1);
        }
        for (; p < p1; p += PL)
            one(__ldg(reinterpret_cast<const uint4*>(x + base + (size_t)p * C)), __ldg(reinterpret_cast<const uint4*>(dy + base + (size_t)p * C)));
        #pragma unroll
        for (int k = 0; k < 8; k++) { sm[2 * (pl * C + cv * 8 + k)] = s1[k]; sm[2 * (pl * C + cv * 8 + k) + 1] = s2[k]; }
    }
    __syncthreads();
    gn_fold(sm, C, G, cpg, PL, bstats + (size_t)n * G * 2);
}
// pass 2: dx = rstd * (dg - mean(dg) - xhat * mean(dg*xhat)) (+ add, optional accumulation of another gradient branch)
__global__ void k_gn_bwd_apply(const __half* __restrict__ x, const __half* __restrict__ dy, const double* __restrict__ stats,
                               const double* __restrict__ bstats, const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C,
                               int G, float eps, int do_silu, const __half* __restrict__ add, __half* __restrict__ dx, int pix_per_cta) {
    __shared__ float sm_mean[64], sm_rstd[64], sm_m1[64], sm_m2[64];
    const int n = blockIdx.y, cpg = C / G, VPP = C / 8, PL = blockDim.x / VPP;
    const double cnt = (double)HW * cpg;
    gn_group_consts(stats, n, G, cnt, eps, sm_mean, sm_rstd);
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        sm_m1[g] = (float)(bstats[((size_t)n * G + g) * 2] / cnt); sm_m2[g] = (float)(bstats[((size_t)n * G + g) * 2 + 1] / cnt);
    }
    __syncthreads();
    const int pl = threadIdx.x / VPP, cv = threadIdx.x % VPP;
    if (pl >= PL) return;
    float mu[8], rs[8], ga[8], be[8], m1[8], m2[8];
    #pragma unroll
    for (int k = 0; k < 8; k++) {
        const int c = cv * 8 + k, g = c / cpg;
        mu[k] = sm_mean[g]; rs[k] = sm_rstd[g]; ga[k] = gamma[c]; be[k] = beta[c]; m1[k] = sm_m1[g]; m2[k] = sm_m2[g];
    }
    const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
    const size_t base = ((size_t)n * HW) * C + (size_t)cv * 8;
    auto one = [&](const uint4& rx, const uint4& rd, const uint4& ra, int p) {
        const __half* hx = reinterpret_cast<const __half*>(&rx); const __half* hd = reinterpret_cast<const __half*>(&rd);
        const __half* ha = reinterpret_cast<const __half*>(&ra);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const float xh = (__half2float(hx[k]) - mu[k]) * rs[k];
            float d = __half2float(hd[k]);
            if (do_silu) d *= silu_grad(fmaf(xh, ga[k], be[k]));
            const float dg = d * ga[k];
            float v = rs[k] * (dg - m1[k] - xh * m2[k]);
            if (add) v += __half2float(ha[k]);
            o[k] = __float2half_rn(v);
        }
        *reinterpret_cast<uint4*>(dx + base + (size_t)p * C) = *reinterpret_cast<const uint4*>(o);
    };
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    int p = p0 + pl;
    for (; p + PL < p1; p += 2 * PL) {                     // 4-6 loads in flight per thread
        const size_t o0 = base + (size_t)p * C, o1 = base + (size_t)(p + PL) * C;
        const uint4 rx0 = __ldg(reinterpret_cast<const uint4*>(x + o0)), rd0 = __ldg(reinterpret_cast<const uint4*>(dy + o0));
        const uint4 rx1 = __ldg(reinterpret_cast<const uint4*>(x + o1)), rd1 = __ldg(reinterpret_cast<const uint4*>(dy + o1));
        const uint4 ra0 = add ? __ldg(reinterpret_cast<const uint4*>(add + o0)) : zero4, ra1 = add ? __ldg(reinterpret_cast<const uint4*>(add + o1)) : zero4;
        one(rx0, rd0, ra0, p); one(rx1, rd1, ra1, p + PL);
    }
    for (; p < p1; p += PL) {
        const size_t o0 = base + (size_t)p * C;
        one(__ldg(reinterpret_cast<const uint4*>(x + o0)), __ldg(reinterpret_cast<const uint4*>(dy + o0)), add ? __ldg(reinterpret_cast<const uint4*>(add + o0)) : zero4, p);
    }
}

// ------------------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (C), one warp per row
// ------------------------------------------------------------------------------------------------------------
__global__ void k_layernorm(const __half* __restrict__ x, __half* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                            int rows, int C, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __half* xr = x + (size_t)row * C;
    float mean, rstd;
    row_stats(xr, C, eps, lane, mean, rstd);
    __half* yr = y + (size_t)row * C;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn((__half2float(h[k]) - mean) * rstd * gamma[c + k] + beta[c + k]);
        *reinterpret_cast<uint4*>(yr + c) = *reinterpret_cast<const uint4*>(o);
    }
}

// ------------------------------------------------------------------------------------------------------------
// row softmax in place: p = softmax(scale * s[:, :valid]); columns >= valid are written as 0.  One warp per row.
// ------------------------------------------------------------------------------------------------------------
__global__ void k_softmax(__half* __restrict__ s, size_t rows, int cols, int valid, float scale) {
    const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    __half* r = s + row * cols;
    float mx = -INFINITY;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) if (c + k < valid) mx = fmaxf(mx, __half2float(h[k]) * scale);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) if (c + k < valid) sum += __expf(__half2float(h[k]) * scale - mx);
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(c + k < valid ? __expf(__half2float(h[k]) * scale - mx) * inv : 0.f);
        *reinterpret_cast<uint4*>(r + c) = *reinterpret_cast<const uint4*>(o);
    }
}
// softmax backward in place on dp: ds = scale * p * (dp - sum(dp * p))
__global__ void k_softmax_bwd(const __half* __restrict__ p, __half* __restrict__ dp, size_t rows, int cols, float scale) {
    const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __half* pr = p + row * cols; __half* dr = dp + row * cols;
    float dot = 0.f;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 a = *reinterpret_cast<const uint4*>(pr + c); const uint4 b = *reinterpret_cast<const uint4*>(dr + c);
        const __half* ha = reinterpret_cast<const __half*>(&a); const __half* hb = reinterpret_cast<const __half*>(&b);
        #pragma unroll
        for (int k = 0; k < 8; k++) dot += __half2float(ha[k]) * __half2float(hb[k]);
    }
    dot = warp_sum(dot);
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 a = *reinterpret_cast<const uint4*>(pr + c); const uint4 b = *reinterpret_cast<const uint4*>(dr + c);
        const __half* ha = reinterpret_cast<const __half*>(&a); const __half* hb = reinterpret_cast<const __half*>(&b);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(scale * __half2float(ha[k]) * (__half2float(hb[k]) - dot));
        *reinterpret_cast<uint4*>(dr + c) = *reinterpret_cast<const uint4*>(o);
    }
}

// ------------------------------------------------------------------------------------------------------------
// layout movers
// ------------------------------------------------------------------------------------------------------------
// batched 2-D transpose fp16: in [Z][R][C] -> out [Z][C][R]  (32x32 tiles through shared memory)
__global__ void k_transpose(const __half* __restrict__ in, __half* __restrict__ out, int R, int C) {
    __shared__ __half tile[32][34];
    const size_t zoff = (size_t)blockIdx.z * R * C;
    int c = blockIdx.x * 32 + threadIdx.x, r0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) if (r0 + j < R && c < C) tile[j][threadIdx.x] = in[zoff + (size_t)(r0 + j) * C + c];
    __syncthreads();
    int r = r0 + threadIdx.x, c0 = blockIdx.x * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) if (c0 + j < C && r < R) out[zoff + (size_t)(c0 + j) * R + r] = tile[threadIdx.x][j];
}
// channel concat: out[p][0:Ca] = a[p], out[p][Ca:Ca+Cb] = b[p]   (8-channel vectors)
__global__ void k_concat(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ out, size_t pixels, int Ca, int Cb) {
    const int va = Ca / 8, vb = Cb / 8, vt = va + vb;
    const size_t total = pixels * vt;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i / vt; const int v = (int)(i % vt);
        const uint4 val = v < va ? *reinterpret_cast<const uint4*>(a + (p * va + v) * 8) : *reinterpret_cast<const uint4*>(b + (p * vb + (v - va)) * 8);
        *reinterpret_cast<uint4*>(out + i * 8) = val;
    }
}
// nearest 2x upsample NHWC
__global__ void k_upsample2x(const __half* __restrict__ in, __half* __restrict__ out, int N, int H, int W, int C) {
    const int vc = C / 8;
    const size_t total = (size_t)N * 2 * H * 2 * W * vc;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); size_t p = i / vc;
        const int w = (int)(p % (2 * W)); p /= (2 * W); const int h = (int)(p % (2 * H)); const int n = (int)(p / (2 * H));
        *reinterpret_cast<uint4*>(out + i * 8) = *reinterpret_cast<const uint4*>(in + ((((size_t)n * H + h / 2) * W + w / 2) * vc + v) * 8);
    }
}
// im2col for a 3x3 stride-2 conv: in [N,H,W,C] -> col [N*Ho*Wo][9*C]; pad_lo = 1 (symmetric pad 1, U-Net) or 0 (pad (0,1,0,1), VAE)
__global__ void k_im2col_s2(const __half* __restrict__ in, __half* __restrict__ col, int N, int H, int W, int C, int Ho, int Wo, int pad_lo) {
    const int vc = C / 8;
    const size_t total = (size_t)N * Ho * Wo * 9 * vc;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); size_t r = i / vc;
        const int tap = (int)(r % 9); r /= 9;
        const int wo = (int)(r % Wo); r /= Wo; const int ho = (int)(r % Ho); const int n = (int)(r / Ho);
        const int h = 2 * ho + tap / 3 - pad_lo, w = 2 * wo + tap % 3 - pad_lo;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (h >= 0 && h < H && w >= 0 && w < W) val = *reinterpret_cast<const uint4*>(in + ((((size_t)n * H + h) * W + w) * vc + v) * 8);
        *reinterpret_cast<uint4*>(col + i * 8) = val;
    }
}
// col2im (gather form) for the same conv: dx[n,h,w,c] = sum over (tap, ho, wo) with 2*ho + ky - pad == h ... of dcol[(n,ho,wo)][tap][c]
__global__ void k_col2im_s2(const __half* __restrict__ dcol, __half* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo, int pad_lo) {
    const int vc = C / 8;
    const size_t total = (size_t)N * H * W * vc;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); size_t p = i / vc;
        const int w = (int)(p % W); p /= W; const int h = (int)(p % H); const int n = (int)(p / H);
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        #pragma unroll
        for (int ky = 0; ky < 3; ky++) {
            const int th = h + pad_lo - ky;
            if (th < 0 || (th & 1)) continue;
            const int ho = th >> 1; if (ho >= Ho) continue;
            #pragma unroll
            for (int kx = 0; kx < 3; kx++) {
                const int tw = w + pad_lo - kx;
                if (tw < 0 || (tw & 1)) continue;
                const int wo = tw >> 1; if (wo >= Wo) continue;
                const uint4 raw = *reinterpret_cast<const uint4*>(dcol + (((((size_t)n * Ho + ho) * Wo + wo) * 9 + ky * 3 + kx) * vc + v) * 8);
                const __half* hh = reinterpret_cast<const __half*>(&raw);
                #pragma unroll
                for (int k = 0; k < 8; k++) acc[k] += __half2float(hh[k]);
            }
        }
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(acc[k]);
        *reinterpret_cast<uint4*>(dx + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}
// dx[n,h,w] = sum of the 4 upsampled children (backward of nearest 2x) -- not needed by the frozen U-Net (no grad), kept out.

// out = a + b (fp16, vectors of 8)
__global__ void k_add(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ out, size_t nvec) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 ra = *reinterpret_cast<const uint4*>(a + i * 8), rb = *reinterpret_cast<const uint4*>(b + i * 8);
        const __half2* ha = reinterpret_cast<const __half2*>(&ra); const __half2* hb = reinterpret_cast<const __half2*>(&rb);
        uint4 ro; __half2* ho = reinterpret_cast<__half2*>(&ro);
        #pragma unroll
        for (int k = 0; k < 4; k++) ho[k] = __hadd2(ha[k], hb[k]);
        *reinterpret_cast<uint4*>(out + i * 8) = ro;
    }
}

// ------------------------------------------------------------------------------------------------------------
// small direct 3x3 convolutions (stride 1, pad 1), NHWC.  Used where the channel count is too small for the
// 64-wide K blocks of the tensor-core tiles: conv_in (Cin = 3 / 4), conv_out (Cout = 4 / 8) and their transposes.
// ------------------------------------------------------------------------------------------------------------
// small Cin (<= 8): thread per (pixel, 8 output channels); in fp16 [N,H,W,CIN], w fp32 [Cout][3][3][CIN] (transposed into shared
// memory as [tap][cin][Cout] so the 8 channels of a thread are two conflict-free float4 reads), out fp16 [N,H,W,Cout].
// Persistent grid (a few CTAs per SM): the weight staging is paid once per CTA, the 27/72 inputs once per 8 outputs.  Cout % 8 == 0.
template <int CIN>
__global__ void k_conv_small_cin(const __half* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias, __half* __restrict__ out,
                                 int N, int H, int W, int Cout) {
    extern __shared__ float sw[];                 // [9*CIN][Cout]
    for (int i = threadIdx.x; i < Cout * 9 * CIN; i += blockDim.x) {
        const int co = i / (9 * CIN), r = i % (9 * CIN);
        sw[r * Cout + co] = w[i];
    }
    __syncthreads();
    const int CG = Cout / 8;
    const size_t total = (size_t)N * H * W * CG;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int cg = (int)(i % CG); size_t p = i / CG;
        const int x = (int)(p % W); const size_t q = p / W; const int y = (int)(q % H); const int n = (int)(q / H);
        float acc[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = bias ? bias[cg * 8 + k] : 0.f;
        #pragma unroll
        for (int ky = 0; ky < 3; ky++) {
            const int yy = y + ky - 1; if (yy < 0 || yy >= H) continue;
            #pragma unroll
            for (int kx = 0; kx < 3; kx++) {
                const int xx = x + kx - 1; if (xx < 0 || xx >= W) continue;
                const __half* ip = in + (((size_t)n * H + yy) * W + xx) * CIN;
                float v[CIN];
                if (CIN == 8) {
                    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(ip));
                    const __half* h = reinterpret_cast<const __half*>(&raw);
                    #pragma unroll
                    for (int c = 0; c < CIN; c++) v[c] = __half2float(h[c]);
                } else {
                    const uint2 raw = __ldg(reinterpret_cast<const uint2*>(ip));
                    const __half* h = reinterpret_cast<const __half*>(&raw);
                    #pragma unroll
                    for (int c = 0; c < CIN; c++) v[c] = __half2float(h[c]);
                }
                const float* wp = sw + (size_t)((ky * 3 + kx) * CIN) * Cout + cg * 8;
                #pragma unroll
                for (int c = 0; c < CIN; c++) {
                    const float4 w0 = *reinterpret_cast<const float4*>(wp + (size_t)c * Cout), w1 = *reinterpret_cast<const float4*>(wp + (size_t)c * Cout + 4);
                    acc[0] = fmaf(v[c], w0.x, acc[0]); acc[1] = fmaf(v[c], w0.y, acc[1]); acc[2] = fmaf(v[c], w0.z, acc[2]); acc[3] = fmaf(v[c], w0.w, acc[3]);
                    acc[4] = fmaf(v[c], w1.x, acc[4]); acc[5] = fmaf(v[c], w1.y, acc[5]); acc[6] = fmaf(v[c], w1.z, acc[6]); acc[7] = fmaf(v[c], w1.w, acc[7]);
                }
            }
        }
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(acc[k]);
        *reinterpret_cast<uint4*>(out + p * Cout + cg * 8) = *reinterpret_cast<const uint4*>(o);
    }
}
// small Cout (<= 8): a group of LPP lanes per pixel (16 when Cin <= 128, else 32) splits Cin in 8-channel vectors; the fp16 weights
// [Cout][3][3][Cin] are staged in shared memory once per CTA; persistent grid-stride loop over pixels; out fp32 [N,H,W,Cout]
template <int COUT>
__global__ void k_conv_small_cout(const __half* __restrict__ in, const __half* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out,
                                  int N, int H, int W, int Cin) {
    extern __shared__ __half swh[];               // [COUT][9][Cin]
    for (int i = threadIdx.x; i < COUT * 9 * Cin / 8; i += blockDim.x) reinterpret_cast<uint4*>(swh)[i] = __ldg(reinterpret_cast<const uint4*>(w) + i);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int LPP = Cin <= 128 ? 16 : 32, sub = lane / LPP, sl = lane % LPP, ppw = 32 / LPP;
    const size_t npix = (size_t)N * H * W;
    const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5), wid = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    for (size_t base = wid * ppw; base < npix; base += warps * ppw) {
        const size_t pix = base + sub;
        const bool live = pix < npix;
        const int x = (int)(pix % W), y = (int)((pix / W) % H), n = (int)(pix / ((size_t)W * H));
        float acc[COUT];
        #pragma unroll
        for (int o = 0; o < COUT; o++) acc[o] = 0.f;
        if (live)
        for (int ky = 0; ky < 3; ky++) {
            const int yy = y + ky - 1; if (yy < 0 || yy >= H) continue;
            for (int kx = 0; kx < 3; kx++) {
                const int xx = x + kx - 1; if (xx < 0 || xx >= W) continue;
                const __half* ip = in + (((size_t)n * H + yy) * W + xx) * Cin;
                for (int c = sl * 8; c < Cin; c += LPP * 8) {
                    const uint4 ri = __ldg(reinterpret_cast<const uint4*>(ip + c));
                    const __half2* hi = reinterpret_cast<const __half2*>(&ri);
                    float2 f[4];
                    #pragma unroll
                    for (int k = 0; k < 4; k++) f[k] = __half22float2(hi[k]);
                    #pragma unroll
                    for (int o = 0; o < COUT; o++) {
                        const uint4 rw = *reinterpret_cast<const uint4*>(swh + ((size_t)(o * 9 + ky * 3 + kx)) * Cin + c);
                        const __half2* hw = reinterpret_cast<const __half2*>(&rw);
                        #pragma unroll
                        for (int k = 0; k < 4; k++) { const float2 g = __half22float2(hw[k]); acc[o] = fmaf(f[k].x, g.x, fmaf(f[k].y, g.y, acc[o])); }
                    }
                }
            }
        }
        #pragma unroll
        for (int o = 0; o < COUT; o++) {
            #pragma unroll
            for (int m = 16; m >= 1; m >>= 1) if (m < LPP) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], m);
        }
        if (live && sl == 0) {
            #pragma unroll
            for (int o = 0; o < COUT; o++) out[pix * COUT + o] = acc[o] + (bias ? bias[o] : 0.f);
        }
    }
}

// y[b][n] = bias[n] + sum_k act(x[b][k]) * W[n][k]   (B <= 8 rows; time embedding MLP and per-ResBlock temb projections)
__global__ void k_linear_small(const float* __restrict__ x, const __half* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                               int B, int N, int K, int silu_in, int silu_out) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= N) return;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = lane * 8; k < K; k += 256) {
        const uint4 rw = *reinterpret_cast<const uint4*>(w + (size_t)n * K + k);
        const __half* hw = reinterpret_cast<const __half*>(&rw);
        for (int b = 0; b < B; b++) {
            #pragma unroll
            for (int j = 0; j < 8; j++) { float v = x[(size_t)b * K + k + j]; if (silu_in) v = silu(v); acc[b] = fmaf(v, __half2float(hw[j]), acc[b]); }
        }
    }
    for (int b = 0; b < B; b++) {
        float v = warp_sum(acc[b]);
        if (lane == 0) { v += bias ? bias[n] : 0.f; if (silu_out) v = silu(v); y[(size_t)b * N + n] = v; }
    }
}

// the same for a table of layers sharing the input x (SiLU applied to x): blockIdx.y = layer
struct SmallLinearJob { const __half* w; const float* bias; float* y; int N; };
__global__ void k_linear_small_grouped(const float* __restrict__ x, const SmallLinearJob* __restrict__ jobs, int B, int K) {
    const SmallLinearJob jb = jobs[blockIdx.y];
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= jb.N) return;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = lane * 8; k < K; k += 256) {
        const uint4 rw = *reinterpret_cast<const uint4*>(jb.w + (size_t)n * K + k);
        const __half* hw = reinterpret_cast<const __half*>(&rw);
        for (int b = 0; b < B; b++) {
            #pragma unroll
            for (int j = 0; j < 8; j++) acc[b] = fmaf(silu(x[(size_t)b * K + k + j]), __half2float(hw[j]), acc[b]);
        }
    }
    for (int b = 0; b < B; b++) {
        const float v = warp_sum(acc[b]);
        if (lane == 0) jb.y[(size_t)b * jb.N + n] = v + (jb.bias ? jb.bias[n] : 0.f);
    }
}

// sinusoidal timestep embedding (diffusers Timesteps, flip_sin_to_cos=True, freq_shift=0): out[b] = [cos | sin]
__global__ void k_time_proj(const long long* __restrict__ t, float* __restrict__ out, int B, int dim) {
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, j = i % half;
    const float freq = expf(-logf(10000.f) * (float)j / (float)half);
    const float a = (float)t[0] * freq;
    out[(size_t)b * dim + j] = cosf(a);
    out[(size_t)b * dim + half + j] = sinf(a);
}

}  // namespace
}  // namespace sdk
