// sd_kernels.cuh -- the memory-bound kernels of the SD guidance path (sd_engine.cu) that the op layer (plan.cu) does not provide:
// GroupNorm, layout movers, the GEGLU weight interleave and the time-embedding MLP.  All activations are NHWC fp16 ("tokens x C"),
// statistics and reductions are fp32 (fp64 for the GroupNorm group sums).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "warp_reduce.cuh"

namespace sdk {
namespace {

__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }
__device__ __forceinline__ float silu_grad(float x) { const float s = 1.f / (1.f + __expf(-x)); return s * (1.f + x * (1.f - s)); }

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
// pivot (nullable): the sums were taken of x - k with k = pivot[c] per channel; lane q's cnt terms give back, in fp64,
// sum x = s + cnt k and sum x^2 = ss + 2 k s + cnt k^2.  p0, p1: the CTA's pixel range.
// Dynamic shared memory: 2 * PL * C floats + 2 * G * PL doubles (gn_smem_bytes).
__device__ __forceinline__ void gn_fold(const float* sm, int C, int G, int cpg, int PL, const __half* __restrict__ pivot, int p0, int p1,
                                        double* __restrict__ out) {
    double* part = reinterpret_cast<double*>(const_cast<float*>(sm) + (((size_t)2 * PL * C + 1) & ~(size_t)1));
    for (int t = threadIdx.x; t < G * PL; t += blockDim.x) {
        const int g = t / PL, q = t - g * PL;
        const double cnt = p1 - p0 > q ? (p1 - p0 - q + PL - 1) / PL : 0;
        double a = 0, b = 0;
        for (int c = g * cpg; c < (g + 1) * cpg; c++) {
            double s = sm[2 * (q * C + c)], ss = sm[2 * (q * C + c) + 1];
            if (pivot) { const double k = __half2float(pivot[c]); ss += k * (2 * s + cnt * k); s += cnt * k; }
            a += s; b += ss;
        }
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

// Launch geometry of the four GroupNorm kernels over N images of HW pixels, C channels in G groups: PL = max(1, 256 / VPP) pixel lanes of
// VPP = C / 8 channel vectors per CTA, and per image `chunks` CTAs of ppc pixels each -- enough CTAs to fill the machine twice, at least
// PL * 8 pixels each (more CTAs would only add partial sums to fold).  False for a shape the kernels cannot take.
struct GnGrid { int chunks = 0, ppc = 0, PL = 0, threads = 0; };
inline bool gn_grid(int N, int HW, int C, int G, int num_sms, GnGrid* q) {
    if (N < 1 || HW < 1 || G < 1 || G > 64 || C % 8 || C % G) return false;
    const int VPP = C / 8;
    q->PL = std::max(1, 256 / VPP); q->threads = q->PL * VPP;
    if (q->threads > 1024) return false;
    const int chunks = std::max(1, std::min((HW + q->PL * 8 - 1) / (q->PL * 8), (2 * num_sms + N - 1) / N));
    q->ppc = (HW + chunks - 1) / chunks; q->chunks = (HW + q->ppc - 1) / q->ppc;
    return true;
}

// Statistics of x - k, k = the image's pixel 0 per channel (a shift by a value of the data): the fp32 sums then carry the rounding of
// terms of the size of the group's spread, not of its mean, and E[x^2] - mean^2 does not cancel away the variance of groups whose |mean|
// is large against their standard deviation.  gn_fold adds the shift back in fp64.
__global__ void k_gn_stats(const __half* __restrict__ x, int HW, int C, int G, int pix_per_cta, double* __restrict__ stats /*[N][G][2]*/) {
    extern __shared__ float sm[];                 // [PL][C][2]: one slot per thread, folded in a FIXED order (run-to-run deterministic)
    const int n = blockIdx.y, cpg = C / G, VPP = C / 8, PL = blockDim.x / VPP;
    const int pl = threadIdx.x / VPP, cv = threadIdx.x % VPP;
    const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
    const __half* img = x + ((size_t)n * HW) * C;
    float s[8], ss[8];
    #pragma unroll
    for (int k = 0; k < 8; k++) { s[k] = 0.f; ss[k] = 0.f; }
    if (pl < PL) {
        const __half* base = img + (size_t)cv * 8;
        float piv[8];
        {
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(base));
            const __half* h = reinterpret_cast<const __half*>(&raw);
            #pragma unroll
            for (int k = 0; k < 8; k++) piv[k] = __half2float(h[k]);
        }
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
                for (int k = 0; k < 8; k++) { const float v = __half2float(h[k]) - piv[k]; s[k] += v; ss[k] = fmaf(v, v, ss[k]); }
            }
        }
        for (; p < p1; p += PL) {
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(base + (size_t)p * C));
            const __half* h = reinterpret_cast<const __half*>(&raw);
            #pragma unroll
            for (int k = 0; k < 8; k++) { const float v = __half2float(h[k]) - piv[k]; s[k] += v; ss[k] = fmaf(v, v, ss[k]); }
        }
        #pragma unroll
        for (int k = 0; k < 8; k++) { sm[2 * (pl * C + cv * 8 + k)] = s[k]; sm[2 * (pl * C + cv * 8 + k) + 1] = ss[k]; }
    }
    __syncthreads();
    gn_fold(sm, C, G, cpg, PL, img, p0, p1, stats + (size_t)n * G * 2);
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
    gn_fold(sm, C, G, cpg, PL, nullptr, 0, 0, bstats + (size_t)n * G * 2);
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

// y = GroupNorm(+SiLU)(x): statistics into the zeroed stats [N][G][2], then the normalisation
inline int gn_forward(const GnGrid& q, const __half* x, __half* y, double* stats, const float* gamma, const float* beta, int N, int HW, int C,
                      int G, float eps, int do_silu, cudaStream_t st) {
    k_gn_stats<<<dim3(q.chunks, N), q.threads, gn_smem_bytes(q.PL, C, G), st>>>(x, HW, C, G, q.ppc, stats);
    k_gn_apply<<<dim3(q.chunks, N), q.threads, 0, st>>>(x, y, stats, gamma, beta, HW, C, G, eps, do_silu, q.ppc);
    return (int)cudaGetLastError();
}
// dx = GroupNorm(+SiLU) input gradient of dy (+ add): the forward's stats, the gradient sums into the zeroed bstats [N][G][2]
inline int gn_backward(const GnGrid& q, const __half* x, const __half* dy, const double* stats, double* bstats, const float* gamma,
                       const float* beta, const __half* add, __half* dx, int N, int HW, int C, int G, float eps, int do_silu, cudaStream_t st) {
    k_gn_bwd_stats<<<dim3(q.chunks, N), q.threads, gn_smem_bytes(q.PL, C, G), st>>>(x, dy, stats, gamma, beta, HW, C, G, eps, do_silu, q.ppc, bstats);
    k_gn_bwd_apply<<<dim3(q.chunks, N), q.threads, 0, st>>>(x, dy, stats, bstats, gamma, beta, HW, C, G, eps, do_silu, add, dx, q.ppc);
    return (int)cudaGetLastError();
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
// col2im (gather form) for the 3x3 stride-2 conv of Builder::conv3_s2: dx[n,h,w,c] = sum over (tap, ho, wo) with 2*ho + ky - pad == h ... of dcol[(n,ho,wo)][tap][c]
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

// y[b][n] = bias[n] + sum_k act(x[b][k]) * W[n][k]  (time embedding MLP and per-ResBlock temb projections; B = the U-Net batch, 2G)
// One warp per output n.  The rows are taken in blocks of 8, each with its accumulators in registers (fully unrolled over the block, so
// the row index is a constant); a block's rows keep the k order of the lanes' FMA chains and the warp tree whatever B is.
__global__ void k_linear_small(const float* __restrict__ x, const __half* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                               int B, int N, int K, int silu_in, int silu_out) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= N) return;
    for (int b0 = 0; b0 < B; b0 += 8) {
        const int nb = min(8, B - b0);
        const float* xb = x + (size_t)b0 * K;
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int k = lane * 8; k < K; k += 256) {
            const uint4 rw = *reinterpret_cast<const uint4*>(w + (size_t)n * K + k);
            const __half* hw = reinterpret_cast<const __half*>(&rw);
            #pragma unroll
            for (int b = 0; b < 8; b++) {
                if (b >= nb) break;
                #pragma unroll
                for (int j = 0; j < 8; j++) { float v = xb[(size_t)b * K + k + j]; if (silu_in) v = silu(v); acc[b] = fmaf(v, __half2float(hw[j]), acc[b]); }
            }
        }
        #pragma unroll
        for (int b = 0; b < 8; b++) {
            if (b >= nb) break;
            float v = warp_sum(acc[b]);
            if (lane == 0) { v += bias ? bias[n] : 0.f; if (silu_out) v = silu(v); y[(size_t)(b0 + b) * N + n] = v; }
        }
    }
}

// the same for a table of layers sharing the input x (SiLU applied to x): blockIdx.y = layer
struct SmallLinearJob { const __half* w; const float* bias; float* y; int N; };
__global__ void k_linear_small_grouped(const float* __restrict__ x, const SmallLinearJob* __restrict__ jobs, int B, int K) {
    const SmallLinearJob jb = jobs[blockIdx.y];
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= jb.N) return;
    for (int b0 = 0; b0 < B; b0 += 8) {
        const int nb = min(8, B - b0);
        const float* xb = x + (size_t)b0 * K;
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int k = lane * 8; k < K; k += 256) {
            const uint4 rw = *reinterpret_cast<const uint4*>(jb.w + (size_t)n * K + k);
            const __half* hw = reinterpret_cast<const __half*>(&rw);
            #pragma unroll
            for (int b = 0; b < 8; b++) {
                if (b >= nb) break;
                #pragma unroll
                for (int j = 0; j < 8; j++) acc[b] = fmaf(silu(xb[(size_t)b * K + k + j]), __half2float(hw[j]), acc[b]);
            }
        }
        #pragma unroll
        for (int b = 0; b < 8; b++) {
            if (b >= nb) break;
            const float v = warp_sum(acc[b]);
            if (lane == 0) jb.y[(size_t)(b0 + b) * jb.N + n] = v + (jb.bias ? jb.bias[n] : 0.f);
        }
    }
}

// one warp per output feature, 8 features per CTA; the grouped form: one grid row per layer of the job table, max_n the widest layer
inline int linear_small(const float* x, const __half* w, const float* bias, float* y, int B, int N, int K, int silu_in, int silu_out, cudaStream_t st) {
    k_linear_small<<<(N + 7) / 8, 256, 0, st>>>(x, w, bias, y, B, N, K, silu_in, silu_out);
    return (int)cudaGetLastError();
}
inline int linear_small_grouped(const float* x, const SmallLinearJob* jobs, int layers, int max_n, int B, int K, cudaStream_t st) {
    k_linear_small_grouped<<<dim3((max_n + 7) / 8, (unsigned)layers), 256, 0, st>>>(x, jobs, B, K);
    return (int)cudaGetLastError();
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
