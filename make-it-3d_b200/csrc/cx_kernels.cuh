// cx_kernels.cuh -- the memory-bound kernels and the fp32 cosine GEMM of the contextual-loss engine (cx_engine.cu): ImageNet
// normalisation, VGG's ReLU / max-pool and their backward, and the contextual loss of S-aiueo32/contextual_loss_pytorch
// (cosine distance, band width h) with its input gradient.
//
// Precision: everything from the relu5_4 features on is fp32.  With x ~ y the row minimum of d = 1 - cos goes to 0, and an fp16
// cosine (error ~1e-4) would push min d + 1e-5 below zero.  Every output element is written by one thread and every reduction
// runs in a fixed order (no atomics), so results are bit-identical from run to run.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "warp_reduce.cuh"

namespace cxk {

constexpr float kEps = 1e-5f;          // the package's epsilon in d / (min d + eps) and -log(cx + eps)

__device__ __forceinline__ float vgg_mean(int c) { return c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f); }
__device__ __forceinline__ float vgg_std(int c) { return c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f); }

// x, y fp32 [N,3,H,W] -> out fp16 [2N,H,W,4] = (v - mean) / std, images of x first, channel 3 zero
__global__ void k_prep(const float* __restrict__ x, const float* __restrict__ y, int N, int H, int W, __half* __restrict__ out) {
    const size_t hw = (size_t)H * W, total = 2 * (size_t)N * hw;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t b = i / hw, pix = i % hw;
        const float* src = b < (size_t)N ? x + b * 3 * hw : y + (b - N) * 3 * hw;
        __align__(8) __half o[4];
        #pragma unroll
        for (int c = 0; c < 3; c++) o[c] = __float2half_rn((src[c * hw + pix] - vgg_mean(c)) / vgg_std(c));
        o[3] = __float2half_rn(0.f);
        *reinterpret_cast<uint2*>(out + i * 4) = *reinterpret_cast<const uint2*>(o);
    }
}

// in place, vectors of 8
__global__ void k_relu(__half* __restrict__ h, size_t nvec) {
    const __half2 z = __float2half2_rn(0.f);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        uint4 r = *reinterpret_cast<uint4*>(h + i * 8);
        __half2* v = reinterpret_cast<__half2*>(&r);
        #pragma unroll
        for (int k = 0; k < 4; k++) v[k] = __hmax2(v[k], z);
        *reinterpret_cast<uint4*>(h + i * 8) = r;
    }
}

// MaxPool2d(2, 2) (odd sizes floored): in [B,H,W,C] -> out [B,H/2,W/2,C], 8 channels per thread
__global__ void k_maxpool2(const __half* __restrict__ in, __half* __restrict__ out, int B, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, CV = C / 8;
    const size_t total = (size_t)B * Ho * Wo * CV;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV); size_t p = i / CV;
        const int xo = (int)(p % Wo); p /= Wo; const int yo = (int)(p % Ho); const size_t b = p / Ho;
        const __half* s = in + ((b * H + 2 * yo) * W + 2 * xo) * C + cv * 8;
        uint4 r = *reinterpret_cast<const uint4*>(s);
        __half2* m = reinterpret_cast<__half2*>(&r);
        const size_t offs[3] = {(size_t)C, (size_t)W * C, (size_t)W * C + C};
        #pragma unroll
        for (int t = 0; t < 3; t++) {
            const uint4 q = *reinterpret_cast<const uint4*>(s + offs[t]);
            const __half2* v = reinterpret_cast<const __half2*>(&q);
            #pragma unroll
            for (int k = 0; k < 4; k++) m[k] = __hmax2(m[k], v[k]);
        }
        *reinterpret_cast<uint4*>(out + i * 8) = r;
    }
}

// MaxPool2d backward fused with the ReLU mask of its input, as a gather: din[n,y,x,c] = dout[n,y/2,x/2,c] if (y, x) is its
// window's argmax (the first maximum in row-major window order, torch's rule) and a[n,y,x,c] > 0, else 0.  a: the pool's input
// (post-ReLU); rows / columns the floor drops get 0.
__global__ void k_maxpool2_bwd(const __half* __restrict__ dout, const __half* __restrict__ a, __half* __restrict__ din, int N, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, CV = C / 8;
    const size_t total = (size_t)N * H * W * CV;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV); size_t p = i / CV;
        const int x = (int)(p % W); p /= W; const int y = (int)(p % H); const size_t n = p / H;
        __align__(16) __half o[8];
        if (y >= 2 * Ho || x >= 2 * Wo) {
            #pragma unroll
            for (int k = 0; k < 8; k++) o[k] = __float2half_rn(0.f);
        } else {
            const int y0 = y & ~1, x0 = x & ~1, me = (y - y0) * 2 + (x - x0);
            __half w[4][8];
            #pragma unroll
            for (int t = 0; t < 4; t++)
                *reinterpret_cast<uint4*>(w[t]) = *reinterpret_cast<const uint4*>(a + ((n * H + y0 + (t >> 1)) * W + x0 + (t & 1)) * C + cv * 8);
            const uint4 g = *reinterpret_cast<const uint4*>(dout + ((n * Ho + y0 / 2) * Wo + x0 / 2) * C + cv * 8);
            const __half* gh = reinterpret_cast<const __half*>(&g);
            #pragma unroll
            for (int k = 0; k < 8; k++) {
                int arg = 0; float best = __half2float(w[0][k]);
                #pragma unroll
                for (int t = 1; t < 4; t++) { const float v = __half2float(w[t][k]); if (v > best) { best = v; arg = t; } }
                o[k] = (arg == me && __half2float(w[me][k]) > 0.f) ? gh[k] : __float2half_rn(0.f);
            }
        }
        *reinterpret_cast<uint4*>(din + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// conv1_1 OIHW fp32 [64][3][3][3] -> fp32 [64][3][3][4] (input channels padded to 4) for Builder::conv_small_cin, and the
// flipped fp16 copy [4][2-ky][2-kx][64] for its input gradient through Builder::conv_small_cout
__global__ void k_conv1_w(const float* __restrict__ src, float* __restrict__ fwd, __half* __restrict__ dgrad, int O) {
    const int n = O * 4 * 9;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = i % 4, t = (i / 4) % 9, o = i / 36;
        const float v = c < 3 ? src[(o * 3 + c) * 9 + t] : 0.f;
        fwd[i] = v;
        dgrad[(c * 9 + (8 - t)) * O + o] = __float2half_rn(v);
    }
}

// y_mu[c] = mean over the N y images and their P positions of F[N + n][p][c]; fixed-order sums.  Block (32 channels x 8 slices).
__global__ void k_ymu(const __half* __restrict__ F, int N, int P, int C, float* __restrict__ ymu) {
    __shared__ float part[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x, sl = threadIdx.y;
    float s = 0.f;
    const __half* base = F + (size_t)N * P * C;
    for (int r = sl; r < N * P; r += 8) s += __half2float(base[(size_t)r * C + c]);
    part[sl][threadIdx.x] = s;
    __syncthreads();
    if (sl == 0) {
        float t = 0.f;
        for (int k = 0; k < 8; k++) t += part[k][threadIdx.x];
        ymu[c] = t / (float)(N * P);
    }
}

// F.normalize(F - y_mu, dim=channels): one warp per row of the [2N*P][C] fp16 features -> fp32 xh rows, norms kept for the backward
__global__ void k_normalize(const __half* __restrict__ F, const float* __restrict__ ymu, int rows, int C, float* __restrict__ xh, float* __restrict__ nrm) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __half* f = F + (size_t)row * C;
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = __half2float(f[c]) - ymu[c]; ss += v * v; }
    ss = warp_sum(ss);
    const float nr = sqrtf(ss), den = fmaxf(nr, 1e-12f);
    for (int c = lane; c < C; c += 32) xh[(size_t)row * C + c] = (__half2float(f[c]) - ymu[c]) / den;
    if (lane == 0) nrm[row] = nr;
}

// fp32 batched GEMM, C[z][m][n] = sum_k A[z][m][k] * B[z](k, n) with B(k, n) = b_nk ? B[n*ldb + k] : B[k*ldb + n].  64 x 64 tiles,
// 16-deep K slices, 4 x 4 outputs per thread, every output summed by one thread in k order (deterministic).
__global__ void __launch_bounds__(256) k_sgemm(const float* __restrict__ A, long long lda, long long sA, const float* __restrict__ B, long long ldb,
                                               long long sB, int b_nk, float* __restrict__ Cm, long long ldc, long long sC, int M, int N, int K) {
    __shared__ float As[16][64 + 4], Bs[16][64 + 4];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    A += blockIdx.z * sA; B += blockIdx.z * sB; Cm += blockIdx.z * sC;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
        #pragma unroll
        for (int t = 0; t < 4; t++) {
            const int e = tid + t * 256;                 // 1024 elements of each tile
            {   const int r = e / 16, k = e % 16;        // A: row r, k contiguous
                As[k][r] = (m0 + r < M && k0 + k < K) ? A[(size_t)(m0 + r) * lda + k0 + k] : 0.f; }
            if (b_nk) { const int r = e / 16, k = e % 16;
                Bs[k][r] = (n0 + r < N && k0 + k < K) ? B[(size_t)(n0 + r) * ldb + k0 + k] : 0.f; }
            else { const int k = e / 64, r = e % 64;
                Bs[k][r] = (n0 + r < N && k0 + k < K) ? B[(size_t)(k0 + k) * ldb + n0 + r] : 0.f; }
        }
        __syncthreads();
        #pragma unroll
        for (int k = 0; k < 16; k++) {
            float a[4], b[4];
            #pragma unroll
            for (int i = 0; i < 4; i++) { a[i] = As[k][ty + 16 * i]; b[i] = Bs[k][tx + 16 * i]; }
            #pragma unroll
            for (int i = 0; i < 4; i++)
                #pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    #pragma unroll
    for (int i = 0; i < 4; i++)
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
            if (m < M && n < N) Cm[(size_t)m * ldc + n] = acc[i][j];
        }
}

// block-wide (256 threads) fixed-order reductions
__device__ __forceinline__ float block_sum(float v, float* sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += sh[w];
    return t;
}
// (value, index) minimum, ties to the lower index
__device__ __forceinline__ void block_argmin(float& v, int& idx, float* shv, int* shi) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o); const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ov < v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { shv[threadIdx.x >> 5] = v; shi[threadIdx.x >> 5] = idx; }
    __syncthreads();
    v = shv[0]; idx = shi[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) if (shv[w] < v || (shv[w] == v && shi[w] < idx)) { v = shv[w]; idx = shi[w]; }
}

// Row pass, one block per row (n, i) of S [N][P][P] (cosine similarities): d = 1 - S, mu = min_j d (argmin kept),
// w = exp((1 - d / (mu + eps)) / h), cx = w / sum_j w.  h: device scalar (the band width of the call).
__global__ void __launch_bounds__(256) k_cx_rows(const float* __restrict__ S, int P, const float* __restrict__ band_width, float* __restrict__ cx,
                                                 float* __restrict__ rmin, int* __restrict__ rarg) {
    __shared__ float shv[8]; __shared__ int shi[8];
    const float h = *band_width;
    const size_t row = blockIdx.x;
    const float* s = S + row * P;
    float mn = INFINITY; int am = 0x7fffffff;
    for (int j = threadIdx.x; j < P; j += blockDim.x) { const float d = 1.f - s[j]; if (d < mn) { mn = d; am = j; } }
    block_argmin(mn, am, shv, shi);
    const float den = mn + kEps;
    float sum = 0.f;
    for (int j = threadIdx.x; j < P; j += blockDim.x) sum += expf((1.f - (1.f - s[j]) / den) / h);
    sum = block_sum(sum, shv);
    for (int j = threadIdx.x; j < P; j += blockDim.x) cx[row * P + j] = expf((1.f - (1.f - s[j]) / den) / h) / sum;
    if (threadIdx.x == 0) { rmin[row] = mn; rarg[row] = am; }
}

// Column pass: cmax[n][j] = max_i cx[n][i][j] (argmax kept, ties to the lower i)
__global__ void k_cx_cols(const float* __restrict__ cx, int P, float* __restrict__ cmax, int* __restrict__ carg) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
    if (j >= P) return;
    const float* c = cx + (size_t)n * P * P + j;
    float best = c[0]; int arg = 0;
    for (int i = 1; i < P; i++) { const float v = c[(size_t)i * P]; if (v > best) { best = v; arg = i; } }
    cmax[(size_t)n * P + j] = best; carg[(size_t)n * P + j] = arg;
}

// loss = mean_n -log(mean_j cmax[n][j] + eps); m[n] = mean_j cmax[n][j] kept for the backward.  One block of 256.
__global__ void k_cx_loss(const float* __restrict__ cmax, int N, int P, float* __restrict__ m, float* __restrict__ loss) {
    __shared__ float sh[8];
    float l = 0.f;
    for (int n = 0; n < N; n++) {
        float s = 0.f;
        for (int j = threadIdx.x; j < P; j += blockDim.x) s += cmax[(size_t)n * P + j];
        s = block_sum(s, sh) / (float)P;
        if (threadIdx.x == 0) m[n] = s;
        l += -logf(s + kEps);
    }
    if (threadIdx.x == 0) *loss = l / (float)N;
}

// Backward of the row pass, one block per row (n, i): G[n][i][j] = dloss / dS[n][i][j].
//   g_ij  = dloss * -1 / (N (m_n + eps) P) where i = argmax_i(j), else 0           (the mean / max / log)
//   T     = sum_j g_ij cx_ij ;  dd~_ij = -(g_ij - T) cx_ij / h                     (row normalisation, exp)
//   U     = sum_j dd~_ij d_ij ;  dd_ij = dd~_ij / (mu + eps) - [j == argmin] U / (mu + eps)^2
//   G_ij  = -dd_ij                                                                 (d = 1 - S)
__global__ void __launch_bounds__(256) k_cx_rows_bwd(const float* __restrict__ S, const float* __restrict__ cx, const float* __restrict__ rmin,
                                                     const int* __restrict__ rarg, const int* __restrict__ carg, const float* __restrict__ m,
                                                     const float* __restrict__ dloss, int N, int P, const float* __restrict__ band_width,
                                                     float* __restrict__ G) {
    __shared__ float sh[8];
    const float h = *band_width;
    const size_t row = blockIdx.x;
    const int n = (int)(row / P), i = (int)(row % P);
    const float gval = *dloss * (-1.f / ((float)N * (m[n] + kEps))) / (float)P;
    const float* s = S + row * P; const float* c = cx + row * P; const int* ca = carg + (size_t)n * P;
    float t = 0.f;
    for (int j = threadIdx.x; j < P; j += blockDim.x) if (ca[j] == i) t += gval * c[j];
    t = block_sum(t, sh);
    float u = 0.f;
    for (int j = threadIdx.x; j < P; j += blockDim.x) u += -((ca[j] == i ? gval : 0.f) - t) * c[j] / h * (1.f - s[j]);
    u = block_sum(u, sh);
    const float den = rmin[row] + kEps; const int am = rarg[row];
    for (int j = threadIdx.x; j < P; j += blockDim.x) {
        const float ddt = -((ca[j] == i ? gval : 0.f) - t) * c[j] / h;
        float dd = ddt / den;
        if (j == am) dd -= u / (den * den);
        G[row * P + j] = -dd;
    }
}

// normalize backward + the relu5_4 ReLU mask, one warp per x row: dxc = (dxh - xh <xh, dxh>) / |xc| (|xc| > 1e-12; else dxh / 1e-12),
// times (F > 0); written in place over dxh.  Also the per-row max |.| for the gradient scale.
__global__ void k_normalize_bwd(float* __restrict__ dxh, const float* __restrict__ xh, const float* __restrict__ nrm, const __half* __restrict__ F,
                                int rows, int C, float* __restrict__ rowmax) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    float* d = dxh + (size_t)row * C; const float* x = xh + (size_t)row * C; const __half* f = F + (size_t)row * C;
    float dot = 0.f;
    for (int c = lane; c < C; c += 32) dot += x[c] * d[c];
    dot = warp_sum(dot);
    const float nr = nrm[row];
    float mx = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float g = nr > 1e-12f ? (d[c] - x[c] * dot) / nr : d[c] / 1e-12f;
        const float v = __half2float(f[c]) > 0.f ? g : 0.f;
        d[c] = v; mx = fmaxf(mx, fabsf(v));
    }
    mx = warp_max(mx);
    if (lane == 0) rowmax[row] = mx;
}

// power-of-two scale that puts the largest feature gradient in [16, 32): fp16 keeps 2^11 of headroom for the growth through the
// VGG input-gradient chain, and elements down to 2^-20 of the largest stay normal.  One block of 256.
__global__ void k_grad_scale(const float* __restrict__ rowmax, int rows, float* __restrict__ scale) {
    __shared__ float sh[8];
    float m = 0.f;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) m = fmaxf(m, rowmax[r]);
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 0; w < 8; w++) m = fmaxf(m, sh[w]);
        int e = 0;
        if (m > 0.f && isfinite(m)) frexpf(m, &e);
        *scale = m > 0.f && isfinite(m) ? ldexpf(1.f, min(max(5 - e, -100), 100)) : 1.f;
    }
}

__global__ void k_set(float* __restrict__ dst, float v) { *dst = v; }

__global__ void k_scale_to_f16(const float* __restrict__ g, const float* __restrict__ scale, __half* __restrict__ out, size_t n) {
    const float s = *scale;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = __float2half_rn(g[i] * s);
}

// image gradient: g4 fp32 [N,H,W,4] (conv1_1's input gradient, scaled) -> dx fp32 [N,3,H,W] = g4 / std / scale
__global__ void k_img_grad(const float* __restrict__ g4, const float* __restrict__ scale, int N, int H, int W, float* __restrict__ dx) {
    const float inv = 1.f / *scale;
    const size_t hw = (size_t)H * W, total = (size_t)N * 3 * hw;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i % hw; const int c = (int)((i / hw) % 3); const size_t n = i / (3 * hw);
        dx[i] = g4[(n * hw + pix) * 4 + c] / vgg_std(c) * inv;
    }
}

}  // namespace cxk
