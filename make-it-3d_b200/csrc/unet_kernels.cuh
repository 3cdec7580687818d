// unet_kernels.cuh -- kernels of the refine stage's gated U-Net (unet_engine.cu).  NCHW fp32 activations; every tensor is a view
// (pointer, per-image stride) so producers write straight into channel slices of the concatenated buffers.  No atomics: every
// reduction is a fixed per-CTA partial followed by a fixed-order pass, so results are bit-identical run to run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace unk {

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }

// ---------------------------------------------------------------------------------------------------------------
// 3x3 stride-1 zero-pad-1 convolution, direct, fp32.  A CTA owns a 32 x 32 pixel tile of one image and COB output channels;
// thread (tx, ty) computes pixels (x0 + tx, y0 + 4 ty + r), r < 4, for all COB channels.  Input channels stream through shared
// memory CI at a time (halo tile + the matching weights, stored [c][tap][o] so a thread reads 4 weights per LDS.128):
//   out[o] = bias[o] + sum_c,t w[o][c][t] in[c](p + t)             (w: [Cout][Cin][3][3], torch's layout)
// The input gradient of such a conv is the same kernel over the weights k_flip_w writes.  Two CTAs per SM (<= 128 registers), so one
// CTA's staging overlaps the other's FMAs.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CT = 32, CI = 8, COB = 16, HALO = CT + 2;

__global__ void __launch_bounds__(256, 2) k_conv3(const float* __restrict__ in, long long in_ns, int Cin, const float* __restrict__ w,
                                                  const float* __restrict__ bias, float* __restrict__ out, long long out_ns, int Cout, int H, int W) {
    __shared__ float s_in[CI][HALO][HALO];
    __shared__ __align__(16) float s_w[CI][9][COB];
    const int tiles_x = (W + CT - 1) / CT;
    const int x0 = (blockIdx.x % tiles_x) * CT, y0 = (blockIdx.x / tiles_x) * CT;
    const int o0 = blockIdx.y * COB, n = blockIdx.z;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, tid = threadIdx.x;
    const size_t HW = (size_t)H * W;
    const float* inn = in + (size_t)n * in_ns;
    float acc[4][COB];
    #pragma unroll
    for (int r = 0; r < 4; r++)
        #pragma unroll
        for (int o = 0; o < COB; o++) acc[r][o] = 0.f;

    for (int c0 = 0; c0 < Cin; c0 += CI) {
        __syncthreads();
        // one halo row per warp and step (lanes load columns 0..31, lanes 0..1 also 32..33), 4 rows' loads in flight per warp
        constexpr int kRows = CI * HALO, kBatch = 4;
        for (int r0 = ty; r0 < kRows; r0 += 8 * kBatch) {
            float a[kBatch], b[kBatch];
            #pragma unroll
            for (int q = 0; q < kBatch; q++) {
                const int row = r0 + 8 * q, c = row / HALO, yy = row - c * HALO, gy = y0 + yy - 1;
                const bool ok = row < kRows && c0 + c < Cin && gy >= 0 && gy < H;
                const float* src = inn + (size_t)(c0 + c) * HW + (size_t)gy * W;
                const int gx = x0 + tx - 1, gx2 = x0 + 31 + tx;
                a[q] = ok && gx >= 0 && gx < W ? __ldg(src + gx) : 0.f;
                b[q] = ok && tx < 2 && gx2 < W ? __ldg(src + gx2) : 0.f;
            }
            #pragma unroll
            for (int q = 0; q < kBatch; q++) {
                const int row = r0 + 8 * q, c = row / HALO, yy = row - c * HALO;
                if (row < kRows) { s_in[c][yy][tx] = a[q]; if (tx < 2) s_in[c][yy][32 + tx] = b[q]; }
            }
        }
        constexpr int kW = CI * 9 * COB, kWPer = (kW + 255) / 256;
        float wv[kWPer];
        #pragma unroll
        for (int k = 0; k < kWPer; k++) {
            const int i = tid + 256 * k, o = i % COB, t = (i / COB) % 9, c = i / (9 * COB), oc = o0 + o, cc = c0 + c;
            wv[k] = i < kW && oc < Cout && cc < Cin ? __ldg(w + ((size_t)oc * Cin + cc) * 9 + t) : 0.f;
        }
        #pragma unroll
        for (int k = 0; k < kWPer; k++) {
            const int i = tid + 256 * k;
            if (i < kW) s_w[i / (9 * COB)][(i / COB) % 9][i % COB] = wv[k];
        }
        __syncthreads();
        #pragma unroll 1
        for (int c = 0; c < CI; c++) {
            #pragma unroll
            for (int kx = 0; kx < 3; kx++) {
                float v[6];
                #pragma unroll
                for (int j = 0; j < 6; j++) v[j] = s_in[c][4 * ty + j][tx + kx];
                #pragma unroll
                for (int ky = 0; ky < 3; ky++) {
                    float wv[COB];
                    #pragma unroll
                    for (int q = 0; q < COB / 4; q++) {
                        const float4 f = *reinterpret_cast<const float4*>(&s_w[c][ky * 3 + kx][4 * q]);
                        wv[4 * q] = f.x; wv[4 * q + 1] = f.y; wv[4 * q + 2] = f.z; wv[4 * q + 3] = f.w;
                    }
                    #pragma unroll
                    for (int r = 0; r < 4; r++)
                        #pragma unroll
                        for (int o = 0; o < COB; o++) acc[r][o] = fmaf(v[r + ky], wv[o], acc[r][o]);
                }
            }
        }
    }
    const int x = x0 + tx;
    if (x >= W) return;
    float* outn = out + (size_t)n * out_ns;
    #pragma unroll
    for (int o = 0; o < COB; o++) {
        const int oc = o0 + o;
        if (oc >= Cout) break;
        const float b = bias ? bias[oc] : 0.f;
        #pragma unroll
        for (int r = 0; r < 4; r++) {
            const int y = y0 + 4 * ty + r;
            if (y < H) outn[(size_t)oc * HW + (size_t)y * W + x] = acc[r][o] + b;
        }
    }
}

// the input-gradient weights of a 3x3 conv with forward weights w [Co][Ci][3][3]: wt [Ci][Co][3][3], wt[i][o][t] = w[o][i][8 - t]
__global__ void k_flip_w(const float* __restrict__ w, int Co, int Ci, float* __restrict__ wt) {
    const int n = Co * Ci * 9;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const int t = e % 9, o = (e / 9) % Co, i = e / (9 * Co);
        wt[e] = w[((size_t)o * Ci + i) * 9 + 8 - t];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Weight and bias gradient of a 3x3 conv: dW[o][c][t] = sum_p dy[o](p) in[c](p + t), db[o] = sum_p dy[o](p).
// Grid (S, Cout / WOB, Cin / WCB).  Chunk k walks the 32 x 4 pixel tiles k, k + S, k + 2S, ... of the whole batch, so the pixel sum
// is split over a fixed set of CTAs; each writes its fp32 partial to part[k][o][c][t] (bias: bpart[k][o]) and k_sum_chunks adds the
// S partials in order.  Thread t: input channel t % 16 and output channels 4 (t / 16) .. + 3, all 9 taps, with a register window
// sliding along the tile row.
// ---------------------------------------------------------------------------------------------------------------
constexpr int WTX = 32, WTY = 4, WOB = 32, WCB = 16, WXP = (WTY + 2) * (WTX + 2) + 1;   // odd channel pitch: no bank conflicts

__global__ void __launch_bounds__(128) k_conv3_wgrad(const float* __restrict__ in, long long in_ns, int Cin, const float* __restrict__ dy,
                                                     long long dy_ns, int Cout, int N, int H, int W, float* __restrict__ part,
                                                     float* __restrict__ bpart) {
    __shared__ float s_x[WCB * WXP];
    __shared__ __align__(16) float s_dy[WTY * WTX][WOB];
    const int S = gridDim.x, k = blockIdx.x, o0 = blockIdx.y * WOB, c0 = blockIdx.z * WCB;
    const int tid = threadIdx.x, cl = tid % WCB, og = tid / WCB;
    const int tiles_x = (W + WTX - 1) / WTX, tiles_y = (H + WTY - 1) / WTY, tiles = N * tiles_x * tiles_y;
    const size_t HW = (size_t)H * W;
    float acc[4][9], bacc[4];
    #pragma unroll
    for (int o = 0; o < 4; o++) { bacc[o] = 0.f;
        #pragma unroll
        for (int t = 0; t < 9; t++) acc[o][t] = 0.f; }
    for (int tile = k; tile < tiles; tile += S) {
        const int n = tile / (tiles_x * tiles_y), rem = tile - n * tiles_x * tiles_y;
        const int y0 = (rem / tiles_x) * WTY, x0 = (rem % tiles_x) * WTX;
        __syncthreads();
        for (int i = tid; i < WCB * (WTY + 2) * (WTX + 2); i += 128) {
            const int c = i / ((WTY + 2) * (WTX + 2)), r = i - c * (WTY + 2) * (WTX + 2), yy = r / (WTX + 2), xx = r - yy * (WTX + 2);
            const int gy = y0 + yy - 1, gx = x0 + xx - 1;
            float v = 0.f;
            if (c0 + c < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W) v = in[(size_t)n * in_ns + (size_t)(c0 + c) * HW + (size_t)gy * W + gx];
            s_x[c * WXP + r] = v;
        }
        for (int i = tid; i < WTY * WTX * WOB; i += 128) {
            const int o = i / (WTY * WTX), p = i - o * (WTY * WTX), yy = p / WTX, xx = p - yy * WTX;
            const int gy = y0 + yy, gx = x0 + xx;
            float v = 0.f;
            if (o0 + o < Cout && gy < H && gx < W) v = dy[(size_t)n * dy_ns + (size_t)(o0 + o) * HW + (size_t)gy * W + gx];
            s_dy[p][o] = v;
        }
        __syncthreads();
        const float* xs = s_x + cl * WXP;
        #pragma unroll 1
        for (int r = 0; r < WTY; r++) {
            float win[3][3];
            #pragma unroll
            for (int ky = 0; ky < 3; ky++) { win[ky][0] = xs[(r + ky) * (WTX + 2)]; win[ky][1] = xs[(r + ky) * (WTX + 2) + 1]; }
            #pragma unroll 4
            for (int x = 0; x < WTX; x++) {
                #pragma unroll
                for (int ky = 0; ky < 3; ky++) win[ky][2] = xs[(r + ky) * (WTX + 2) + x + 2];
                const float4 d = *reinterpret_cast<const float4*>(&s_dy[r * WTX + x][4 * og]);
                const float dv[4] = {d.x, d.y, d.z, d.w};
                #pragma unroll
                for (int o = 0; o < 4; o++) {
                    #pragma unroll
                    for (int ky = 0; ky < 3; ky++)
                        #pragma unroll
                        for (int kx = 0; kx < 3; kx++) acc[o][ky * 3 + kx] = fmaf(dv[o], win[ky][kx], acc[o][ky * 3 + kx]);
                    bacc[o] += dv[o];
                }
                #pragma unroll
                for (int ky = 0; ky < 3; ky++) { win[ky][0] = win[ky][1]; win[ky][1] = win[ky][2]; }
            }
        }
    }
    const int c = c0 + cl;
    #pragma unroll
    for (int o = 0; o < 4; o++) {
        const int oc = o0 + 4 * og + o;
        if (oc >= Cout) break;
        if (c < Cin) {
            float* d = part + ((size_t)k * Cout + oc) * Cin * 9 + (size_t)c * 9;
            #pragma unroll
            for (int t = 0; t < 9; t++) d[t] = acc[o][t];
        }
        if (bpart && blockIdx.z == 0 && cl == 0) bpart[(size_t)k * Cout + oc] = bacc[o];
    }
}

// out[e] = sum_{k < S} part[k][e], k in order
__global__ void k_sum_chunks(const float* __restrict__ part, int S, size_t E, float* __restrict__ out) {
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < E; e += (size_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < S; k++) s += part[(size_t)k * E + e];
        out[e] = s;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// memory-bound kernels
// ---------------------------------------------------------------------------------------------------------------
// fm = [f | m] (2C channels, contiguous per image) -> g = ELU(f) * sigmoid(m), written to a view
__global__ void k_gate(const float* __restrict__ fm, int C, int N, size_t HW, float* __restrict__ g, long long g_ns) {
    const size_t total = (size_t)N * C * HW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i % HW, c = (i / HW) % C, n = i / (HW * C);
        const float* b = fm + n * 2 * C * HW;
        g[n * g_ns + c * HW + p] = elu(b[c * HW + p]) * sigm(b[(C + c) * HW + p]);
    }
}

// Per-channel partial sums, double accumulation: grid (C, S).  mode 0: (sum x, sum x^2) of x.  mode 1 (BatchNorm backward):
// (sum dy, sum dy * xhat), xhat = (x - mean[c]) * rstd[c].  part[(c * S + k) * 2 + {0, 1}].
__global__ void __launch_bounds__(256) k_chan_partial(const float* __restrict__ x, long long x_ns, const float* __restrict__ dy, long long dy_ns,
                                                      const float* __restrict__ mean, const float* __restrict__ rstd, int N, size_t HW, int mode,
                                                      double* __restrict__ part) {
    const int c = blockIdx.x, S = gridDim.y, k = blockIdx.y;
    const size_t M = (size_t)N * HW, per = (M + S - 1) / S, b = (size_t)k * per, e = b + per < M ? b + per : M;
    double s0 = 0.0, s1 = 0.0;
    const float mu = mode ? mean[c] : 0.f, rs = mode ? rstd[c] : 0.f;
    for (size_t i = b + threadIdx.x; i < e; i += blockDim.x) {
        const size_t n = i / HW, p = i - n * HW;
        const float v = x[n * x_ns + (size_t)c * HW + p];
        if (mode == 0) { s0 += v; s1 += (double)v * v; }
        else { const float d = dy[n * dy_ns + (size_t)c * HW + p]; s0 += d; s1 += (double)d * ((v - mu) * rs); }
    }
    __shared__ double r0[256], r1[256];
    r0[threadIdx.x] = s0; r1[threadIdx.x] = s1;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) { r0[threadIdx.x] += r0[threadIdx.x + w]; r1[threadIdx.x] += r1[threadIdx.x + w]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { part[((size_t)c * S + k) * 2] = r0[0]; part[((size_t)c * S + k) * 2 + 1] = r1[0]; }
}

// batch statistics: mean, biased variance, rstd = 1 / sqrt(var + eps)
__global__ void k_bn_stats(const double* __restrict__ part, int C, int S, double M, float eps, float* mean, float* var, float* rstd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s0 = 0.0, s1 = 0.0;
    for (int k = 0; k < S; k++) { s0 += part[((size_t)c * S + k) * 2]; s1 += part[((size_t)c * S + k) * 2 + 1]; }
    const double mu = s0 / M, v = fmax(s1 / M - mu * mu, 0.0);
    mean[c] = (float)mu; var[c] = (float)v; rstd[c] = (float)(1.0 / sqrt(v + (double)eps));
}

// running statistics -> mean, rstd (eval mode)
__global__ void k_bn_eval_stats(const float* __restrict__ rmean, const float* __restrict__ rvar, int C, float eps, float* mean, float* rstd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mean[c] = rmean[c]; rstd[c] = (float)(1.0 / sqrt((double)rvar[c] + (double)eps));
}

// BatchNorm backward reduction: dbeta = sum dy, dgamma = sum dy * xhat; sums kept for the apply pass
__global__ void k_bn_bwd_stats(const double* __restrict__ part, int C, int S, float* dgamma, float* dbeta, float* sdy, float* sdyx) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s0 = 0.0, s1 = 0.0;
    for (int k = 0; k < S; k++) { s0 += part[((size_t)c * S + k) * 2]; s1 += part[((size_t)c * S + k) * 2 + 1]; }
    dbeta[c] = (float)s0; dgamma[c] = (float)s1; sdy[c] = (float)s0; sdyx[c] = (float)s1;
}

__global__ void k_bn_apply(const float* __restrict__ g, const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                           const float* __restrict__ beta, int C, int N, size_t HW, float* __restrict__ out, long long out_ns) {
    const size_t total = (size_t)N * C * HW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i % HW, c = (i / HW) % C, n = i / (HW * C);
        out[n * out_ns + c * HW + p] = (g[i] - mean[c]) * rstd[c] * gamma[c] + beta[c];
    }
}

// Gate backward with the BatchNorm backward folded in.  dy: gradient of the block output (a view).  bn = 0: no norm (up blocks).
// bn = 1, train: dg = gamma rstd (dy - (sdy + xhat sdyx) / M);  bn = 2, eval: dg = gamma rstd dy.
// d[f|m]: df = dg sigmoid(m) ELU'(f), dm = dg ELU(f) sigmoid'(m).
__global__ void k_gate_bwd(const float* __restrict__ dy, long long dy_ns, const float* __restrict__ fm, const float* __restrict__ g,
                           const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                           const float* __restrict__ sdy, const float* __restrict__ sdyx, int bn, int C, int N, size_t HW,
                           float* __restrict__ dfm) {
    const size_t total = (size_t)N * C * HW;
    const float invM = 1.f / (float)((size_t)N * HW);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i % HW, c = (i / HW) % C, n = i / (HW * C);
        float d = dy[n * dy_ns + c * HW + p];
        if (bn == 1) {
            const float xh = (g[i] - mean[c]) * rstd[c];
            d = gamma[c] * rstd[c] * (d - (sdy[c] + xh * sdyx[c]) * invM);
        } else if (bn == 2) {
            d = gamma[c] * rstd[c] * d;
        }
        const size_t fo = n * 2 * C * HW + c * HW + p, mo = fo + C * HW;
        const float f = fm[fo], s = sigm(fm[mo]);
        dfm[fo] = d * s * (f > 0.f ? 1.f : expf(f));
        dfm[mo] = d * elu(f) * s * (1.f - s);
    }
}

// 2 x 2 average pool (H, W even) and its gradient, added into din
__global__ void k_avgpool(const float* __restrict__ in, long long in_ns, int C, int N, int H, int W, float* __restrict__ out, long long out_ns) {
    const int Ho = H / 2, Wo = W / 2;
    const size_t total = (size_t)N * C * Ho * Wo;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wo), y = (int)((i / Wo) % Ho); const size_t c = (i / ((size_t)Wo * Ho)) % C, n = i / ((size_t)Wo * Ho * C);
        const float* a = in + n * in_ns + c * H * W + (size_t)(2 * y) * W + 2 * x;
        out[n * out_ns + c * Ho * Wo + (size_t)y * Wo + x] = (a[0] + a[1] + a[W] + a[W + 1]) * 0.25f;
    }
}
__global__ void k_avgpool_bwd_add(const float* __restrict__ dout, long long dout_ns, int C, int N, int H, int W, float* __restrict__ din, long long din_ns) {
    const int Ho = H / 2, Wo = W / 2;
    const size_t total = (size_t)N * C * H * W;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H); const size_t c = (i / ((size_t)W * H)) % C, n = i / ((size_t)W * H * C);
        din[n * din_ns + c * H * W + (size_t)y * W + x] += 0.25f * dout[n * dout_ns + c * Ho * Wo + (size_t)(y / 2) * Wo + x / 2];
    }
}

// bilinear x2, align_corners=False (PyTorch's source index: max(0, (o + 0.5) / 2 - 0.5), neighbour clamped at the last row/column)
__device__ __forceinline__ void up_src(int o, int in, int& i0, int& i1, float& l1) {
    const float s = fmaxf(0.5f * ((float)o + 0.5f) - 0.5f, 0.f);
    i0 = (int)s; i1 = i0 < in - 1 ? i0 + 1 : i0; l1 = s - (float)i0;
}
__global__ void k_upsample2(const float* __restrict__ in, long long in_ns, int C, int N, int h, int w, float* __restrict__ out, long long out_ns) {
    const int Ho = 2 * h, Wo = 2 * w;
    const size_t total = (size_t)N * C * Ho * Wo;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wo), y = (int)((i / Wo) % Ho); const size_t c = (i / ((size_t)Wo * Ho)) % C, n = i / ((size_t)Wo * Ho * C);
        int y0, y1, x0, x1; float ly, lx;
        up_src(y, h, y0, y1, ly); up_src(x, w, x0, x1, lx);
        const float* a = in + n * in_ns + c * h * w;
        const float v = (1.f - ly) * ((1.f - lx) * a[(size_t)y0 * w + x0] + lx * a[(size_t)y0 * w + x1]) +
                        ly * ((1.f - lx) * a[(size_t)y1 * w + x0] + lx * a[(size_t)y1 * w + x1]);
        out[n * out_ns + c * Ho * Wo + (size_t)y * Wo + x] = v;
    }
}
// its gradient as a gather: input (y, x) collects from the output rows / columns 2y - 2 .. 2y + 2 that reference it
__device__ __forceinline__ float up_weight(int o, int i, int in) {
    int i0, i1; float l1; up_src(o, in, i0, i1, l1);
    return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}
__global__ void k_upsample2_bwd(const float* __restrict__ dout, long long dout_ns, int C, int N, int h, int w, float* __restrict__ din, long long din_ns) {
    const int Ho = 2 * h, Wo = 2 * w;
    const size_t total = (size_t)N * C * h * w;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % w), y = (int)((i / w) % h); const size_t c = (i / ((size_t)w * h)) % C, n = i / ((size_t)w * h * C);
        const float* d = dout + n * dout_ns + c * Ho * Wo;
        float s = 0.f;
        for (int oy = max(2 * y - 2, 0); oy <= min(2 * y + 2, Ho - 1); oy++) {
            const float wy = up_weight(oy, y, h);
            if (wy == 0.f) continue;
            float r = 0.f;
            for (int ox = max(2 * x - 2, 0); ox <= min(2 * x + 2, Wo - 1); ox++) {
                const float wx = up_weight(ox, x, w);
                if (wx != 0.f) r += wx * d[(size_t)oy * Wo + ox];
            }
            s += wy * r;
        }
        din[n * din_ns + c * h * w + (size_t)y * w + x] = s;
    }
}

// final 1x1 conv 16 -> 3 + sigmoid; backward: dz = dout y (1 - y), dg = W^T dz
constexpr int FC = 16, FO = 3;
__global__ void k_final(const float* __restrict__ g, const float* __restrict__ w, const float* __restrict__ b, int N, size_t HW, float* __restrict__ y) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)N * HW; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / HW, p = i - n * HW;
        float z[FO];
        #pragma unroll
        for (int o = 0; o < FO; o++) z[o] = b[o];
        #pragma unroll
        for (int c = 0; c < FC; c++) {
            const float v = g[(n * FC + c) * HW + p];
            #pragma unroll
            for (int o = 0; o < FO; o++) z[o] = fmaf(w[o * FC + c], v, z[o]);
        }
        #pragma unroll
        for (int o = 0; o < FO; o++) y[(n * FO + o) * HW + p] = sigm(z[o]);
    }
}
__global__ void k_final_bwd(const float* __restrict__ dout, const float* __restrict__ y, const float* __restrict__ w, int N, size_t HW,
                            float* __restrict__ dz, float* __restrict__ dg) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)N * HW; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / HW, p = i - n * HW;
        float d[FO];
        #pragma unroll
        for (int o = 0; o < FO; o++) { const size_t j = (n * FO + o) * HW + p; const float v = y[j]; d[o] = dout[j] * v * (1.f - v); dz[j] = d[o]; }
        #pragma unroll
        for (int c = 0; c < FC; c++) {
            float s = 0.f;
            #pragma unroll
            for (int o = 0; o < FO; o++) s = fmaf(w[o * FC + c], d[o], s);
            dg[(n * FC + c) * HW + p] = s;
        }
    }
}
// final conv's weight / bias gradient partials: part[k][o * 17 + c] (c = 16: the bias), fixed thread and warp order
__global__ void __launch_bounds__(256) k_final_wgrad(const float* __restrict__ dz, const float* __restrict__ g, int N, size_t HW, float* __restrict__ part) {
    const int S = gridDim.x, k = blockIdx.x;
    const size_t M = (size_t)N * HW, per = (M + S - 1) / S, b = (size_t)k * per, e = b + per < M ? b + per : M;
    float acc[FO][FC + 1];
    #pragma unroll
    for (int o = 0; o < FO; o++)
        #pragma unroll
        for (int c = 0; c <= FC; c++) acc[o][c] = 0.f;
    for (size_t i = b + threadIdx.x; i < e; i += blockDim.x) {
        const size_t n = i / HW, p = i - n * HW;
        float d[FO];
        #pragma unroll
        for (int o = 0; o < FO; o++) { d[o] = dz[(n * FO + o) * HW + p]; acc[o][FC] += d[o]; }
        #pragma unroll
        for (int c = 0; c < FC; c++) {
            const float v = g[(n * FC + c) * HW + p];
            #pragma unroll
            for (int o = 0; o < FO; o++) acc[o][c] = fmaf(d[o], v, acc[o][c]);
        }
    }
    __shared__ float red[8][FO * (FC + 1)];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    #pragma unroll
    for (int o = 0; o < FO; o++)
        #pragma unroll
        for (int c = 0; c <= FC; c++) {
            float v = acc[o][c];
            #pragma unroll
            for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
            if (lane == 0) red[wid][o * (FC + 1) + c] = v;
        }
    __syncthreads();
    if (threadIdx.x < FO * (FC + 1)) {
        float s = 0.f;
        for (int q = 0; q < 8; q++) s += red[q][threadIdx.x];
        part[(size_t)k * FO * (FC + 1) + threadIdx.x] = s;
    }
}
// sum the final conv's partials in order -> dW [3][16], db [3]
__global__ void k_final_wgrad_sum(const float* __restrict__ part, int S, float* __restrict__ dw, float* __restrict__ db) {
    const int j = threadIdx.x;
    if (j >= FO * (FC + 1)) return;
    float s = 0.f;
    for (int k = 0; k < S; k++) s += part[(size_t)k * FO * (FC + 1) + j];
    const int o = j / (FC + 1), c = j % (FC + 1);
    if (c == FC) db[o] = s; else dw[o * FC + c] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// per-call parameter traffic: up to 48 fp32 tensors gathered from the caller's parameters into the workspace (or the reverse for
// the gradients) in one launch
// ---------------------------------------------------------------------------------------------------------------
struct CopyList { const float* src[48]; float* dst[48]; int n[48]; int count; };
__global__ void k_copy_list(const CopyList l) {
    const int t = blockIdx.y;
    if (t >= l.count || !l.src[t] || !l.dst[t]) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < l.n[t]; i += gridDim.x * blockDim.x) l.dst[t][i] = l.src[t][i];
}

// running statistics of up to 3 BatchNorm layers: running = (1 - momentum) running + momentum batch (unbiased variance),
// num_batches_tracked += 1.  A null pointer skips that tensor.
struct RunningList { float* rmean[3]; float* rvar[3]; long long* nbt[3]; const float* mean[3]; const float* var[3]; int C[3]; double M[3]; float momentum; };
__global__ void k_bn_running(const RunningList r) {
    const int l = blockIdx.x, c = threadIdx.x;
    if (c == 0 && r.nbt[l]) r.nbt[l][0] += 1;
    if (c >= r.C[l]) return;
    const float m = r.momentum;
    if (r.rmean[l]) r.rmean[l][c] = (1.f - m) * r.rmean[l][c] + m * r.mean[l][c];
    if (r.rvar[l]) r.rvar[l][c] = (1.f - m) * r.rvar[l][c] + m * (float)((double)r.var[l][c] * r.M[l] / (r.M[l] - 1.0));
}

}  // namespace unk
