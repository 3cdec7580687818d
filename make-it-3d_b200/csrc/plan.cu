// plan.cu -- the op layer of the planned engines, compiled once: the plan::Builder methods that plan the tile GEMM (tc_gemm.cuh), the
// fused attention (attn.cuh) and the memory-bound kernels below, their launchers, and the replay of a launch list as a CUDA graph.
// The engines (engine_plan.cuh, transformer_plan.cuh) see only host declarations; every kernel an op builder launches lives here.
#include <algorithm>

#include "engine_plan.cuh"
#include "tc_gemm.cuh"
#include "attn.cuh"
#include "warp_reduce.cuh"

// ------------------------------------------------------------------------------------------------------------
// memory-bound kernels of the op layer.  Activations are NHWC fp16 ("tokens x C"); statistics and reductions are fp32.
// ------------------------------------------------------------------------------------------------------------
namespace sdk {
namespace {

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

}  // namespace
}  // namespace sdk

namespace clipk {
namespace {

// x[b*Tpad + t] = tok_emb[tokens[b, t]] + pos[t] for t < L; rows L .. Tpad-1 are zero.  Token ids outside [0, vocab) are clamped
// into it (never read out of bounds).
__global__ void k_text_embed(const long long* __restrict__ tokens, const float* __restrict__ tok_emb, const float* __restrict__ pos,
                             __half* __restrict__ x, int B, int L, int Tpad, int C, int vocab) {
    const int vc = C / 8;
    const size_t total = (size_t)B * Tpad * vc;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); const size_t r = i / vc;
        const int t = (int)(r % Tpad), b = (int)(r / Tpad);
        __align__(16) __half o[8];
        if (t < L) {
            const long long id = min(max(tokens[(size_t)b * L + t], 0ll), (long long)vocab - 1);
            #pragma unroll
            for (int k = 0; k < 8; k++) o[k] = __float2half_rn(tok_emb[(size_t)id * C + v * 8 + k] + pos[(size_t)t * C + v * 8 + k]);
        } else {
            #pragma unroll
            for (int k = 0; k < 8; k++) o[k] = __float2half_rn(0.f);
        }
        *reinterpret_cast<uint4*>(x + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// LayerNorm input gradient, one warp per row (statistics recomputed from x exactly as k_layernorm computes them):
// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ add),  g = dy * gamma.
__global__ void k_layernorm_bwd(const __half* __restrict__ x, const __half* __restrict__ dy, const float* __restrict__ gamma,
                                const __half* __restrict__ add, __half* __restrict__ dx, int rows, int C, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __half* xr = x + (size_t)row * C; const __half* dr = dy + (size_t)row * C;
    float mean, rstd;
    row_stats(xr, C, eps, lane, mean, rstd);
    float g1 = 0.f, g2 = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 rx = *reinterpret_cast<const uint4*>(xr + c), rd = *reinterpret_cast<const uint4*>(dr + c);
        const __half* hx = reinterpret_cast<const __half*>(&rx); const __half* hd = reinterpret_cast<const __half*>(&rd);
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const float g = __half2float(hd[k]) * gamma[c + k];
            g1 += g; g2 += g * (__half2float(hx[k]) - mean) * rstd;
        }
    }
    g1 = warp_sum(g1) / C; g2 = warp_sum(g2) / C;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 rx = *reinterpret_cast<const uint4*>(xr + c), rd = *reinterpret_cast<const uint4*>(dr + c);
        const __half* hx = reinterpret_cast<const __half*>(&rx); const __half* hd = reinterpret_cast<const __half*>(&rd);
        uint4 ra = make_uint4(0, 0, 0, 0);
        if (add) ra = *reinterpret_cast<const uint4*>(add + (size_t)row * C + c);
        const __half* ha = reinterpret_cast<const __half*>(&ra);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const float xh = (__half2float(hx[k]) - mean) * rstd;
            o[k] = __float2half_rn(rstd * (__half2float(hd[k]) * gamma[c + k] - g1 - xh * g2) + __half2float(ha[k]));
        }
        *reinterpret_cast<uint4*>(dx + (size_t)row * C + c) = *reinterpret_cast<const uint4*>(o);
    }
}

// Causal row softmax in place over [Z][tq][cols] scores: row r (query q = r % tq) keeps keys j <= q (and j < valid); the other
// columns are written as 0.  One warp per row.
__global__ void k_softmax_causal(__half* __restrict__ s, size_t rows, int cols, int valid, int tq, float scale) {
    const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int lim = min(valid, (int)(row % tq) + 1);
    __half* r = s + row * cols;
    float mx = -INFINITY;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) if (c + k < lim) mx = fmaxf(mx, __half2float(h[k]) * scale);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        #pragma unroll
        for (int k = 0; k < 8; k++) if (c + k < lim) sum += __expf(__half2float(h[k]) * scale - mx);
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int c = lane * 8; c < cols; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(r + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(c + k < lim ? __expf(__half2float(h[k]) * scale - mx) * inv : 0.f);
        *reinterpret_cast<uint4*>(r + c) = *reinterpret_cast<const uint4*>(o);
    }
}

}  // namespace
}  // namespace clipk

// ------------------------------------------------------------------------------------------------------------
// launchers of the tile GEMM and the fused attention
// ------------------------------------------------------------------------------------------------------------
namespace tc {

template <int BN, bool kQuickGelu = false, bool kVgg = false, bool kGelu = false>
inline int launch_bn(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, int batch, cudaStream_t st) {
    static bool attr = false;
    auto kernel = [] {
        if constexpr (kVgg) return k_tc_gemm_vgg<BN>;
        else if constexpr (kGelu) return k_tc_gemm_gelu<BN>;
        else return k_tc_gemm<BN, kQuickGelu>;
    }();
    if (!attr) {
        MI3D_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<BN>::kSmemBytes));
        attr = true;
    }
    GemmParams q = p;
    q.m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M; q.n_tiles = p.N / BN;
    if (q.splits <= 1) { q.splits = 1; q.kb_per_split = q.num_k_blocks; }
    q.num_tiles = q.m_tiles * q.n_tiles * batch * q.splits;
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    const int resident = (Cfg<BN>::kSmemBytes <= 110 * 1024) ? 2 : 1;       // persistent grid: one (or two) CTAs per SM loop over the tiles
    const int grid = q.num_tiles < sms * resident ? q.num_tiles : sms * resident;
    kernel<<<grid, kThreads, Cfg<BN>::kSmemBytes, st>>>(ma, mb, q);
    return (int)cudaGetLastError();
}

inline int launch(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, int block_n, int batch, cudaStream_t st) {
    if (p.K % BLOCK_K || p.N % block_n || p.out_z1 < 1) return MI3D_ERR_ARG;
    if (((uintptr_t)p.bias | (uintptr_t)p.row_bias | (uintptr_t)p.splitk_ws) & 15) return MI3D_ERR_ARG;     // read / RED-added 16 bytes at a time
    if (p.conv == 2 || p.epi_mode == EPI_RELU || p.epi_mode == EPI_RELU_BWD) {
        if (p.splits > 1 || (p.epi_mode == EPI_RELU_BWD && !p.aux)) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, false, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, false, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, false, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    if (p.epi_mode == EPI_QUICKGELU || p.epi_mode == EPI_QUICKGELU_BWD) {
        if (p.splits > 1) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    if (p.epi_mode == EPI_GELU) {
        if (p.splits > 1 || p.conv || !p.out) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, false, false, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, false, false, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, false, false, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    switch (block_n) {
        case 64: return launch_bn<64>(ma, mb, p, batch, st);
        case 128: return launch_bn<128>(ma, mb, p, batch, st);
        case 160: return launch_bn<160>(ma, mb, p, batch, st);
        case 256: return launch_bn<256>(ma, mb, p, batch, st);
    }
    return MI3D_ERR_ARG;
}

// ws: fp32 [M][N] scratch (zeroed here)
inline int launch_splitk(const CUtensorMap& ma, const CUtensorMap& mb, GemmParams p, int block_n, int splits, float* ws, cudaStream_t st) {
    p.kb_per_split = (p.num_k_blocks + splits - 1) / splits;
    p.splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;          // every K-range non-empty
    p.splitk_ws = ws;
    MI3D_CHECK(cudaMemsetAsync(ws, 0, (size_t)p.M * p.N * sizeof(float), st));
    int r = launch(ma, mb, p, block_n, 1, st);
    if (r) return r;
    p.splits = 1;
    const size_t total = (size_t)p.m_valid * p.N / 8;
    k_splitk_finish<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ws, p);
    return (int)cudaGetLastError();
}

}  // namespace tc

namespace attn {

template <int D> static inline int launch_d(const Maps& m, __half* o, long long ldo, int B, int T, int kv_valid, int heads, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        MI3D_CHECK(cudaFuncSetAttribute(k_flash_attn<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Shape<D>::kSmemBytes));
        attr = true;
    }
    Params p; p.T = T; p.kv_valid = kv_valid; p.ldo = (int)ldo; p.scale_log2e = (float)(1.4426950408889634 / std::sqrt((double)D)); p.o = o;
    dim3 grid((unsigned)((T + 127) / 128), (unsigned)heads, (unsigned)B);
    k_flash_attn<D><<<grid, kThreads, Shape<D>::kSmemBytes, st>>>(m.q, m.k, m.v, p);
    return (int)cudaGetLastError();
}

static inline int launch(const Maps& m, __half* o, long long ldo, int B, int T, int kv_valid, int heads, cudaStream_t st) {
    if (kv_valid < 1 || T < 1) return MI3D_ERR_ARG;
    switch (m.d) {
        case 40: return launch_d<40>(m, o, ldo, B, T, kv_valid, heads, st);
        case 64: return launch_d<64>(m, o, ldo, B, T, kv_valid, heads, st);
        case 80: return launch_d<80>(m, o, ldo, B, T, kv_valid, heads, st);
        case 160: return launch_d<160>(m, o, ldo, B, T, kv_valid, heads, st);
        default: return MI3D_ERR_ARG;
    }
}

}  // namespace attn

namespace plan {

int Builder::do_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st) {
    if (p.splits > 1) return tc::launch_splitk(ma, mb, p, bn, p.splits, splitk_ws, st);
    return tc::launch(ma, mb, p, bn, batch, st);
}

int Builder::timed_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st) {
    if (!profile) return do_launch(ma, mb, p, bn, batch, st);
    if (prof_used == prof_events.size()) { cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); prof_events.push_back({a, b}); }
    if (prof_shapes.size() < prof_events.size()) prof_shapes.resize(prof_events.size());
    prof_shapes[prof_used] = {p.M, p.N, p.K, bn, p.splits, p.conv, batch, p.epi_mode};
    auto& ev = prof_events[prof_used++];
    cudaEventRecord(ev.first, st);
    const int r = do_launch(ma, mb, p, bn, batch, st);
    cudaEventRecord(ev.second, st);
    return r;
}

int Builder::load_param(const Param& P, const float* src, const float* partner, cudaStream_t st) {
    (void)partner;
    const int nb = blocks_for(P.numel);
    const int O = P.shape.empty() ? 1 : P.shape[0], I = (int)(P.numel / (size_t)O);   // a conv [O][I][kh][kw] as the matrix [O][I*kh*kw]
    switch (P.kind) {
        case PK_F32: MI3D_CHECK(cudaMemcpyAsync(P.dst, src, P.numel * 4, cudaMemcpyDeviceToDevice, st)); break;
        case PK_LINEAR: case PK_CONV1: sdk::k_f32_to_f16<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.numel); break;
        case PK_LINEAR_T: sdk::k_transpose_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, O, I); break;
        case PK_LINEAR_BOTH: case PK_CONV1_BOTH:
            sdk::k_f32_to_f16<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.numel);
            sdk::k_transpose_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst2, O, I); break;
        case PK_CONV3: case PK_CONV_SMALL_COUT: case PK_CONV_SMALL_COUT_BOTH:   // conv_small_cout: the forward weights only
            sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.shape[0], P.shape[1], 0); break;
        case PK_CONV3_BOTH:                                                     // dst2: the flipped, transposed dgrad weights
            sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.shape[0], P.shape[1], 0);
            sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst2, P.shape[0], P.shape[1], 1); break;
        case PK_CONV3_S2_BOTH:
            // dgrad of the im2col GEMM needs the plain transpose of the [Cout][9*Cin] matrix: [9*Cin][Cout]
            // (k_conv_w wrote [O][ky][kx][I]; transpose that fp16 matrix)
            sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.shape[0], P.shape[1], 0);
            sdk::k_transpose<<<dim3((9 * P.shape[1] + 31) / 32, (P.shape[0] + 31) / 32, 1), dim3(32, 8), 0, st>>>((const __half*)P.dst, (__half*)P.dst2, P.shape[0], 9 * P.shape[1]);
            break;
        default: return MI3D_ERR_ARG;
    }
    return (int)cudaGetLastError();
}

void Builder::gemm(const Mat& a, const Mat& b, int N, const Out& o, const Epi& e, int batch, bool b_batched) {
    if (dry) return;
    const long long mt = (a.rows + 127) / 128;
    int bn = tc::pick_block_n(N, mt * batch, num_sms, tc::has_block_n_160(e.mode, 0));
    if (bn == 0 || a.K % 64) { err = MI3D_ERR_ARG; return; }
    int splits = 1;
    if (batch == 1 && e.mode == tc::EPI_PLAIN && o.p16 && a.rows % 128 == 0 && (size_t)a.rows * N <= splitk_elems) {
        if (N % 128 == 0 && mt * (N / 128) * 2 <= num_sms) bn = 128;            // few, fat tiles + split-K beats many thin tiles
        splits = tc::plan_splits(mt * (N / bn), a.K / 64, num_sms);
    }
    CUtensorMap ma, mb;
    int r = tc::make_map_matrix(&ma, a.p, a.K, a.rows, a.ld, 128, a.z1, a.sz1, a.z2, a.sz2);
    if (!r) r = tc::make_map_matrix(&mb, b.p, b.K, b.rows, b.ld, bn, b.z1, b.sz1, b.z2, b.sz2);
    if (r) { err = r; return; }
    tc::GemmParams p = {};
    p.M = (int)a.rows; p.N = N; p.K = a.K; p.num_k_blocks = a.K / 64; p.conv = 0;
    p.a_z1 = a.z1; p.b_z1 = b.z1; p.b_batched = b_batched ? 1 : 0;
    p.out = o.p16; p.out_f32 = o.p32; p.ldc = o.ldc; p.out_z1 = o.z1; p.out_s_lo = o.s_lo; p.out_s_hi = o.s_hi;
    p.bias = e.bias; p.row_bias = e.row_bias; p.rows_per_group = e.rows_per_group; p.residual = e.residual; p.ld_res = e.ld_res;
    p.epi_mode = e.mode; p.alpha = e.alpha; p.m_valid = (int)a.rows; p.splits = splits; p.aux = e.aux;
    push([this, ma, mb, p, bn, batch](cudaStream_t st) { return timed_launch(ma, mb, p, bn, batch, st); });
}

void Builder::conv3(const T4& x, const __half* w, int Cout, const T4& y, const float* bias, const float* row_bias, const __half* residual) {
    if (dry) return;
    const long long M = x.rows();
    int bw = x.w < 128 ? x.w : 128, bh = 128 / bw; if (bh > x.h) bh = x.h; const int bn_img = 128 / (bw * bh);
    if (M % 128 || x.c % 64 || bw * bh * bn_img != 128 || x.w % bw || x.h % bh || x.n % bn_img) {
        // a width that neither divides 128 nor is a multiple of it (96 / 48 / 24 / 12 for 768 x 768 SD), or pixels off the 128-row
        // grid: the spatial-block tiles of conv3_block, which overhang the edges instead of spanning whole rows
        if (x.c % 64) { err = MI3D_ERR_ARG; return; }
        conv3_block(x, w, Cout, y, bias, tc::EPI_PLAIN, nullptr, residual, row_bias);
        return;
    }
    int bn = tc::pick_block_n(Cout, M / 128, num_sms);
    if (!bn) { err = MI3D_ERR_ARG; return; }
    int splits = 1;
    if ((size_t)M * Cout <= splitk_elems) {
        if (Cout % 128 == 0 && (M / 128) * (Cout / 128) * 2 <= num_sms) bn = 128;
        splits = tc::plan_splits((M / 128) * (Cout / bn), 9 * (x.c / 64), num_sms);
    }
    CUtensorMap ma, mb;
    int r = tc::make_map_nhwc(&ma, x.p, x.c, x.w, x.h, x.n, bw, bh, bn_img);
    if (!r) r = tc::make_map_matrix(&mb, w, 9ull * x.c, Cout, 9ull * x.c, bn);
    if (r) { err = r; return; }
    tc::GemmParams p = {};
    p.M = (int)M; p.N = Cout; p.K = 9 * x.c; p.num_k_blocks = 9 * (x.c / 64); p.conv = 1;
    p.conv_H = x.h; p.conv_W = x.w; p.conv_bw = bw; p.conv_bh = bh; p.cin_blocks = x.c / 64;
    p.a_z1 = 1; p.b_z1 = 1; p.b_batched = 0; p.out = y.p; p.ldc = Cout; p.out_z1 = 1;
    p.bias = bias; p.row_bias = row_bias; p.rows_per_group = x.h * x.w; p.residual = residual; p.ld_res = Cout;
    p.epi_mode = tc::EPI_PLAIN; p.alpha = 1.f; p.m_valid = (int)M; p.splits = splits;
    push([this, ma, mb, p, bn](cudaStream_t st) { return timed_launch(ma, mb, p, bn, 1, st); });
}

void Builder::conv3_block(const T4& x, const __half* w, int Cout, const T4& y, const float* bias, int mode, const __half* aux,
                          const __half* residual, const float* row_bias) {
    if (dry) return;
    if (x.c % 64 || Cout % 64 || y.n != x.n || y.h != x.h || y.w != x.w || y.c != Cout) { err = MI3D_ERR_ARG; return; }
    int bw = 128, bh = 1; long long best = -1;
    for (int cw = 8; cw <= 128; cw *= 2) {
        const long long area = (long long)((x.w + cw - 1) / cw) * cw * ((x.h + 128 / cw - 1) / (128 / cw)) * (128 / cw);
        if (best < 0 || area < best) { best = area; bw = cw; bh = 128 / cw; }
    }
    const long long tiles = (long long)x.n * ((x.w + bw - 1) / bw) * ((x.h + bh - 1) / bh);
    const int bn = tc::pick_block_n(Cout, tiles, num_sms, tc::has_block_n_160(mode, 2));
    if (!bn) { err = MI3D_ERR_ARG; return; }
    CUtensorMap ma, mb;
    int r = tc::make_map_nhwc(&ma, x.p, x.c, x.w, x.h, x.n, bw, bh, 1);
    if (!r) r = tc::make_map_matrix(&mb, w, 9ull * x.c, Cout, 9ull * x.c, bn);
    if (r) { err = r; return; }
    tc::GemmParams p = {};
    p.M = (int)(tiles * 128); p.N = Cout; p.K = 9 * x.c; p.num_k_blocks = 9 * (x.c / 64); p.conv = 2;
    p.conv_H = x.h; p.conv_W = x.w; p.conv_bw = bw; p.conv_bh = bh; p.cin_blocks = x.c / 64;
    p.a_z1 = 1; p.b_z1 = 1; p.b_batched = 0; p.out = y.p; p.ldc = Cout; p.out_z1 = 1;
    p.bias = bias; p.row_bias = row_bias; p.rows_per_group = x.h * x.w;          // row_bias: one row per image
    p.epi_mode = mode; p.alpha = 1.f; p.m_valid = (int)x.rows(); p.splits = 1; p.aux = const_cast<__half*>(aux);
    p.residual = residual; p.ld_res = Cout;
    push([this, ma, mb, p, bn](cudaStream_t st) { return timed_launch(ma, mb, p, bn, 1, st); });
}

void Builder::layernorm(const __half* x, long long rows, int C, const float* ga, const float* be, __half* y, float eps) {
    push([=](cudaStream_t st) {
        sdk::k_layernorm<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, y, ga, be, (int)rows, C, eps);
        return (int)cudaGetLastError();
    });
}

void Builder::softmax(__half* s, size_t rows, int cols, int valid, float scale, int causal_tq) {
    push([=](cudaStream_t st) {
        if (causal_tq > 0) clipk::k_softmax_causal<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(s, rows, cols, valid, causal_tq, scale);
        else sdk::k_softmax<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(s, rows, cols, valid, scale);
        return (int)cudaGetLastError();
    });
}

void Builder::layernorm_bwd(const __half* x, const __half* dy, const float* gamma, const __half* add, __half* dx, long long rows, int C, float eps) {
    push([=](cudaStream_t st) {
        clipk::k_layernorm_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, dy, gamma, add, dx, (int)rows, C, eps);
        return (int)cudaGetLastError();
    });
}

void Builder::softmax_bwd(const __half* p, __half* dp, size_t rows, int cols, float scale) {
    push([=](cudaStream_t st) {
        sdk::k_softmax_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(p, dp, rows, cols, scale);
        return (int)cudaGetLastError();
    });
}

void Builder::f32_to_f16(const float* src, __half* dst, size_t n) {
    push([=](cudaStream_t st) {
        sdk::k_f32_to_f16<<<blocks_for(n), 256, 0, st>>>(src, dst, n);
        return (int)cudaGetLastError();
    });
}

void Builder::text_embed(const long long* tokens, const float* tok_emb, const float* pos, __half* x, int B, int L, int Tpad, int C, int vocab) {
    push([=](cudaStream_t st) {
        clipk::k_text_embed<<<blocks_for((size_t)B * Tpad * C / 8), 256, 0, st>>>(tokens, tok_emb, pos, x, B, L, Tpad, C, vocab);
        return (int)cudaGetLastError();
    });
}

__half* Builder::conv3_s2(const T4& x, const __half* w, const T4& y, const float* bias, int pad_lo) {
    const int Ho = y.h, Wo = y.w, C = x.c;
    const long long Mo = (long long)x.n * Ho * Wo;
    __half* col = alloc16((size_t)Mo * 9 * C);
    const T4 xx = x;
    push([=](cudaStream_t st) {
        sdk::k_im2col_s2<<<blocks_for((size_t)Mo * 9 * C / 8), 256, 0, st>>>(xx.p, col, xx.n, xx.h, xx.w, C, Ho, Wo, pad_lo);
        return (int)cudaGetLastError();
    });
    linear(col, Mo, 9 * C, w, y.c, y.p, bias);
    return col;
}

// Persistent grids: as many CTAs per SM as the weight staging area allows.  The staging area exceeds the default 48 KB of dynamic
// shared memory at SD's channel counts; the limits below bound it.
void Builder::conv_small_cin(const T4& x, const float* w, const float* bias, const T4& y) {
    const size_t sm = (size_t)y.c * 9 * x.c * sizeof(float);
    if ((x.c != 4 && x.c != 8) || y.c % 8 || sm > (x.c == 8 ? 200 : 100) * 1024) { err = MI3D_ERR_ARG; return; }
    if (dry) return;
    static const bool attr = [] {
        cudaFuncSetAttribute(sdk::k_conv_small_cin<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(sdk::k_conv_small_cin<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        return true;
    }();
    (void)attr;
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (200 * 1024) / std::max<size_t>(sm, 1)));
    const int grid = (int)std::min<size_t>((y.numel() / 8 + 255) / 256, (size_t)num_sms * per_sm);
    const T4 a = x, o = y;
    push([=](cudaStream_t st) {
        if (a.c == 8) sdk::k_conv_small_cin<8><<<grid, 256, sm, st>>>(a.p, w, bias, o.p, a.n, a.h, a.w, o.c);
        else sdk::k_conv_small_cin<4><<<grid, 256, sm, st>>>(a.p, w, bias, o.p, a.n, a.h, a.w, o.c);
        return (int)cudaGetLastError();
    });
}

void Builder::conv_small_cout(const T4& x, const __half* w, const float* bias, float* out, int cout) {
    if ((cout != 4 && cout != 8) || x.c % 8) { err = MI3D_ERR_ARG; return; }
    if (dry) return;
    static const bool attr = [] {
        cudaFuncSetAttribute(sdk::k_conv_small_cout<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        cudaFuncSetAttribute(sdk::k_conv_small_cout<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        return true;
    }();
    (void)attr;
    const int ppw = x.c <= 128 ? 2 : 1;
    const int grid = (int)std::min<size_t>(((size_t)x.rows() / ppw + 7) / 8 + 1, (size_t)num_sms * 8);
    const size_t sm = (size_t)cout * 9 * x.c * 2;
    const T4 a = x;
    push([=](cudaStream_t st) {
        if (cout == 8) sdk::k_conv_small_cout<8><<<grid, 256, sm, st>>>(a.p, w, bias, out, a.n, a.h, a.w, a.c);
        else sdk::k_conv_small_cout<4><<<grid, 256, sm, st>>>(a.p, w, bias, out, a.n, a.h, a.w, a.c);
        return (int)cudaGetLastError();
    });
}

void Builder::transpose(const __half* in, __half* out, int Z, int R, int C) {
    push([=](cudaStream_t st) {
        sdk::k_transpose<<<dim3((C + 31) / 32, (R + 31) / 32, Z), dim3(32, 8), 0, st>>>(in, out, R, C);
        return (int)cudaGetLastError();
    });
}

void Builder::attention_core(const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv, int B, int T,
                             int Tk, int Tk_valid, int heads, int d, __half* o, int C) {
    if (!attn::supported(d)) { err = MI3D_ERR_ARG; return; }
    if (dry) return;
    attn::Maps m;
    if (int r = attn::make_maps(&m, q, ldq, k, ldk, v, ldv, B, T, Tk, heads, d)) { err = r; return; }
    push([=](cudaStream_t st) {
        if (!profile) return attn::launch(m, o, C, B, T, Tk_valid, heads, st);
        // profiling: same event bracket as the tile kernel; recorded with conv = 2 (M = queries, N = keys, K = head_dim, batch = B * heads)
        if (prof_used == prof_events.size()) { cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); prof_events.push_back({a, b}); }
        if (prof_shapes.size() < prof_events.size()) prof_shapes.resize(prof_events.size());
        prof_shapes[prof_used] = {T, Tk_valid, d, 0, 1, 2, B * heads, 0};
        auto& ev = prof_events[prof_used++];
        cudaEventRecord(ev.first, st);
        const int r = attn::launch(m, o, C, B, T, Tk_valid, heads, st);
        cudaEventRecord(ev.second, st);
        return r;
    });
}

int Builder::run_eager(std::vector<Op>& ops, cudaStream_t st) {
    for (auto& op : ops) { int r = op(st); if (r) return r; }
    return MI3D_OK;
}

int Builder::run(std::vector<Op>& ops, cudaStream_t st) {
    ListGraph& g = graphs[&ops];
    if (!use_graph || profile || g.failed) return run_eager(ops, st);
    if (g.exec) return (int)cudaGraphLaunch(g.exec, st);
    if (g.calls++ == 0) return run_eager(ops, st);            // first call: plain launches (one-time function attributes, warm caches)
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); g.failed = true; return run_eager(ops, st); }
    const int r = run_eager(ops, st);
    const cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (r || ce != cudaSuccess || !graph || cudaGraphInstantiate(&g.exec, graph, 0) != cudaSuccess) {
        cudaGetLastError(); g.failed = true; g.exec = nullptr;
        if (graph) cudaGraphDestroy(graph);
        return r ? r : run_eager(ops, st);
    }
    cudaGraphDestroy(graph);
    return (int)cudaGraphLaunch(g.exec, st);
}

Builder::~Builder() { for (auto& kv : graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec); }

}  // namespace plan
