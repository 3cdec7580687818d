// dpt_engine.cu -- the DPT-Hybrid depth model (C ABI: include/mi3d.h, section B8).
//
// What the reference's `DPTDepthModel(backbone="vitb_rn50_384", non_negative=True)` computes (main.py:111-127, 196-214) for one
// normalised 384 x 384 image: a ResNet-50v2 trunk with weight-standardised convs and GroupNorm, a 12-layer ViT-B/16 on its 24 x 24
// features (577 tokens), the reassemble stage, four RefineNet fusion blocks and the depth head (oracle/dpt_ref.py restates it).  One
// statically planned list of launches: the tile GEMM for every 1x1 conv and linear (a stride-2 3x3 conv goes through Builder::conv3_s2),
// its spatial-block mode for the stride-1 3x3 convs, the pre-LN blocks of transformer_plan.cuh with fused attention and the EPI_GELU
// epilogue, and the memory-bound kernels below.  Activations NHWC fp16, statistics and accumulation fp32, GEMM weights fp16 (norms,
// biases, cls / pos_embed and the final 32 -> 1 conv fp32).  Forward only, at the reference's one shape.  No split-K and no atomics:
// the output is bit-identical run to run.
#include "transformer_plan.cuh"
#include "warp_reduce.cuh"

namespace dptk {
namespace {

__device__ __forceinline__ float block_sum(float v, float* red) {       // fixed-order reduction over the block (blockDim.x <= 1024)
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float s = 0.f;
    if (w == 0) {
        s = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.f;
        s = warp_sum(s);
        if (lane == 0) red[32] = s;
    }
    __syncthreads();
    return red[32];
}

// Weight standardisation, once at load: w [O][I][KK] fp32 -> (w - mean) / sqrt(var + 1e-8) stored [O][KK][I] fp16 (the implicit-GEMM
// K order: tap-major, then input channel).  Per output channel, biased variance, two passes in fp32.  This is the batch-norm form of
// timm's StdConv2dSame(eps=1e-8) that transformers' BiT uses; timm 0.4.5 may compute (w - mean) / (std + eps) instead, which differs by
// a per-channel scale of order 1e-8 / std, far below fp16 storage error and removed anyway by the GroupNorm after every such conv.
__global__ void k_ws_conv(const float* __restrict__ src, __half* __restrict__ dst, int I, int KK) {
    __shared__ float red[33];
    const int o = blockIdx.x, n = I * KK;
    const float* w = src + (size_t)o * n;
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += w[i];
    const float mean = block_sum(s, red) / n;
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float d = w[i] - mean; ss += d * d; }
    const float rstd = 1.f / sqrtf(block_sum(ss, red) / n + 1e-8f);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ci = i / KK, k = i % KK;
        dst[(size_t)o * n + (size_t)k * I + ci] = __float2half_rn((w[i] - mean) * rstd);
    }
}

// Stem: 7x7 stride-2 conv 3 -> 64 on the fp32 NCHW image, TF-"same" padding (2 before, 3 after): 384^2 -> 192^2 NHWC fp16.
// w: [64][7][7][3] fp16 (standardised), staged as fp32 [tap * 3 + ci][co].  One thread per (pixel, 8 output channels).
__global__ void k_stem(const float* __restrict__ img, const __half* __restrict__ w, __half* __restrict__ out) {
    __shared__ float ws[147][64];
    for (int i = threadIdx.x; i < 64 * 147; i += blockDim.x) ws[i % 147][i / 147] = __half2float(w[i]);
    __syncthreads();
    constexpr int H = 384, Ho = 192;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < Ho * Ho * 8; idx += gridDim.x * blockDim.x) {
        const int cv = idx & 7, p = idx >> 3, oy = p / Ho, ox = p % Ho;
        float acc[8];
        #pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0.f;
        for (int ky = 0; ky < 7; ky++) {
            const int iy = 2 * oy + ky - 2;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 7; kx++) {
                const int ix = 2 * ox + kx - 2;
                if (ix < 0 || ix >= H) continue;
                #pragma unroll
                for (int ci = 0; ci < 3; ci++) {
                    const float v = __ldg(img + ((size_t)ci * H + iy) * H + ix);
                    const float* wr = &ws[(ky * 7 + kx) * 3 + ci][cv * 8];
                    #pragma unroll
                    for (int j = 0; j < 8; j++) acc[j] = fmaf(v, wr[j], acc[j]);
                }
            }
        }
        __align__(16) __half o[8];
        #pragma unroll
        for (int j = 0; j < 8; j++) o[j] = __float2half_rn(acc[j]);
        *reinterpret_cast<uint4*>(out + (size_t)p * 64 + cv * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// GroupNorm (batch 1, G = gridDim.x groups, one CTA per group) with the trunk's epilogues:
// y = [relu](gn(x) [+ res]).  Mean, then the variance about it, in fp32 with a fixed reduction order.
__global__ void k_gn(const __half* __restrict__ x, __half* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const __half* __restrict__ res, int HW, int C, float eps, int relu) {
    __shared__ float red[33];
    const int g = blockIdx.x, cpg = C / gridDim.x;
    const int n = HW * cpg;
    auto at = [&](int e) { return (size_t)(e / cpg) * C + g * cpg + e % cpg; };
    float s = 0.f;
    for (int e = threadIdx.x; e < n; e += blockDim.x) s += __half2float(x[at(e)]);
    const float mean = block_sum(s, red) / n;
    float ss = 0.f;
    for (int e = threadIdx.x; e < n; e += blockDim.x) { const float d = __half2float(x[at(e)]) - mean; ss += d * d; }
    const float rstd = rsqrtf(block_sum(ss, red) / n + eps);
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const size_t o = at(e); const int c = g * cpg + e % cpg;
        float v = (__half2float(x[o]) - mean) * rstd * gamma[c] + beta[c];
        if (res) v += __half2float(res[o]);
        if (relu) v = fmaxf(v, 0.f);
        y[o] = __float2half_rn(v);
    }
}

// 3x3 stride-2 max-pool, TF-"same" padding on an even input (0 before, 1 after, the pad never wins): [H][W][C] -> [H/2][W/2][C]
__global__ void k_maxpool_s2(const __half* __restrict__ in, __half* __restrict__ out, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, vc = C / 8;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Ho * Wo * vc; i += gridDim.x * blockDim.x) {
        const int v = i % vc, p = i / vc, oy = p / Wo, ox = p % Wo;
        float m[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) m[k] = -INFINITY;
        for (int y = 2 * oy; y < min(2 * oy + 3, H); y++)
            for (int x = 2 * ox; x < min(2 * ox + 3, W); x++) {
                const uint4 raw = *reinterpret_cast<const uint4*>(in + ((size_t)y * W + x) * C + v * 8);
                const __half* h = reinterpret_cast<const __half*>(&raw);
                #pragma unroll
                for (int k = 0; k < 8; k++) m[k] = fmaxf(m[k], __half2float(h[k]));
            }
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(m[k]);
        *reinterpret_cast<uint4*>(out + (size_t)i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// the input of a 1x1 stride-2 conv ("same" padding is zero there): out[y][x] = in[2y][2x]
__global__ void k_subsample2(const __half* __restrict__ in, __half* __restrict__ out, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, vc = C / 8;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Ho * Wo * vc; i += gridDim.x * blockDim.x) {
        const int v = i % vc, p = i / vc, oy = p / Wo, ox = p % Wo;
        *reinterpret_cast<uint4*>(out + (size_t)i * 8) = *reinterpret_cast<const uint4*>(in + ((size_t)(2 * oy) * W + 2 * ox) * C + v * 8);
    }
}

// token row 0: cls_token + pos_embed[0]
__global__ void k_cls_row(const float* __restrict__ cls, const float* __restrict__ pos, __half* __restrict__ x, int C) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) x[c] = __float2half_rn(cls[c] + pos[c]);
}

// The readout projection's cls half as a per-image bias: bb[n] = b[n] + sum_k W[n][C + k] cls[k], W [C][2C] fp16.  One warp per n.
__global__ void k_cls_bias(const __half* __restrict__ W, const float* __restrict__ b, const __half* __restrict__ cls, float* __restrict__ bb, int C) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= C) return;
    const __half* wr = W + (size_t)n * 2 * C + C;
    float s = 0.f;
    for (int k = lane; k < C; k += 32) s = fmaf(__half2float(wr[k]), __half2float(cls[k]), s);
    s = warp_sum(s);
    if (lane == 0) bb[n] = b[n] + s;
}

// The residual conv unit's input pass: rx = relu(x1) and, for a fusion block's first unit, s = x0 + x1 (its residual).  8 per thread.
__global__ void k_relu_add(const __half* __restrict__ x1, const __half* __restrict__ x0, __half* __restrict__ rx, __half* __restrict__ s, size_t nvec) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 a = *reinterpret_cast<const uint4*>(x1 + i * 8);
        const __half* ha = reinterpret_cast<const __half*>(&a);
        __align__(16) __half r[8], o[8];
        uint4 b = make_uint4(0, 0, 0, 0);
        if (x0) b = *reinterpret_cast<const uint4*>(x0 + i * 8);
        const __half* hb = reinterpret_cast<const __half*>(&b);
        #pragma unroll
        for (int k = 0; k < 8; k++) {
            const float v = __half2float(ha[k]);
            r[k] = __float2half_rn(fmaxf(v, 0.f));
            o[k] = __float2half_rn(v + __half2float(hb[k]));
        }
        *reinterpret_cast<uint4*>(rx + i * 8) = *reinterpret_cast<const uint4*>(r);
        if (x0) *reinterpret_cast<uint4*>(s + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// bilinear x2 upsample, align_corners=True, NHWC fp16 [H][W][C] -> [2H][2W][C]; source coordinates and weights as PyTorch computes them
__global__ void k_up2_ac(const __half* __restrict__ in, __half* __restrict__ out, int H, int W, int C) {
    const int Ho = 2 * H, Wo = 2 * W, vc = C / 8;
    const float sy = (float)(H - 1) / (float)(Ho - 1), sx = (float)(W - 1) / (float)(Wo - 1);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)Ho * Wo * vc; i += (size_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vc); const int p = (int)(i / vc), oy = p / Wo, ox = p % Wo;
        const float fy = sy * oy, fx = sx * ox;
        const int y0 = (int)fy, x0 = (int)fx, y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
        const float ly = fy - y0, lx = fx - x0;
        auto ld = [&](int y, int x) { return *reinterpret_cast<const uint4*>(in + ((size_t)y * W + x) * C + v * 8); };
        const uint4 a = ld(y0, x0), b = ld(y0, x1), c = ld(y1, x0), d = ld(y1, x1);
        const __half *ha = reinterpret_cast<const __half*>(&a), *hb = reinterpret_cast<const __half*>(&b),
                     *hc = reinterpret_cast<const __half*>(&c), *hd = reinterpret_cast<const __half*>(&d);
        __align__(16) __half o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++)
            o[k] = __float2half_rn((1.f - ly) * ((1.f - lx) * __half2float(ha[k]) + lx * __half2float(hb[k])) +
                                   ly * ((1.f - lx) * __half2float(hc[k]) + lx * __half2float(hd[k])));
        *reinterpret_cast<uint4*>(out + i * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

// the head's last conv: out[p] = relu(b + sum_{c < 32} w[c] h[p][c]) in fp32; h rows are 64 wide (channels 32.. are the zero padding)
__global__ void k_head_out(const __half* __restrict__ h, const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ out, int P) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
        float s = b[0];
        #pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint4 raw = *reinterpret_cast<const uint4*>(h + (size_t)p * 64 + q * 8);
            const __half* hv = reinterpret_cast<const __half*>(&raw);
            #pragma unroll
            for (int k = 0; k < 8; k++) s = fmaf(w[q * 8 + k], __half2float(hv[k]), s);
        }
        out[p] = fmaxf(s, 0.f);
    }
}

// taps: NHWC fp16 [HW][C] -> NCHW fp32 [C][HW]
__global__ void k_nhwc_to_nchw_f32(const __half* __restrict__ in, float* __restrict__ out, int HW, int C) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)HW * C; i += (size_t)gridDim.x * blockDim.x)
        out[i] = __half2float(in[(i % HW) * C + i / HW]);
}

}  // namespace
}  // namespace dptk

namespace dpt {

using namespace plan;
constexpr int kC = 768, kGrid = 24, kT = 577, kImg = 384;

struct Engine : TowerBuilder {
    Tower t;
    std::vector<BlockW> w;
    std::vector<BlockA> a;
    float* img = nullptr;
    float* out = nullptr;
    T4 taps[4];
    std::vector<Op> fwd;

    static unsigned grid(size_t n) { return (unsigned)blocks_for(n); }
    void launch(std::function<void(cudaStream_t)> f) {
        push([f](cudaStream_t st) { f(st); return (int)cudaGetLastError(); });
    }

    const __half* conv_ws(const std::string& name, int cin, int cout, int k) {
        return (const __half*)param(name, {cout, cin, k, k}, PK_CONV_WS).dst;
    }
    const __half* conv3w(const std::string& name, int cin, int cout) {
        return (const __half*)param(name, {cout, cin, 3, 3}, PK_CONV3).dst;
    }
    const __half* lin_w(const std::string& name, std::vector<int> shape) { return (const __half*)param(name, shape, PK_LINEAR).dst; }

    void gn(const T4& x, const T4& y, const std::string& name, const __half* res, bool relu) {
        const float* ga = pf(name + ".weight", {x.c}); const float* be = pf(name + ".bias", {x.c});
        const __half* xp = x.p; __half* yp = y.p; const int HW = x.h * x.w, C = x.c;
        launch([=](cudaStream_t st) { dptk::k_gn<<<32, 1024, 0, st>>>(xp, yp, ga, be, res, HW, C, 1e-5f, relu ? 1 : 0); });
    }
    void conv1x1(const T4& x, const __half* wt, const T4& y, const float* bias = nullptr) { linear(x.p, x.rows(), x.c, wt, y.c, y.p, bias); }

    T4 bottleneck(const T4& x, const std::string& p, int mid, int cout, int stride, bool first) {
        const int Ho = x.h / stride, Wo = x.w / stride;
        const __half* sc = x.p;
        if (first) {
            const __half* wd = conv_ws(p + "downsample.conv.weight", x.c, cout, 1);
            T4 xs = x;
            if (stride == 2) {
                xs = act(1, Ho, Wo, x.c);
                const __half* xp = x.p; __half* o = xs.p; const int H = x.h, W = x.w, C = x.c;
                launch([=](cudaStream_t st) { dptk::k_subsample2<<<grid((size_t)Ho * Wo * C / 8), 256, 0, st>>>(xp, o, H, W, C); });
            }
            T4 d = act(1, Ho, Wo, cout), dn = act(1, Ho, Wo, cout);
            conv1x1(xs, wd, d);
            gn(d, dn, p + "downsample.norm", nullptr, false);
            sc = dn.p;
        }
        T4 a1 = act(1, x.h, x.w, mid), a1n = act(1, x.h, x.w, mid);
        conv1x1(x, conv_ws(p + "conv1.weight", x.c, mid, 1), a1);
        gn(a1, a1n, p + "norm1", nullptr, true);
        T4 a2 = act(1, Ho, Wo, mid), a2n = act(1, Ho, Wo, mid);
        const __half* w2 = conv_ws(p + "conv2.weight", mid, mid, 3);
        if (stride == 2) conv3_s2(a1n, w2, a2, nullptr, 0);
        else conv3_block(a1n, w2, mid, a2, nullptr, tc::EPI_PLAIN);
        gn(a2, a2n, p + "norm2", nullptr, true);
        T4 a3 = act(1, Ho, Wo, cout), o = act(1, Ho, Wo, cout);
        conv1x1(a2n, conv_ws(p + "conv3.weight", mid, cout, 1), a3);
        gn(a3, o, p + "norm3", sc, true);
        return o;
    }

    // layer_3 / layer_4: GELU(Linear([tokens | cls])) -> 1x1 conv (-> 3x3/2 conv); the cls half of the Linear is a per-image bias
    T4 reassemble(const __half* tok, int k) {
        const std::string q = "pretrained.act_postprocess" + std::to_string(k) + ".";
        const __half* wr = lin_w(q + "0.project.0.weight", {kC, 2 * kC});
        const float* br = pf(q + "0.project.0.bias", {kC});
        float* bb = alloc32(kC);
        launch([=](cudaStream_t st) { dptk::k_cls_bias<<<kC / 8, 256, 0, st>>>(wr, br, tok, bb, kC); });
        T4 g = act(1, kGrid, kGrid, kC);
        {
            Mat ma{tok + kC, kC, kGrid * kGrid, kC}; Mat mb{wr, 2 * kC, kC, kC};
            Out o; o.p16 = g.p; o.ldc = kC;
            Epi e; e.bias = bb; e.mode = tc::EPI_GELU;
            gemm(ma, mb, kC, o, e);
        }
        T4 l = act(1, kGrid, kGrid, kC);
        const __half* w3 = lin_w(q + "3.weight", {kC, kC, 1, 1});
        conv1x1(g, w3, l, pf(q + "3.bias", {kC}));
        if (k == 3) return l;
        T4 l4 = act(1, kGrid / 2, kGrid / 2, kC);
        const __half* w4 = conv3w(q + "4.weight", kC, kC);
        conv3_s2(l, w4, l4, pf(q + "4.bias", {kC}), 1);
        return l4;
    }

    // x0 + x + conv2(relu(conv1(relu(x)))) (x0 null: x + ...)
    T4 rcu(const T4& x, const std::string& n, const __half* x0) {
        T4 rx = act(x.n, x.h, x.w, x.c), s = x0 ? act(x.n, x.h, x.w, x.c) : x;
        const __half* xp = x.p; __half *rp = rx.p, *sp = s.p; const size_t nv = x.numel() / 8;
        launch([=](cudaStream_t st) { dptk::k_relu_add<<<grid(nv), 256, 0, st>>>(xp, x0, rp, sp, nv); });
        T4 c1 = act(x.n, x.h, x.w, 256), o = act(x.n, x.h, x.w, 256);
        const __half* w1 = conv3w(n + ".conv1.weight", 256, 256); const float* b1 = pf(n + ".conv1.bias", {256});
        conv3_block(rx, w1, 256, c1, b1, tc::EPI_RELU);
        const __half* w2 = conv3w(n + ".conv2.weight", 256, 256); const float* b2 = pf(n + ".conv2.bias", {256});
        conv3_block(c1, w2, 256, o, b2, tc::EPI_PLAIN, nullptr, s.p);
        return o;
    }
    void up2(const T4& x, const T4& y) {
        const __half* xp = x.p; __half* yp = y.p; const int H = x.h, W = x.w, C = x.c;
        launch([=](cudaStream_t st) { dptk::k_up2_ac<<<grid(y.numel() / 8), 256, 0, st>>>(xp, yp, H, W, C); });
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); named.clear();
        splitk_elems = 0;                         // no split-K: its fp32 RED order would make results vary run to run
        fwd.clear(); cur = &fwd;
        const std::string M = "pretrained.model.", B = M + "patch_embed.backbone.";
        const float* cls = pf(M + "cls_token", {1, 1, kC});
        const float* pos = pf(M + "pos_embed", {1, kT, kC});
        img = alloc32((size_t)3 * kImg * kImg);
        // ---- trunk ----
        T4 s0 = act(1, 192, 192, 64), s1 = act(1, 192, 192, 64), x = act(1, 96, 96, 64);
        {
            const __half* ws = conv_ws(B + "stem.conv.weight", 3, 64, 7);
            const float* im = img; __half* o = s0.p;
            launch([=](cudaStream_t st) { dptk::k_stem<<<num_sms * 2, 256, 0, st>>>(im, ws, o); });
            gn(s0, s1, B + "stem.norm", nullptr, true);
            const __half* ip = s1.p; __half* xp = x.p;
            launch([=](cudaStream_t st) { dptk::k_maxpool_s2<<<grid(96 * 96 * 8), 256, 0, st>>>(ip, xp, 192, 192, 64); });
        }
        const int mids[3] = {64, 128, 256}, outs[3] = {256, 512, 1024}, depths[3] = {3, 4, 9};
        for (int s = 0; s < 3; s++) {
            for (int i = 0; i < depths[s]; i++)
                x = bottleneck(x, B + "stages." + std::to_string(s) + ".blocks." + std::to_string(i) + ".", mids[s], outs[s],
                               (s > 0 && i == 0) ? 2 : 1, i == 0);
            if (s < 2) taps[s] = x;
        }
        // ---- tokens: row 0 = cls + pos[0], rows 1..576 = proj(features) + bias + pos[1..]; rows 577.. stay zero (finite) ----
        t.C = kC; t.L = 12; t.heads = 12; t.T = kT; t.Tpad = pad64(kT); t.ln_eps = 1e-6f;
        const long long Mt = t.Tpad;
        std::vector<__half*> r(t.L + 1);
        for (auto& p : r) p = alloc16((size_t)Mt * kC);
        {
            const __half* wp = lin_w(M + "patch_embed.proj.weight", {kC, 1024, 1, 1});
            const float* bp = pf(M + "patch_embed.proj.bias", {kC});
            __half* x0 = r[0];
            launch([=](cudaStream_t st) { dptk::k_cls_row<<<1, 256, 0, st>>>(cls, pos, x0, kC); });
            Mat ma{x.p, 1024, kGrid * kGrid, 1024}; Mat mb{wp, 1024, kC, 1024};
            Out o; o.p16 = r[0] + kC; o.ldc = kC;
            Epi e; e.bias = bp; e.row_bias = pos + kC; e.rows_per_group = 1;
            gemm(ma, mb, kC, o, e);
        }
        // ---- ViT-B/16: 12 pre-LN blocks, fused attention over the 577 valid keys ----
        w.assign(t.L, BlockW());
        BlockA s;
        s.ln1 = alloc16(Mt * kC); s.qkv = alloc16(Mt * 3 * kC); s.qkvT = nullptr; s.S = nullptr; s.ao = alloc16(Mt * kC);
        s.h = alloc16(Mt * kC); s.ln2 = alloc16(Mt * kC); s.pre = nullptr; s.act = alloc16(Mt * 4 * kC);
        a.assign(t.L, s);
        for (int i = 0; i < t.L; i++) {
            const std::string p = M + "blocks." + std::to_string(i) + ".";
            BlockW& bw = w[i];
            bw.ln1 = pf(p + "norm1.weight", {kC}); bw.ln1_b = pf(p + "norm1.bias", {kC});
            bw.w_in = lin_w(p + "attn.qkv.weight", {3 * kC, kC}); bw.b_in = pf(p + "attn.qkv.bias", {3 * kC});
            bw.w_out = lin_w(p + "attn.proj.weight", {kC, kC}); bw.b_out = pf(p + "attn.proj.bias", {kC});
            bw.ln2 = pf(p + "norm2.weight", {kC}); bw.ln2_b = pf(p + "norm2.bias", {kC});
            bw.w_fc = lin_w(p + "mlp.fc1.weight", {4 * kC, kC}); bw.b_fc = pf(p + "mlp.fc1.bias", {4 * kC});
            bw.w_proj = lin_w(p + "mlp.fc2.weight", {kC, 4 * kC}); bw.b_proj = pf(p + "mlp.fc2.bias", {kC});
            bw.t_in = bw.t_out = bw.t_fc = bw.t_proj = nullptr;
            a[i].x = r[i]; a[i].out = r[i + 1];
            block_fwd(t, bw, a[i], 1, 0, tc::EPI_GELU);
        }
        // ---- reassemble (hooks: blocks 8 and 11) ----
        taps[2] = reassemble(r[9], 3);
        taps[3] = reassemble(r[12], 4);
        // ---- decoder ----
        const int cins[4] = {256, 512, kC, kC};
        T4 rn[4];
        for (int k = 0; k < 4; k++) {
            rn[k] = act(1, taps[k].h, taps[k].w, 256);
            conv3_block(taps[k], conv3w("scratch.layer" + std::to_string(k + 1) + "_rn.weight", cins[k], 256), 256, rn[k], nullptr, tc::EPI_PLAIN);
        }
        T4 path;
        for (int k = 4; k >= 1; k--) {
            const std::string q = "scratch.refinenet" + std::to_string(k) + ".";
            T4 v = rn[k - 1];
            if (k < 4) v = rcu(v, q + "resConfUnit1", path.p);
            v = rcu(v, q + "resConfUnit2", nullptr);
            // out_conv (1x1) before the align-corners upsample: they commute exactly (the bilinear weights sum to 1), at 4x less work
            T4 oc = act(1, v.h, v.w, 256);
            const __half* wo = lin_w(q + "out_conv.weight", {256, 256, 1, 1});
            conv1x1(v, wo, oc, pf(q + "out_conv.bias", {256}));
            path = act(1, 2 * v.h, 2 * v.w, 256);
            up2(oc, path);
        }
        // ---- head: 3x3 256->128, bilinear x2, 3x3 128->32 + ReLU (Cout padded to 64 with zero weights / bias), 1x1 32->1 + ReLU ----
        T4 h1 = act(1, 192, 192, 128), h1u = act(1, kImg, kImg, 128), h2 = act(1, kImg, kImg, 64);
        const __half* w0 = conv3w("scratch.output_conv.0.weight", 256, 128);     // registered in state_dict order: weight, then bias
        conv3_block(path, w0, 128, h1, pf("scratch.output_conv.0.bias", {128}), tc::EPI_PLAIN);
        up2(h1, h1u);
        __half* w2 = alloc16((size_t)64 * 9 * 128);
        float* b2 = alloc32(64);
        param_view("scratch.output_conv.2.weight", {32, 128, 3, 3}, PK_CONV3, w2);
        param_view("scratch.output_conv.2.bias", {32}, PK_F32, b2);
        conv3_block(h1u, w2, 64, h2, b2, tc::EPI_RELU);
        const float* w4 = pf("scratch.output_conv.4.weight", {1, 32, 1, 1});
        const float* b4 = pf("scratch.output_conv.4.bias", {1});
        out = alloc32((size_t)kImg * kImg);
        {
            const __half* hp = h2.p; float* o = out;
            launch([=](cudaStream_t st) { dptk::k_head_out<<<grid(kImg * kImg), 256, 0, st>>>(hp, w4, b4, o, kImg * kImg); });
        }
        cur = nullptr;
        return err;
    }

    int load_param(const Param& P, const float* src, const float* partner, cudaStream_t st) override {
        if (P.kind != PK_CONV_WS) return Builder::load_param(P, src, partner, st);
        dptk::k_ws_conv<<<P.shape[0], 256, 0, st>>>(src, (__half*)P.dst, P.shape[1], P.shape[2] * P.shape[3]);
        return (int)cudaGetLastError();
    }
};

}  // namespace dpt

extern "C" {

size_t mi3d_dpt_workspace_bytes(void) { return plan::workspace_bytes<dpt::Engine>(); }

mi3d_engine_t mi3d_dpt_create(void* workspace, size_t workspace_bytes) { return plan::create<dpt::Engine>(workspace, workspace_bytes); }

int mi3d_dpt_forward(mi3d_engine_t h, const float* img, float* out, mi3d_stream_t stream) {
    dpt::Engine* ep = plan::engine_of<dpt::Engine>(h);
    if (!ep || !img || !out) return MI3D_ERR_ARG;
    dpt::Engine& e = *ep;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemcpyAsync(e.img, img, (size_t)3 * dpt::kImg * dpt::kImg * sizeof(float), cudaMemcpyDeviceToDevice, st));
    int r = e.run_eager(e.fwd, st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(out, e.out, (size_t)dpt::kImg * dpt::kImg * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return MI3D_OK;
}

int mi3d_dpt_tap(mi3d_engine_t h, int i, float* dst, mi3d_stream_t stream) {
    dpt::Engine* ep = plan::engine_of<dpt::Engine>(h);
    if (!ep || !dst || i < 0 || i > 3) return MI3D_ERR_ARG;
    const plan::T4& t = ep->taps[i];
    const size_t n = t.numel();
    dptk::k_nhwc_to_nchw_f32<<<plan::Builder::blocks_for(n), 256, 0, (cudaStream_t)stream>>>(t.p, dst, t.h * t.w, t.c);
    return (int)cudaGetLastError();
}

}  // extern "C"
