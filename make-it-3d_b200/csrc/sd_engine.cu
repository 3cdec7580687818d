// sd_engine.cu -- Stable-Diffusion guidance engine for the SDS step (C ABI: include/mi3d.h, section B3).
//
// Replaces what nerf/sd.py:117-174,212-220 runs inside diffusers (UNet2DConditionModel, AutoencoderKL.encode,
// DDIMScheduler.add_noise) with a statically planned list of launches over ONE tensor-core tile kernel
// (tc_gemm.cuh: wgmma / TMA) plus the memory-bound kernels of sd_kernels.cuh:
//   * every Linear, 1x1 conv, attention product and im2col'ed strided conv   -> tc plain GEMM
//   * every 3x3 stride-1 conv (U-Net ResBlocks, VAE encoder, their dgrads)   -> tc implicit GEMM (TMA-shifted taps)
//   * GroupNorm(+SiLU), LayerNorm, softmax, GEGLU (GEMM epilogue), time-embedding, CFG + SDS gradient -> sdk kernels
// The plan (buffers in a caller-provided workspace, TMA descriptors, launch parameters) is built once at
// mi3d_sd_create(); a step is a fixed sequence of launches on the caller's stream -> CUDA-graph capturable.
// Activations: NHWC fp16.  Accumulation / statistics: fp32 (fp64 group sums).  Weights: fp16 copies of the fp32
// diffusers parameters, re-laid-out at load time (conv OIHW -> O,ky,kx,I ; GEGLU rows interleaved ; dgrad copies).
#include "engine_plan.cuh"
#include "sd_kernels.cuh"

namespace sd {

using namespace plan;

// ------------------------------------------------------------------------------------------------------------
// Sampling step kernels (mi3d_sd_sample).  Both run as ONE CTA: the step index is read by every thread and advanced after a
// barrier, so no launch in the replayed list depends on a host-side argument.
// ------------------------------------------------------------------------------------------------------------
constexpr int kMaxSampleSteps = 1000;                     // num_train_timesteps: set_timesteps accepts n <= T
struct SampleState { int step; int pred_type; float gs; int pad; };

// call head: the caller's schedule and x_T into the engine's buffers, step index 0
__global__ void k_sample_begin(const mi3d_sd_schedule* __restrict__ sched, int n, const float* __restrict__ x, mi3d_sd_schedule* __restrict__ tab,
                               float* __restrict__ lat, int count, SampleState* __restrict__ s, int pred_type, float gs) {
    const int stride = gridDim.x * blockDim.x;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(count, n); i += stride) {
        if (i < count) lat[i] = x[i];
        if (i < n) tab[i] = sched[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *s = SampleState{0, pred_type, gs, 0};
}

// step head: t_i into the U-Net's timestep slot; U-Net input [x, x] NHWC fp16 from the fp32 NCHW latents (no noise added)
__global__ void __launch_bounds__(1024) k_sample_in(const mi3d_sd_schedule* __restrict__ tab, const SampleState* __restrict__ s,
                                                    const float* __restrict__ lat, __half* __restrict__ xin, long long* __restrict__ tslot, int pix) {
    const int step = s->step;
    if (threadIdx.x == 0) *tslot = tab[step].t;
    for (int i = threadIdx.x; i < pix; i += blockDim.x) {
        __align__(8) __half o[4];
        #pragma unroll
        for (int c = 0; c < 4; c++) o[c] = __float2half_rn(lat[(size_t)c * pix + i]);
        *reinterpret_cast<uint2*>(xin + (size_t)i * 4) = *reinterpret_cast<const uint2*>(o);
        *reinterpret_cast<uint2*>(xin + ((size_t)pix + i) * 4) = *reinterpret_cast<const uint2*>(o);
    }
}

// step tail: CFG as nerf/sd.py:193-194 writes it, then DDIMScheduler.step with eta 0 and clip_sample off:
//   epsilon:      x0 = (x - sqrt(1 - a_t) e) / sqrt(a_t),   eps = e
//   v_prediction: x0 = sqrt(a_t) x - sqrt(1 - a_t) e,       eps = sqrt(a_t) e + sqrt(1 - a_t) x
//   x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps; in place, then the step index advances
__global__ void __launch_bounds__(1024) k_sample_step(const float* __restrict__ unet_out /*[2][pix][4]*/, const mi3d_sd_schedule* __restrict__ tab,
                                                      SampleState* __restrict__ s, float* __restrict__ lat, int pix) {
    const int step = s->step, v = s->pred_type;
    const float gs = s->gs, a_t = tab[step].alpha_t, a_p = tab[step].alpha_prev;
    const float sa = sqrtf(a_t), sb = sqrtf(1.f - a_t), sp = sqrtf(a_p), sq = sqrtf(1.f - a_p);
    for (int i = threadIdx.x; i < pix; i += blockDim.x) {
        const float4 un = *reinterpret_cast<const float4*>(unet_out + (size_t)i * 4);
        const float4 tx = *reinterpret_cast<const float4*>(unet_out + ((size_t)pix + i) * 4);
        const float u4[4] = {un.x, un.y, un.z, un.w}, t4[4] = {tx.x, tx.y, tx.z, tx.w};
        #pragma unroll
        for (int c = 0; c < 4; c++) {
            const float e = t4[c] + gs * (t4[c] - u4[c]);
            const float x = lat[(size_t)c * pix + i];
            const float x0 = v ? sa * x - sb * e : (x - sb * e) / sa;
            const float eps = v ? sa * e + sb * x : e;
            lat[(size_t)c * pix + i] = sp * x0 + sq * eps;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) s->step = step + 1;
}

// dx of Builder::conv3_s2 from the gradient of its im2col matrix (grid-stride over dx's 8-channel vectors)
int col2im_s2(const __half* dcol, __half* dx, int N, int H, int W, int C, int Ho, int Wo, int pad_lo, cudaStream_t st) {
    sdk::k_col2im_s2<<<Builder::blocks_for((size_t)N * H * W * C / 8), 256, 0, st>>>(dcol, dx, N, H, W, C, Ho, Wo, pad_lo);
    return (int)cudaGetLastError();
}

struct Engine : Builder {
    mi3d_unet_cfg ucfg; mi3d_vae_cfg vcfg;
    // either part may be absent (NULL); a VAE-only engine takes its GroupNorm group count from the VAE
    Engine(const mi3d_unet_cfg* u, const mi3d_vae_cfg* v) : ucfg(u ? *u : mi3d_unet_cfg{}), vcfg(v ? *v : mi3d_vae_cfg{}) {
        if (v && !u) ucfg.groups = v->groups;
    }
    std::vector<Op> unet_ops, enc_ops, enc_bwd_ops;
    // GroupNorm statistics of one op list live in one pool, cleared by a single memset at the head of the list.  Each GroupNorm takes
    // 2 * n * groups doubles, so the pool grows with the batch: a measuring pass of build() records what each list needs, and the pool is
    // that size, at least kPoolBytes (so a batch-2 U-Net / one-image VAE keeps the buffer offsets it always had).
    uint8_t* pool = nullptr; size_t pool_used = 0, pool_cap = 0; static constexpr size_t kPoolBytes = 256 * 1024;
    bool measuring = false; std::map<const std::vector<Op>*, size_t> pool_need;
    void begin_list(std::vector<Op>* l) {
        cur = l; pool_cap = std::max(kPoolBytes, pool_need[l]); pool = (uint8_t*)alloc(pool_cap); pool_used = 0;
        uint8_t* pp = pool; const size_t bytes = pool_cap;
        push([pp, bytes](cudaStream_t st) { return (int)cudaMemsetAsync(pp, 0, bytes, st); });
    }
    double* pool_stats(size_t n_doubles) {
        const size_t b = n_doubles * sizeof(double);
        if (measuring) pool_need[cur] = pool_used + b;
        else if (pool_used + b > pool_cap) { err = MI3D_ERR_ARG; return (double*)pool; }
        double* p = (double*)(pool + pool_used); pool_used += b; return p;
    }
    // per-ResBlock time-embedding projections of the whole U-Net, evaluated by one grouped launch right after the embedding MLP
    std::vector<sdk::SmallLinearJob> temb_jobs; sdk::SmallLinearJob* temb_jobs_dev = nullptr; int temb_max_n = 0;
    // fixed I/O buffers
    T4 unet_in; float* unet_out = nullptr; __half* ctx16 = nullptr; float* temb = nullptr; long long* t_dev = nullptr;
    T4 vae_in; float* vae_moments = nullptr; float* vae_gmoments = nullptr; __half* vae_gin = nullptr;
    T4 dec_in; float* dec_out = nullptr; std::vector<Op> dec_ops;          // VAE decoder (denoise side branch, nerf/sd.py:201-210)
    int ctx_pad = 128;

    struct GN { double* stats; const float* gamma; const float* beta; float eps; int silu; T4 x; int G; };
    GN groupnorm(const T4& x, const std::string& pname, float eps, int silu, const T4& y) {
        GN g; g.x = x; g.G = ucfg.groups; g.eps = eps; g.silu = silu;
        g.gamma = pf(pname + ".weight", {x.c}); g.beta = pf(pname + ".bias", {x.c});
        g.stats = pool_stats((size_t)x.n * g.G * 2);
        if (dry) return g;
        const int HW = x.h * x.w, C = x.c, G = g.G, N = x.n;
        sdk::GnGrid q;
        if (!sdk::gn_grid(N, HW, C, G, num_sms, &q)) { err = MI3D_ERR_ARG; return g; }
        const __half* xp = x.p; __half* yp = y.p; const GN gg = g;
        push([=](cudaStream_t st) { return sdk::gn_forward(q, xp, yp, gg.stats, gg.gamma, gg.beta, N, HW, C, G, gg.eps, gg.silu, st); });
        return g;
    }
    // dx = GN(+SiLU) backward of dy (+ add)
    void groupnorm_bwd(const GN& g, const __half* dy, const __half* add, __half* dx) {
        double* bstats = pool_stats((size_t)g.x.n * g.G * 2);
        if (dry) return;
        const int HW = g.x.h * g.x.w, C = g.x.c, G = g.G, N = g.x.n;
        sdk::GnGrid q;
        if (!sdk::gn_grid(N, HW, C, G, num_sms, &q)) { err = MI3D_ERR_ARG; return; }
        const GN gg = g;
        push([=](cudaStream_t st) { return sdk::gn_backward(q, gg.x.p, dy, gg.stats, bstats, gg.gamma, gg.beta, add, dx, N, HW, C, G, gg.eps, gg.silu, st); });
    }
    void linear_small(const float* x, const __half* w, const float* bias, float* y, int B, int N, int K, int silu_in, int silu_out) {
        push([=](cudaStream_t st) { return sdk::linear_small(x, w, bias, y, B, N, K, silu_in, silu_out, st); });
    }

    // ------------------------------------------------------------------------------------------------------
    // diffusers blocks (diffusers naming)
    // ------------------------------------------------------------------------------------------------------
    // Each param() / pf() is a statement of its own, never another call's argument: the seeded stand-in weights are drawn in registry order.
    // what the VAE encoder's input-gradient pass (build_vae_bwd) reads of a forward block
    struct ResTape { std::string pre; T4 x; int cout; GN g1, g2; };
    struct AttnTape { std::string pre; T4 x; GN g; __half *q, *k, *v, *P; };

    // ResnetBlock2D: the U-Net's (has_temb, eps 1e-5), the VAE encoder's (tape: weights with a dgrad copy, *tape filled) and the
    // VAE decoder's (eps 1e-6)
    T4 resnet(const std::string& pre, const T4& x, int cout, bool has_temb, float eps, ResTape* tape = nullptr) {
        const int cin = x.c;
        T4 a1 = act(x.n, x.h, x.w, cin);
        GN g1 = groupnorm(x, pre + ".norm1", eps, 1, a1);
        const float* rb = nullptr;
        if (has_temb) {
            const int tdim = ucfg.block_out[0] * 4;
            const __half* wt = (const __half*)param(pre + ".time_emb_proj.weight", {cout, tdim}, PK_LINEAR).dst;
            const float* bt = pf(pre + ".time_emb_proj.bias", {cout});
            float* tp = alloc32((size_t)x.n * cout);
            temb_jobs.push_back({wt, bt, tp, cout});          // evaluated by the grouped launch at the head of the U-Net
            temb_max_n = std::max(temb_max_n, cout);
            rb = tp;
        }
        const PKind k3 = tape ? PK_CONV3_BOTH : PK_CONV3, k1 = tape ? PK_CONV1_BOTH : PK_CONV1;
        const __half* w1 = (const __half*)param(pre + ".conv1.weight", {cout, cin, 3, 3}, k3).dst;
        T4 h1 = act(x.n, x.h, x.w, cout);
        const float* b1 = pf(pre + ".conv1.bias", {cout});
        conv3(a1, w1, cout, h1, b1, rb);
        T4 a2 = act(x.n, x.h, x.w, cout);
        GN g2 = groupnorm(h1, pre + ".norm2", eps, 1, a2);
        const __half* sc = x.p;
        if (cin != cout) {
            const __half* ws = (const __half*)param(pre + ".conv_shortcut.weight", {cout, cin, 1, 1}, k1).dst;
            T4 s = act(x.n, x.h, x.w, cout);
            const float* bs = pf(pre + ".conv_shortcut.bias", {cout});
            linear(x.p, x.rows(), cin, ws, cout, s.p, bs);
            sc = s.p;
        }
        const __half* w2 = (const __half*)param(pre + ".conv2.weight", {cout, cout, 3, 3}, k3).dst;
        T4 out = act(x.n, x.h, x.w, cout);
        const float* b2 = pf(pre + ".conv2.bias", {cout});
        conv3(a2, w2, cout, out, b2, nullptr, sc);
        if (tape) *tape = ResTape{pre, x, cout, g1, g2};
        return out;
    }

    T4 transformer(const std::string& pre, const T4& x, int heads) {
        const int C = x.c, B = x.n, T = x.h * x.w; const long long M = x.rows();
        const int d = C / heads, cross = ucfg.cross_dim;
        T4 n = act(x.n, x.h, x.w, C);
        groupnorm(x, pre + ".norm", 1e-6f, 0, n);
        __half* h = alloc16(M * C);
        // proj_in / proj_out: Linear [C, C] (SD-2.x) or 1x1 Conv2d [C, C, 1, 1] (SD-1.x), the same [C][C] fp16 matrix either way
        const std::vector<int> pshape = ucfg.proj_conv ? std::vector<int>{C, C, 1, 1} : std::vector<int>{C, C};
        const PKind pkind = ucfg.proj_conv ? PK_CONV1 : PK_LINEAR;
        const float* b_in = pf(pre + ".proj_in.bias", {C});
        const __half* w_in = (const __half*)param(pre + ".proj_in.weight", pshape, pkind).dst;
        linear(n.p, M, C, w_in, C, h, b_in);
        const std::string tb = pre + ".transformer_blocks.0";
        // ---- self attention ----
        __half* ln = alloc16(M * C);
        layernorm(h, M, C, tb + ".norm1", ln);
        // to_q / to_k / to_v are registered back to back, and each starts on an alloc() boundary: for C % 32 == 0 they are one [3C][C]
        // matrix, and one GEMM produces q | k | v side by side.  Any other layout fails the build.
        const __half* wq = (const __half*)param(tb + ".attn1.to_q.weight", {C, C}, PK_LINEAR).dst;
        const __half* wk = (const __half*)param(tb + ".attn1.to_k.weight", {C, C}, PK_LINEAR).dst;
        const __half* wv = (const __half*)param(tb + ".attn1.to_v.weight", {C, C}, PK_LINEAR).dst;
        if (wk != wq + (size_t)C * C || wv != wk + (size_t)C * C) err = MI3D_ERR_ARG;
        __half* ao = alloc16(M * C);
        __half* qkv = alloc16(M * 3 * C);
        linear(ln, M, C, wq, 3 * C, qkv);
        attention_core(qkv, 3 * C, qkv + C, 3 * C, qkv + 2 * C, 3 * C, B, T, T, T, heads, d, ao, C);
        __half* h2 = alloc16(M * C);
        const float* bo1 = pf(tb + ".attn1.to_out.0.bias", {C});
        const __half* wo1 = (const __half*)param(tb + ".attn1.to_out.0.weight", {C, C}, PK_LINEAR).dst;
        linear(ao, M, C, wo1, C, h2, bo1, h);
        // ---- cross attention (keys/values from the text context, padded to ctx_pad rows per batch) ----
        __half* ln2 = alloc16(M * C);
        layernorm(h2, M, C, tb + ".norm2", ln2);
        const long long Mc = (long long)B * ctx_pad;
        __half* q2 = alloc16(M * C);
        const __half* wq2 = (const __half*)param(tb + ".attn2.to_q.weight", {C, C}, PK_LINEAR).dst;
        linear(ln2, M, C, wq2, C, q2);
        // to_k / to_v likewise one [2C][cross] matrix (C * cross % 512 == 0): one GEMM produces k | v
        const __half* wk2 = (const __half*)param(tb + ".attn2.to_k.weight", {C, cross}, PK_LINEAR).dst;
        const __half* wv2 = (const __half*)param(tb + ".attn2.to_v.weight", {C, cross}, PK_LINEAR).dst;
        if (wv2 != wk2 + (size_t)C * cross) err = MI3D_ERR_ARG;
        __half* ao2 = alloc16(M * C);
        __half* kv = alloc16(Mc * 2 * C);
        linear(ctx16, Mc, cross, wk2, 2 * C, kv);
        attention_core(q2, C, kv, 2 * C, kv + C, 2 * C, B, T, ctx_pad, ucfg.ctx_len, heads, d, ao2, C);
        __half* h3 = alloc16(M * C);
        const float* bo2 = pf(tb + ".attn2.to_out.0.bias", {C});
        const __half* wo2 = (const __half*)param(tb + ".attn2.to_out.0.weight", {C, C}, PK_LINEAR).dst;
        linear(ao2, M, C, wo2, C, h3, bo2, h2);
        // ---- GEGLU feed-forward ----
        __half* ln3 = alloc16(M * C);
        layernorm(h3, M, C, tb + ".norm3", ln3);
        Param& wg = param(tb + ".ff.net.0.proj.weight", {8 * C, C}, PK_GEGLU_W);
        Param& bg = param(tb + ".ff.net.0.proj.bias", {8 * C}, PK_GEGLU_B);
        wg.partner = bg.name; bg.partner = wg.name;
        __half* f1 = alloc16(M * 4 * C);
        linear(ln3, M, C, (const __half*)wg.dst, 8 * C, f1, (const float*)bg.dst, nullptr, tc::EPI_GEGLU);
        __half* h4 = alloc16(M * C);
        const float* bf = pf(tb + ".ff.net.2.bias", {C});
        const __half* wf = (const __half*)param(tb + ".ff.net.2.weight", {C, 4 * C}, PK_LINEAR).dst;
        linear(f1, M, 4 * C, wf, C, h4, bf, h3);
        T4 out = act(x.n, x.h, x.w, C);
        const float* b_out = pf(pre + ".proj_out.bias", {C});
        const __half* w_out = (const __half*)param(pre + ".proj_out.weight", pshape, pkind).dst;
        linear(h4, M, C, w_out, C, out.p, b_out, x.p);
        return out;
    }

    T4 downsample(const std::string& pre, const T4& x, int pad_lo, bool both) {
        const int C = x.c;
        const __half* w = (const __half*)param(pre + ".conv.weight", {C, C, 3, 3}, both ? PK_CONV3_S2_BOTH : PK_CONV3).dst;
        T4 y = act(x.n, x.h / 2, x.w / 2, C);
        const float* b = pf(pre + ".conv.bias", {C});
        conv3_s2(x, w, y, b, pad_lo);
        return y;
    }

    // Upsample2D: nearest 2x, then a 3x3 conv
    T4 upsample(const std::string& pre, const T4& x) {
        T4 up = act(x.n, x.h * 2, x.w * 2, x.c);
        const T4 xx = x;
        push([=](cudaStream_t st) {
            sdk::k_upsample2x<<<blocks_for(up.numel() / 8), 256, 0, st>>>(xx.p, up.p, xx.n, xx.h, xx.w, xx.c);
            return (int)cudaGetLastError();
        });
        T4 y = act(up.n, up.h, up.w, up.c);
        const float* b = pf(pre + ".conv.bias", {x.c});
        const __half* w = (const __half*)param(pre + ".conv.weight", {x.c, x.c, 3, 3}, PK_CONV3).dst;
        conv3(up, w, x.c, y, b);
        return y;
    }

    T4 concat(const T4& a, const T4& b) {
        T4 o = act(a.n, a.h, a.w, a.c + b.c);
        const T4 aa = a, bb = b;
        push([=](cudaStream_t st) {
            sdk::k_concat<<<blocks_for(o.numel() / 8), 256, 0, st>>>(aa.p, bb.p, o.p, (size_t)aa.rows(), aa.c, bb.c);
            return (int)cudaGetLastError();
        });
        return o;
    }

    void build_unet() {
        begin_list(&unet_ops);
        const mi3d_unet_cfg& c = ucfg;
        const int B = c.batch, HW = c.latent_hw, nlev = c.n_levels, L = c.layers_per_block;
        const int c0 = c.block_out[0], tdim = c0 * 4;
        unet_in = act(B, HW, HW, c.in_ch);
        t_dev = (long long*)alloc(sizeof(long long));
        ctx16 = alloc16((size_t)B * ctx_pad * c.cross_dim);
        // time embedding
        float* tproj = alloc32((size_t)B * c0);
        float* t1 = alloc32((size_t)B * tdim);
        temb = alloc32((size_t)B * tdim);
        {
            long long* tptr = t_dev;
            push([=](cudaStream_t st) {
                sdk::k_time_proj<<<(B * c0 / 2 + 127) / 128, 128, 0, st>>>(tptr, tproj, B, c0);
                return (int)cudaGetLastError();
            });
            const float* b1 = pf("time_embedding.linear_1.bias", {tdim});
            const __half* w1 = (const __half*)param("time_embedding.linear_1.weight", {tdim, c0}, PK_LINEAR).dst;
            linear_small(tproj, w1, b1, t1, B, tdim, c0, 0, 1);
            const float* b2 = pf("time_embedding.linear_2.bias", {tdim});
            const __half* w2 = (const __half*)param("time_embedding.linear_2.weight", {tdim, tdim}, PK_LINEAR).dst;
            linear_small(t1, w2, b2, temb, B, tdim, tdim, 0, 0);
            temb_jobs.clear(); temb_max_n = 0;
            temb_jobs_dev = (sdk::SmallLinearJob*)alloc(64 * sizeof(sdk::SmallLinearJob));
            const float* te = temb;
            push([this, te, B, tdim](cudaStream_t st) {
                if (temb_jobs.empty()) return 0;
                return sdk::linear_small_grouped(te, temb_jobs_dev, (int)temb_jobs.size(), temb_max_n, B, tdim, st);
            });
        }
        // conv_in (Cin = 4): direct
        T4 h = act(B, HW, HW, c0);
        {
            const float* w = (const float*)param("conv_in.weight", {c0, c.in_ch, 3, 3}, PK_CONV_F32_OHWI).dst;
            const float* b = pf("conv_in.bias", {c0});
            if (c.in_ch != 4) err = MI3D_ERR_ARG;
            conv_small_cin(unet_in, w, b, h);
        }
        tap("unet.conv_in", h.p, h.numel() * 2);
        std::vector<T4> skips; skips.push_back(h);
        for (int i = 0; i < nlev; i++) {
            const bool has_attn = i < nlev - 1;
            for (int j = 0; j < L; j++) {
                const std::string rp = "down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
                h = resnet(rp, h, c.block_out[i], true, 1e-5f);
                if (has_attn) h = transformer("down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), h, c.heads[i]);
                skips.push_back(h);
            }
            if (i < nlev - 1) {
                h = downsample("down_blocks." + std::to_string(i) + ".downsamplers.0", h, 1, false);
                skips.push_back(h);
            }
            tap("unet.down" + std::to_string(i), h.p, h.numel() * 2);
        }
        h = resnet("mid_block.resnets.0", h, h.c, true, 1e-5f);
        h = transformer("mid_block.attentions.0", h, c.heads[nlev - 1]);
        h = resnet("mid_block.resnets.1", h, h.c, true, 1e-5f);
        tap("unet.mid", h.p, h.numel() * 2);
        for (int i = 0; i < nlev; i++) {
            const int lev = nlev - 1 - i;
            const bool has_attn = i > 0;
            for (int j = 0; j < L + 1; j++) {
                T4 s = skips.back(); skips.pop_back();
                T4 cat = concat(h, s);
                h = resnet("up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), cat, c.block_out[lev], true, 1e-5f);
                if (has_attn) h = transformer("up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), h, c.heads[lev]);
            }
            if (i < nlev - 1) h = upsample("up_blocks." + std::to_string(i) + ".upsamplers.0", h);
            tap("unet.up" + std::to_string(i), h.p, h.numel() * 2);
        }
        T4 a = act(h.n, h.h, h.w, h.c);
        groupnorm(h, "conv_norm_out", 1e-5f, 1, a);
        unet_out = alloc32((size_t)B * HW * HW * c.out_ch);
        {
            const __half* w = (const __half*)param("conv_out.weight", {c.out_ch, c0, 3, 3}, PK_CONV_SMALL_COUT).dst;
            const float* b = pf("conv_out.bias", {c.out_ch});
            if (c.out_ch != 4) err = MI3D_ERR_ARG;
            conv_small_cout(a, w, b, unet_out, 4);
        }
        if (temb_jobs.size() > 64) err = MI3D_ERR_ARG;
        if (!dry && !err && !temb_jobs.empty())
            if (cudaMemcpy(temb_jobs_dev, temb_jobs.data(), temb_jobs.size() * sizeof(sdk::SmallLinearJob), cudaMemcpyHostToDevice) != cudaSuccess) err = MI3D_ERR_ARG;
        cur = nullptr;
    }

    // ------------------------------------------------------------------------------------------------------
    // VAE encoder forward + input-gradient backward (AutoencoderKL.encode, nerf/sd.py:212-220)
    // ------------------------------------------------------------------------------------------------------
    struct DownTape { T4 x, y; std::string pre; };

    std::vector<ResTape> vres; std::vector<DownTape> vdown; AttnTape vattn; GN vgn_out; T4 v_a_out, v_h_last, v_conv_in_out;
    std::vector<int> vorder;   // 0 = res, 1 = down, 2 = attn ; forward order for the reverse walk

    // the VAE's Attention: one head over the pixels of each image (batched over x.n images; P is [n][pix][pix]) (tape: weights with a
    // transposed copy, *tape filled)
    T4 vae_attention(const std::string& pre, const T4& x, AttnTape* tape) {
        const PKind kind = tape ? PK_LINEAR_BOTH : PK_LINEAR;
        const long long M = x.rows(); const int C = x.c, nb = x.n, pix = x.h * x.w;
        T4 n = act(x.n, x.h, x.w, C);
        GN g = groupnorm(x, pre + ".group_norm", 1e-6f, 0, n);
        __half *q = alloc16(M * C), *k = alloc16(M * C), *v = alloc16(M * C), *vT = alloc16(M * C);
        const float* bq = pf(pre + ".to_q.bias", {C});
        const __half* wq = (const __half*)param(pre + ".to_q.weight", {C, C}, kind).dst;
        linear(n.p, M, C, wq, C, q, bq);
        const float* bk = pf(pre + ".to_k.bias", {C});
        const __half* wk = (const __half*)param(pre + ".to_k.weight", {C, C}, kind).dst;
        linear(n.p, M, C, wk, C, k, bk);
        const float* bv = pf(pre + ".to_v.bias", {C});
        const __half* wv = (const __half*)param(pre + ".to_v.weight", {C, C}, kind).dst;
        linear(n.p, M, C, wv, C, v, bv);
        transpose(v, vT, nb, pix, C);
        __half* P = alloc16((size_t)M * pix);
        per_image_gemm(q, C, pix, C, k, C, pix, P, pix, nb);
        softmax(P, (size_t)M, pix, pix, 1.0f / sqrtf((float)C));
        __half* ao = alloc16(M * C);
        per_image_gemm(P, pix, pix, pix, vT, pix, C, ao, C, nb);
        T4 out = act(x.n, x.h, x.w, C);
        const float* bo = pf(pre + ".to_out.0.bias", {C});
        const __half* wo = (const __half*)param(pre + ".to_out.0.weight", {C, C}, kind).dst;
        linear(ao, M, C, wo, C, out.p, bo, x.p);
        if (tape) *tape = AttnTape{pre, x, g, q, k, v, P};
        return out;
    }
    // out_i[rows][N] = A_i[rows][K] B_i[N][K]^T for the nb images i: A_i = a + i * rows * K, B_i = b + i * N * K, out_i = o + i * rows * N
    // (every operand packed per image).  One image is the plain GEMM.
    void per_image_gemm(const __half* a, long long lda, long long rows, int K, const __half* b, long long ldb, int N, __half* o, long long ldo, int nb) {
        Mat am{a, lda, rows, K}; Mat bm{b, ldb, N, K}; am.z1 = nb; bm.z1 = nb;
        Out oo; oo.p16 = o; oo.ldc = ldo; oo.z1 = nb; oo.s_lo = rows * ldo;
        Epi e; gemm(am, bm, N, oo, e, nb, nb > 1);
    }

    // the VAE's mid block: resnet, attention, resnet; taped (the encoder's) in vres / vattn / vorder for build_vae_bwd
    T4 vae_mid(const std::string& pre, T4 h, bool taped) {
        ResTape t0, t1;
        h = resnet(pre + ".resnets.0", h, h.c, false, 1e-6f, taped ? &t0 : nullptr);
        h = vae_attention(pre + ".attentions.0", h, taped ? &vattn : nullptr);
        h = resnet(pre + ".resnets.1", h, h.c, false, 1e-6f, taped ? &t1 : nullptr);
        if (taped) { vres.push_back(t0); vres.push_back(t1); vorder.insert(vorder.end(), {0, 2, 0}); }
        return h;
    }

    void build_vae() {
        begin_list(&enc_ops);
        const mi3d_vae_cfg& c = vcfg;
        const int S = c.image_hw, nlev = c.n_levels, L = c.layers_per_block, nb = vae_images();
        vae_in = act(nb, S, S, 4);         // 3 channels padded to 4 (the 4th is zero)
        T4 h = act(nb, S, S, c.block_out[0]);
        {
            const float* w = (const float*)param("encoder.conv_in.weight", {c.block_out[0], c.in_ch, 3, 3}, PK_CONV_F32_OHWI).dst;
            const float* b = pf("encoder.conv_in.bias", {c.block_out[0]});
            conv_small_cin(vae_in, w, b, h);
        }
        v_conv_in_out = h;
        for (int i = 0; i < nlev; i++) {
            for (int j = 0; j < L; j++) {
                ResTape t;
                h = resnet("encoder.down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), h, c.block_out[i], false, 1e-6f, &t);
                vres.push_back(t); vorder.push_back(0);
            }
            if (i < nlev - 1) {
                DownTape d; d.x = h; d.pre = "encoder.down_blocks." + std::to_string(i) + ".downsamplers.0";
                h = downsample(d.pre, h, 0, true);
                d.y = h; vdown.push_back(d); vorder.push_back(1);
            }
        }
        h = vae_mid("encoder.mid_block", h, true);
        const int ch = h.c;
        v_h_last = h;
        v_a_out = act(h.n, h.h, h.w, ch);
        vgn_out = groupnorm(h, "encoder.conv_norm_out", 1e-6f, 1, v_a_out);
        // conv_out (ch -> 2*latent) direct + quant_conv (1x1, 2l -> 2l) folded in a tiny kernel at the API level
        const int l2 = 2 * c.latent_ch;
        float* co = alloc32((size_t)h.rows() * l2);
        {
            const __half* w = (const __half*)param("encoder.conv_out.weight", {l2, ch, 3, 3}, PK_CONV_SMALL_COUT_BOTH).dst;
            const float* b = pf("encoder.conv_out.bias", {l2});
            if (l2 != 8) err = MI3D_ERR_ARG;
            conv_small_cout(v_a_out, w, b, co, 8);
        }
        vae_moments = co;
        pf("quant_conv.weight", {l2, l2, 1, 1}); pf("quant_conv.bias", {l2});
        cur = nullptr;
    }

    // ------------------------------------------------------------------------------------------------------
    // VAE decoder (diffusers AutoencoderKL.decode: post_quant_conv folded into the API kernel, then Decoder): forward only.
    // ------------------------------------------------------------------------------------------------------
    void build_vae_dec() {
        begin_list(&dec_ops);
        const mi3d_vae_cfg& c = vcfg;
        const int nlev = c.n_levels, L = c.layers_per_block, hw = c.image_hw >> (nlev - 1);
        int ch = c.block_out[nlev - 1];
        dec_in = act(1, hw, hw, 4);                         // post_quant_conv(latents / 0.18215), NHWC fp16, written by the API kernel
        pf("post_quant_conv.weight", {c.latent_ch, c.latent_ch, 1, 1}); pf("post_quant_conv.bias", {c.latent_ch});
        T4 h = act(1, hw, hw, ch);
        {
            const float* w = (const float*)param("decoder.conv_in.weight", {ch, c.latent_ch, 3, 3}, PK_CONV_F32_OHWI).dst;
            const float* b = pf("decoder.conv_in.bias", {ch});
            if (c.latent_ch != 4) err = MI3D_ERR_ARG;
            conv_small_cin(dec_in, w, b, h);
        }
        h = vae_mid("decoder.mid_block", h, false);
        for (int i = 0; i < nlev; i++) {
            const int co = c.block_out[nlev - 1 - i];
            for (int j = 0; j < L + 1; j++) h = resnet("decoder.up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), h, co, false, 1e-6f);
            ch = co;
            if (i < nlev - 1) h = upsample("decoder.up_blocks." + std::to_string(i) + ".upsamplers.0", h);
        }
        T4 a = act(h.n, h.h, h.w, h.c);
        groupnorm(h, "decoder.conv_norm_out", 1e-6f, 1, a);
        dec_out = alloc32((size_t)a.rows() * 4);
        {
            // conv_out ch -> 3: the 4-output direct kernel; its 4th weight row / bias entry is the (zeroed) pad allocated right behind
            const __half* w = (const __half*)param("decoder.conv_out.weight", {c.in_ch, ch, 3, 3}, PK_CONV_SMALL_COUT).dst;
            alloc16((size_t)9 * ch);
            const float* b = pf("decoder.conv_out.bias", {c.in_ch});
            alloc32(4);
            if (c.in_ch != 3) err = MI3D_ERR_ARG;
            conv_small_cout(a, w, b, dec_out, 4);
        }
        cur = nullptr;
    }

    void build_vae_bwd() {
        begin_list(&enc_bwd_ops);
        const mi3d_vae_cfg& c = vcfg;
        const int l2 = 2 * c.latent_ch;
        const T4 hl = v_h_last; const int ch = hl.c;
        vae_gmoments = alloc32((size_t)hl.rows() * l2);        // d/d(conv_out output) fp32 [pix][8], filled by the API kernel
        // conv_out^T : small-Cout transposed = "small Cin" conv with Cin = 8 -> output ch channels (fp16 in)
        T4 g8 = act(hl.n, hl.h, hl.w, 8);
        T4 da = act(hl.n, hl.h, hl.w, ch);
        {
            const float* wf = (const float*)param("encoder.conv_out.weight#dgrad_f32", {ch, 8, 3, 3}, PK_CONV_F32_OHWI).dst;
            f32_to_f16(vae_gmoments, g8.p, g8.numel());          // fp32 -> fp16 staging of the 8-channel gradient
            conv_small_cin(g8, wf, nullptr, da);
        }
        T4 dh = act(hl.n, hl.h, hl.w, ch);
        groupnorm_bwd(vgn_out, da.p, nullptr, dh.p);
        // reverse walk
        int ri = (int)vres.size() - 1, di = (int)vdown.size() - 1;
        for (int oi = (int)vorder.size() - 1; oi >= 0; oi--) {
            const int kind = vorder[oi];
            if (kind == 0) {
                const ResTape& t = vres[ri--]; const int cin = t.x.c, cout = t.cout;
                // out = sc(x) + conv2(a2) ; a2 = silu(gn2(h1)) ; h1 = conv1(a1) ; a1 = silu(gn1(x))
                T4 da2 = act(t.x.n, t.x.h, t.x.w, cout);
                conv3_dgrad(dh, t.pre + ".conv2.weight", cout, da2);
                T4 dh1 = act(t.x.n, t.x.h, t.x.w, cout);
                groupnorm_bwd(t.g2, da2.p, nullptr, dh1.p);
                T4 da1 = act(t.x.n, t.x.h, t.x.w, cin);
                conv3_dgrad(dh1, t.pre + ".conv1.weight", cin, da1);
                // shortcut branch gradient
                const __half* dsc = dh.p;
                if (cin != cout) {
                    Param& ws = params[pindex[t.pre + ".conv_shortcut.weight"]];
                    T4 d = act(t.x.n, t.x.h, t.x.w, cin);
                    linear(dh.p, t.x.rows(), cout, (const __half*)ws.dst2, cin, d.p);     // dst2 = W^T [cin][cout]
                    dsc = d.p;
                }
                T4 dx = act(t.x.n, t.x.h, t.x.w, cin);
                groupnorm_bwd(t.g1, da1.p, dsc, dx.p);
                dh = dx;
            } else if (kind == 1) {
                const DownTape& d = vdown[di--];
                const int C = d.x.c; const long long Mo = d.y.rows();
                Param& w = params[pindex[d.pre + ".conv.weight"]];
                // dcol[Mo, 9C] = dy[Mo, C] . Wt   with Wt = [9C][C]  (dst2 of a PK_CONV3_S2_BOTH weight = plain transpose, see Builder::load_param)
                __half* dcol = alloc16((size_t)Mo * 9 * C);
                linear(dh.p, Mo, C, (const __half*)w.dst2, 9 * C, dcol);
                T4 dx = act(d.x.n, d.x.h, d.x.w, C);
                const T4 xx = d.x, yy = d.y;
                push([=](cudaStream_t st) { return col2im_s2(dcol, dx.p, xx.n, xx.h, xx.w, C, yy.h, yy.w, 0, st); });
                dh = dx;
            } else {
                const AttnTape& a = vattn; const int C = a.x.c, nb = a.x.n, pix = a.x.h * a.x.w; const long long M = a.x.rows();
                auto W2 = [&](const std::string& n) { return (const __half*)params[pindex[a.pre + n]].dst2; };   // transposed copies [in][out]
                // out = x + ao Wo^T + b
                __half* dao = alloc16(M * C);
                linear(dh.p, M, C, W2(".to_out.0.weight"), C, dao);
                // per image: dV = P^T dao ; dP = dao V^T
                __half* PT = alloc16((size_t)M * pix); transpose(a.P, PT, nb, pix, pix);
                __half* daoT = alloc16(M * C); transpose(dao, daoT, nb, pix, C);
                __half* dV = alloc16(M * C);
                per_image_gemm(PT, pix, pix, pix, daoT, pix, C, dV, C, nb);
                __half* dP = alloc16((size_t)M * pix);
                per_image_gemm(dao, C, pix, C, a.v, C, pix, dP, pix, nb);
                const float scale = 1.0f / sqrtf((float)C);
                softmax_bwd(a.P, dP, (size_t)M, pix, scale);
                // dQ = dS K ; dK = dS^T Q
                __half* kT = alloc16(M * C); transpose(a.k, kT, nb, pix, C);
                __half* qT = alloc16(M * C); transpose(a.q, qT, nb, pix, C);
                __half* dST = alloc16((size_t)M * pix); transpose(dP, dST, nb, pix, pix);
                __half* dQ = alloc16(M * C); __half* dK = alloc16(M * C);
                per_image_gemm(dP, pix, pix, pix, kT, pix, C, dQ, C, nb);
                per_image_gemm(dST, pix, pix, pix, qT, pix, C, dK, C, nb);
                // dn = dQ Wq + dK Wk + dV Wv
                __half* dn1 = alloc16(M * C); __half* dn2 = alloc16(M * C); __half* dn3 = alloc16(M * C);
                linear(dQ, M, C, W2(".to_q.weight"), C, dn1);
                linear(dK, M, C, W2(".to_k.weight"), C, dn2, nullptr, dn1);
                linear(dV, M, C, W2(".to_v.weight"), C, dn3, nullptr, dn2);
                T4 dx = act(a.x.n, a.x.h, a.x.w, C);
                groupnorm_bwd(a.g, dn3, dh.p, dx.p);
                dh = dx;
            }
        }
        // conv_in^T: d/d(input image, 4 padded channels) -- small-Cout direct conv with flipped weights, fp32 out
        vae_gin = nullptr;
        float* gimg = alloc32((size_t)vae_in.rows() * 4);
        named["vae.grad_in"] = {gimg, (size_t)vae_in.rows() * 4 * sizeof(float)};
        {
            const __half* w = (const __half*)param("encoder.conv_in.weight#dgrad", {4, c.block_out[0], 3, 3}, PK_CONV_SMALL_COUT).dst;
            conv_small_cout(dh, w, nullptr, gimg, 4);
        }
        vae_grad_img = gimg;
        cur = nullptr;
    }
    float* vae_grad_img = nullptr;

    // ------------------------------------------------------------------------------------------------------
    // DDIM sampling step (produce_latents, nerf/sd.py:183-197): [x, x] -> U-Net -> CFG + DDIM update in place.  The schedule, the
    // latents and the step index live in engine buffers, so the list is static and replays as one graph per step.
    // ------------------------------------------------------------------------------------------------------
    std::vector<Op> sample_ops;
    mi3d_sd_schedule* sample_sched = nullptr; float* sample_lat = nullptr; SampleState* sample_state = nullptr;
    void build_sample() {
        // allocated after every other list so that the existing buffers keep their offsets
        const int pix = ucfg.latent_hw * ucfg.latent_hw;
        sample_sched = (mi3d_sd_schedule*)alloc(kMaxSampleSteps * sizeof(mi3d_sd_schedule));
        sample_lat = alloc32((size_t)4 * pix);
        sample_state = (SampleState*)alloc(sizeof(SampleState));
        cur = &sample_ops;
        const mi3d_sd_schedule* tab = sample_sched; float* lat = sample_lat; SampleState* s = sample_state;
        __half* xin = unet_in.p; long long* tslot = t_dev; const float* uo = unet_out;
        push([=](cudaStream_t st) { k_sample_in<<<1, 1024, 0, st>>>(tab, s, lat, xin, tslot, pix); return (int)cudaGetLastError(); });
        for (const Op& op : unet_ops) push(op);
        push([=](cudaStream_t st) { k_sample_step<<<1, 1024, 0, st>>>(uo, tab, s, lat, pix); return (int)cudaGetLastError(); });
        cur = nullptr;
    }

    // images per encode (mi3d_vae_cfg.batch; 0 means one)
    int vae_images() const { return std::max(1, vcfg.batch); }

    // a measuring pass (host only) records each list's GroupNorm-statistics need, then the plan is built for real (or sized)
    int build(bool dry_run) {
        if (vcfg.batch < 0) return MI3D_ERR_ARG;
        measuring = true; pool_need.clear();
        const int r = build_pass(true);
        measuring = false;
        return r ? r : build_pass(dry_run);
    }
    int build_pass(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); unet_ops.clear(); enc_ops.clear(); enc_bwd_ops.clear(); dec_ops.clear();
        sample_ops.clear(); vres.clear(); vdown.clear(); vorder.clear(); named.clear();
        splitk_elems = (size_t)2048 * 2560; splitk_ws = alloc32(splitk_elems);       // covers M <= 2048 rows x N <= 2560
        if (ucfg.n_levels > 0) build_unet();
        if (vcfg.n_levels > 0) { build_vae(); build_vae_bwd(); if (vcfg.decoder) build_vae_dec(); }
        if (ucfg.n_levels > 0 && ucfg.batch == 2 && ucfg.in_ch == 4 && ucfg.out_ch == 4) build_sample();
        return err;
    }

    int load_param(const Param& P, const float* src, const float* partner, cudaStream_t st) override {
        const int nb = blocks_for(P.numel);
        using namespace sdk;
        switch (P.kind) {
            case PK_GEGLU_W: {
                if (!partner) return MI3D_ERR_ARG;
                const Param& Bp = params[pindex[P.partner]];
                k_geglu_w<<<nb, 256, 0, st>>>(src, partner, (__half*)P.dst, (float*)Bp.dst, P.shape[0] / 2, P.shape[1]);
                break;
            }
            case PK_GEGLU_B: break;     // written together with the weight
            case PK_CONV_F32_OHWI: {
                // fp32 direct-conv weights.  Base form: OIHW [O][I][3][3] -> [O][ky][kx][Ipad] with Ipad = 4 (conv_in) ;
                // "#dgrad_f32" form (conv_out transposed): src is conv_out OIHW [8][ch][3][3] -> [ch][2-ky][2-kx][8]
                std::vector<float> tmp;   // host staging keeps this one-off path simple
                const bool dg = P.name.find("#dgrad_f32") != std::string::npos;
                const int O = dg ? P.shape[1] : P.shape[0], I = dg ? P.shape[0] : P.shape[1];
                std::vector<float> hsrc((size_t)O * I * 9);
                MI3D_CHECK(cudaMemcpyAsync(hsrc.data(), src, hsrc.size() * 4, cudaMemcpyDeviceToHost, st));
                MI3D_CHECK(cudaStreamSynchronize(st));
                if (!dg) {
                    const int Ip = 4;
                    tmp.assign((size_t)O * 9 * Ip, 0.f);
                    for (int o = 0; o < O; o++) for (int c = 0; c < I; c++) for (int t = 0; t < 9; t++) tmp[((size_t)o * 9 + t) * Ip + c] = hsrc[((size_t)o * I + c) * 9 + t];
                } else {
                    // hsrc = conv_out [O=8][I=ch][3][3]; want w'[ci=ch][ky'][kx'][co=8] = hsrc[co][ci][2-ky'][2-kx']
                    tmp.assign((size_t)I * 9 * O, 0.f);
                    for (int o = 0; o < O; o++) for (int c = 0; c < I; c++) for (int t = 0; t < 9; t++) tmp[((size_t)c * 9 + (8 - t)) * O + o] = hsrc[((size_t)o * I + c) * 9 + t];
                }
                MI3D_CHECK(cudaMemcpyAsync(P.dst, tmp.data(), std::min(tmp.size(), dg ? P.numel : tmp.size()) * 4, cudaMemcpyHostToDevice, st));
                MI3D_CHECK(cudaStreamSynchronize(st));
                break;
            }
            case PK_CONV_SMALL_COUT: case PK_CONV_SMALL_COUT_BOTH: {
                const bool dg = P.name.find("#dgrad") != std::string::npos;
                if (!dg) return Builder::load_param(P, src, partner, st);
                else {
                    // conv_in transposed: src conv_in OIHW [c0][3][3][3]; want [4 (padded cin)][2-ky][2-kx][c0] fp16
                    const int c0 = P.shape[1];
                    std::vector<float> hsrc((size_t)c0 * 3 * 9);
                    MI3D_CHECK(cudaMemcpyAsync(hsrc.data(), src, hsrc.size() * 4, cudaMemcpyDeviceToHost, st));
                    MI3D_CHECK(cudaStreamSynchronize(st));
                    std::vector<__half> tmp((size_t)4 * 9 * c0, __float2half(0.f));
                    for (int o = 0; o < c0; o++) for (int c = 0; c < 3; c++) for (int t = 0; t < 9; t++) tmp[((size_t)c * 9 + (8 - t)) * c0 + o] = __float2half(hsrc[((size_t)o * 3 + c) * 9 + t]);
                    MI3D_CHECK(cudaMemcpyAsync(P.dst, tmp.data(), tmp.size() * 2, cudaMemcpyHostToDevice, st));
                    MI3D_CHECK(cudaStreamSynchronize(st));
                }
                break;
            }
            default: return Builder::load_param(P, src, partner, st);
        }
        return (int)cudaGetLastError();
    }
};

// ------------------------------------------------------------------------------------------------------------
// API-level elementwise kernels (latent arithmetic of nerf/sd.py:124-171)
// ------------------------------------------------------------------------------------------------------------
// DDIMScheduler.step, eta = 0, after set_timesteps(num_train_timesteps) (nerf/sd.py:154-155): prev = t - 1, alpha_prev = alphas[max(t-1, 0)]
// (set_alpha_to_one = False).  x0 = (x_t - sqrt(1 - a_t) eps) / sqrt(a_t);  x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps
__global__ void k_ddim_step(const float* __restrict__ noise_pred, const float* __restrict__ latents_noisy, const float* __restrict__ alphas,
                            const long long* __restrict__ t, float* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long tt = *t;
    const float a_t = alphas[tt], a_p = alphas[tt > 0 ? tt - 1 : 0];
    const float x0 = (latents_noisy[i] - sqrtf(1.f - a_t) * noise_pred[i]) / sqrtf(a_t);
    out[i] = sqrtf(a_p) * x0 + sqrtf(1.f - a_p) * noise_pred[i];
}

// decoder input: z = post_quant_conv(latents / 0.18215) (1x1 conv, 4 -> 4), latents fp32 NCHW [1,4,h,w] -> NHWC fp16 [pix][4]
__global__ void k_dec_in(const float* __restrict__ latents, const float* __restrict__ w, const float* __restrict__ b, __half* __restrict__ out, int pix) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    float x[4];
    #pragma unroll
    for (int c = 0; c < 4; c++) x[c] = latents[(size_t)c * pix + i] / 0.18215f;
    __align__(8) __half o[4];
    #pragma unroll
    for (int k = 0; k < 4; k++) o[k] = __float2half_rn(b[k] + w[4 * k] * x[0] + w[4 * k + 1] * x[1] + w[4 * k + 2] * x[2] + w[4 * k + 3] * x[3]);
    *reinterpret_cast<uint2*>(out + 4 * (size_t)i) = *reinterpret_cast<const uint2*>(o);
}

// imgs = (decoder_out / 2 + 0.5).clamp(0, 1) (nerf/sd.py:208), [pix][4] fp32 -> NCHW fp32 [1,3,S,S]
__global__ void k_dec_out(const float* __restrict__ o, float* __restrict__ imgs, int pix) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    #pragma unroll
    for (int c = 0; c < 3; c++) imgs[(size_t)c * pix + i] = fminf(fmaxf(o[4 * (size_t)i + c] / 2.f + 0.5f, 0.f), 1.f);
}

// Each API kernel below handles view blockIdx.y of a batch: view v's image, latents, noise and gradients are the v-th [C,h,w] slice.
// bilinear resize (align_corners=False, F.interpolate semantics) of pred_rgb [3,H,W] fp32 NCHW to S x S, then 2x-1, NHWC fp16 (4 ch)
__global__ void k_interp_in(const float* __restrict__ rgb, int H, int W, __half* __restrict__ out, int S) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S * S) return;
    rgb += (size_t)blockIdx.y * 3 * H * W; out += (size_t)blockIdx.y * S * S * 4;
    const int ox = i % S, oy = i / S;
    const float sx = (float)W / S, sy = (float)H / S;
    float fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f), fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f);
    const int x0 = min((int)fx, W - 1), y0 = min((int)fy, H - 1);
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float lx = fx - x0, ly = fy - y0;
    __align__(8) __half o[4];
    #pragma unroll
    for (int c = 0; c < 3; c++) {
        const float* p = rgb + (size_t)c * H * W;
        const float v = (1 - ly) * ((1 - lx) * p[y0 * W + x0] + lx * p[y0 * W + x1]) + ly * ((1 - lx) * p[y1 * W + x0] + lx * p[y1 * W + x1]);
        o[c] = __float2half_rn(2.f * v - 1.f);
    }
    o[3] = __float2half_rn(0.f);
    *reinterpret_cast<uint2*>(out + (size_t)i * 4) = *reinterpret_cast<const uint2*>(o);
}
// backward of the above: grad_rgb[c,y,x] (+)= 2 * sum over output pixels of weight * g[oy,ox,c]  (gather over the footprint)
__global__ void k_interp_bwd(const float* __restrict__ g /*[S*S][4]*/, int S, float* __restrict__ grad_rgb, int H, int W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    g += (size_t)blockIdx.y * S * S * 4; grad_rgb += (size_t)blockIdx.y * 3 * H * W;
    const int x = i % W, y = i / W;
    const float sx = (float)W / S, sy = (float)H / S;
    // output pixels whose source footprint can touch (x, y): fx in (x-1, x+1)
    const int ox_lo = max(0, (int)floorf((x - 1 + 0.5f) / sx - 0.5f)), ox_hi = min(S - 1, (int)ceilf((x + 1 + 0.5f) / sx - 0.5f));
    const int oy_lo = max(0, (int)floorf((y - 1 + 0.5f) / sy - 0.5f)), oy_hi = min(S - 1, (int)ceilf((y + 1 + 0.5f) / sy - 0.5f));
    float acc[3] = {0.f, 0.f, 0.f};
    for (int oy = oy_lo; oy <= oy_hi; oy++) {
        const float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f);
        const int y0 = min((int)fy, H - 1), y1 = min(y0 + 1, H - 1); const float ly = fy - y0;
        float wy = 0.f; if (y0 == y) wy += 1 - ly; if (y1 == y) wy += ly;
        if (wy == 0.f) continue;
        for (int ox = ox_lo; ox <= ox_hi; ox++) {
            const float fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
            const int x0 = min((int)fx, W - 1), x1 = min(x0 + 1, W - 1); const float lx = fx - x0;
            float wx = 0.f; if (x0 == x) wx += 1 - lx; if (x1 == x) wx += lx;
            if (wx == 0.f) continue;
            const float* gp = g + ((size_t)oy * S + ox) * 4;
            acc[0] += wy * wx * gp[0]; acc[1] += wy * wx * gp[1]; acc[2] += wy * wx * gp[2];
        }
    }
    #pragma unroll
    for (int c = 0; c < 3; c++) grad_rgb[(size_t)c * H * W + i] = 2.f * acc[c];
}
// moments = quant_conv(conv_out) ; latents = (mean + exp(0.5*clamp(logvar)) * eps) * 0.18215  -> fp32 NCHW [4,h,w]
__global__ void k_sample_latents(const float* __restrict__ conv_out /*[pix][8]*/, const float* __restrict__ qw /*[8][8]*/, const float* __restrict__ qb,
                                 const float* __restrict__ eps /*[4,h,w]*/, float* __restrict__ latents, int pix) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    const size_t v = blockIdx.y;
    conv_out += v * pix * 8; eps += v * pix * 4; latents += v * pix * 4;
    float m[8];
    #pragma unroll
    for (int o = 0; o < 8; o++) { float a = qb[o]; for (int k = 0; k < 8; k++) a = fmaf(qw[o * 8 + k], conv_out[(size_t)i * 8 + k], a); m[o] = a; }
    #pragma unroll
    for (int c = 0; c < 4; c++) {
        const float lv = fminf(fmaxf(m[4 + c], -30.f), 20.f);
        latents[(size_t)c * pix + i] = (m[c] + expf(0.5f * lv) * eps[(size_t)c * pix + i]) * 0.18215f;
    }
}
// backward: d conv_out[pix][8] from d latents
__global__ void k_sample_latents_bwd(const float* __restrict__ conv_out, const float* __restrict__ qw, const float* __restrict__ qb,
                                     const float* __restrict__ eps, const float* __restrict__ g_lat, float* __restrict__ g_conv_out, int pix) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    const size_t v = blockIdx.y;
    conv_out += v * pix * 8; eps += v * pix * 4; g_lat += v * pix * 4; g_conv_out += v * pix * 8;
    float m[8], gm[8];
    #pragma unroll
    for (int o = 0; o < 8; o++) { float a = qb[o]; for (int k = 0; k < 8; k++) a = fmaf(qw[o * 8 + k], conv_out[(size_t)i * 8 + k], a); m[o] = a; }
    #pragma unroll
    for (int c = 0; c < 4; c++) {
        const float g = g_lat[(size_t)c * pix + i] * 0.18215f;
        gm[c] = g;
        const float lv = m[4 + c];
        const bool pass = lv >= -30.f && lv <= 20.f;
        gm[4 + c] = pass ? g * eps[(size_t)c * pix + i] * 0.5f * expf(0.5f * lv) : 0.f;
    }
    #pragma unroll
    for (int k = 0; k < 8; k++) { float a = 0.f; for (int o = 0; o < 8; o++) a = fmaf(qw[o * 8 + k], gm[o], a); g_conv_out[(size_t)i * 8 + k] = a; }
}
// DDIM add_noise + duplicate for CFG + NCHW fp32 -> NHWC fp16 : x_in[b][p][c] = sqrt(a_t) z[c][p] + sqrt(1-a_t) eps[c][p] for the U-Net rows
// b = v (uncond) and b = G + v (text) of view v
__global__ void k_add_noise(const float* __restrict__ lat, const float* __restrict__ noise, const float* __restrict__ alphas, const long long* __restrict__ t,
                            __half* __restrict__ xin, int pix, int G) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    const int v = blockIdx.y;
    lat += (size_t)v * pix * 4; noise += (size_t)v * pix * 4;
    const float a = alphas[t[0]];
    const float sa = sqrtf(a), sb = sqrtf(1.f - a);
    __align__(8) __half o[4];
    #pragma unroll
    for (int c = 0; c < 4; c++) o[c] = __float2half_rn(sa * lat[(size_t)c * pix + i] + sb * noise[(size_t)c * pix + i]);
    *reinterpret_cast<uint2*>(xin + ((size_t)v * pix + i) * 4) = *reinterpret_cast<const uint2*>(o);
    *reinterpret_cast<uint2*>(xin + ((size_t)(G + v) * pix + i) * 4) = *reinterpret_cast<const uint2*>(o);
}
// ctx fp32 [B][L][D] -> fp16 [B][Lpad][D], zero rows beyond L
__global__ void k_ctx_pad(const float* __restrict__ ctx, __half* __restrict__ out, int B, int L, int Lpad, int D) {
    const size_t total = (size_t)B * Lpad * D;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int d = (int)(i % D); const size_t r = i / D; const int l = (int)(r % Lpad), b = (int)(r / Lpad);
        out[i] = __float2half_rn(l < L ? ctx[((size_t)b * L + l) * D + d] : 0.f);
    }
}
// CFG (sd.py:150-151: text + gs*(text - uncond)), SDS weight w = 1 - alpha_t, grad = nan_to_num(w (eps_hat - eps)); NHWC fp32 in, NCHW fp32 out.
// View v pairs U-Net rows v (uncond) and G + v (text).
__global__ void k_cfg_sds(const float* __restrict__ unet_out /*[2G][pix][4]*/, const float* __restrict__ noise, const float* __restrict__ alphas,
                          const long long* __restrict__ t, float gs, float* __restrict__ noise_pred, float* __restrict__ grad, int pix, int G) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pix) return;
    const size_t v = blockIdx.y;
    const float* un_p = unet_out + v * pix * 4; const float* tx_p = unet_out + (G + v) * pix * 4;
    noise += v * pix * 4;
    if (noise_pred) noise_pred += v * pix * 4;
    if (grad) grad += v * pix * 4;
    const float w = 1.f - alphas[t[0]];
    #pragma unroll
    for (int c = 0; c < 4; c++) {
        const float un = un_p[(size_t)i * 4 + c], tx = tx_p[(size_t)i * 4 + c];
        const float np = tx + gs * (tx - un);
        if (noise_pred) noise_pred[(size_t)c * pix + i] = np;
        float g = w * (np - noise[(size_t)c * pix + i]);
        if (isnan(g)) g = 0.f; else if (isinf(g)) g = g > 0 ? 3.4028234664e38f : -3.4028234664e38f;
        if (grad) grad[(size_t)c * pix + i] = g;
    }
}

// The per-view launches: grid (pixel blocks, G views).  The API entry points below and the mi3d_op_* test entry points both call these.
int interp_in(const float* rgb, int H, int W, __half* out, int S, int G, cudaStream_t st) {
    k_interp_in<<<dim3((S * S + 255) / 256, G), 256, 0, st>>>(rgb, H, W, out, S);
    return (int)cudaGetLastError();
}
int interp_bwd(const float* g, int S, float* grad_rgb, int H, int W, int G, cudaStream_t st) {
    k_interp_bwd<<<dim3((H * W + 127) / 128, G), 128, 0, st>>>(g, S, grad_rgb, H, W);
    return (int)cudaGetLastError();
}
int sample_latents(const float* conv_out, const float* qw, const float* qb, const float* eps, float* latents, int pix, int G, cudaStream_t st) {
    k_sample_latents<<<dim3((pix + 127) / 128, G), 128, 0, st>>>(conv_out, qw, qb, eps, latents, pix);
    return (int)cudaGetLastError();
}
int sample_latents_bwd(const float* conv_out, const float* qw, const float* qb, const float* eps, const float* g_lat, float* g_conv_out, int pix,
                       int G, cudaStream_t st) {
    k_sample_latents_bwd<<<dim3((pix + 127) / 128, G), 128, 0, st>>>(conv_out, qw, qb, eps, g_lat, g_conv_out, pix);
    return (int)cudaGetLastError();
}
int add_noise(const float* lat, const float* noise, const float* alphas, const long long* t, __half* xin, int pix, int G, cudaStream_t st) {
    k_add_noise<<<dim3((pix + 127) / 128, G), 128, 0, st>>>(lat, noise, alphas, t, xin, pix, G);
    return (int)cudaGetLastError();
}
int cfg_sds(const float* unet_out, const float* noise, const float* alphas, const long long* t, float gs, float* noise_pred, float* grad, int pix,
            int G, cudaStream_t st) {
    k_cfg_sds<<<dim3((pix + 127) / 128, G), 128, 0, st>>>(unet_out, noise, alphas, t, gs, noise_pred, grad, pix, G);
    return (int)cudaGetLastError();
}

}  // namespace sd

extern "C" {

size_t mi3d_sd_workspace_bytes(const mi3d_unet_cfg* u, const mi3d_vae_cfg* v) { return plan::workspace_bytes<sd::Engine>(u, v); }

mi3d_engine_t mi3d_sd_create(const mi3d_unet_cfg* u, const mi3d_vae_cfg* v, void* workspace, size_t workspace_bytes) {
    return plan::create<sd::Engine>(workspace, workspace_bytes, u, v);
}

int mi3d_sd_profile(mi3d_engine_t h, int enable, float* gemm_ms, int* launches) { return mi3d_sd_profile_dump(h, enable, gemm_ms, launches, nullptr); }

// dump_path_host (nullable): one text line per timed launch "M N K block_n splits conv batch epi ms" (bench.py derives FLOPs from it)
int mi3d_sd_profile_dump(mi3d_engine_t h, int enable, float* gemm_ms, int* launches, const char* dump) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep) return MI3D_ERR_ARG;
    sd::Engine& e = *ep;
    if (enable) { e.profile = true; e.prof_used = 0; return MI3D_OK; }
    e.profile = false;
    float total = 0.f; int n_tile = 0;
    FILE* f = dump ? fopen(dump, "w") : nullptr;
    for (size_t i = 0; i < e.prof_used; i++) {
        float ms = 0.f;
        MI3D_CHECK(cudaEventSynchronize(e.prof_events[i].second));
        MI3D_CHECK(cudaEventElapsedTime(&ms, e.prof_events[i].first, e.prof_events[i].second));
        if (e.prof_shapes[i].conv != 2) { total += ms; n_tile++; }
        if (f) { const auto& q = e.prof_shapes[i]; fprintf(f, "%d %d %d %d %d %d %d %d %.4f\n", q.M, q.N, q.K, q.bn, q.splits, q.conv, q.batch, q.epi, ms); }
    }
    if (f) fclose(f);
    if (gemm_ms) *gemm_ms = total;
    if (launches) *launches = n_tile;
    return MI3D_OK;
}

// nerf/sd.py:124,133,212-220 : pred_rgb [G,3,H,W] fp32 -> bilinear to image_hw -> VAE encode -> posterior sample * 0.18215, G = the planned
// images per encode
int mi3d_sd_encode(mi3d_engine_t h, const float* pred_rgb, int H, int W, const float* eps_posterior, float* latents, mi3d_stream_t stream) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep || ep->vcfg.n_levels == 0) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream; sd::Engine& e = *ep;
    const int S = e.vcfg.image_hw, G = e.vae_images();
    int r = sd::interp_in(pred_rgb, H, W, e.vae_in.p, S, G, st); if (r) return r;
    r = e.run(e.enc_ops, st); if (r) return r;
    const int pix = (int)e.v_h_last.rows() / G;
    const float* qw = (const float*)e.params[e.pindex["quant_conv.weight"]].dst; const float* qb = (const float*)e.params[e.pindex["quant_conv.bias"]].dst;
    return sd::sample_latents(e.vae_moments, qw, qb, eps_posterior, latents, pix, G, st);
}

// backward of mi3d_sd_encode w.r.t. pred_rgb (weights frozen): grad_pred_rgb [G,3,H,W] fp32 (overwritten)
int mi3d_sd_encode_backward(mi3d_engine_t h, const float* grad_latents, const float* eps_posterior, int H, int W, float* grad_pred_rgb, mi3d_stream_t stream) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep || ep->vcfg.n_levels == 0) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream; sd::Engine& e = *ep;
    const int G = e.vae_images(), pix = (int)e.v_h_last.rows() / G, S = e.vcfg.image_hw;
    const float* qw = (const float*)e.params[e.pindex["quant_conv.weight"]].dst; const float* qb = (const float*)e.params[e.pindex["quant_conv.bias"]].dst;
    int r = sd::sample_latents_bwd(e.vae_moments, qw, qb, eps_posterior, grad_latents, e.vae_gmoments, pix, G, st); if (r) return r;
    r = e.run(e.enc_bwd_ops, st); if (r) return r;
    return sd::interp_bwd(e.vae_grad_img, S, grad_pred_rgb, H, W, G, st);
}

// nerf/sd.py:154-155: one DDIM step t -> t-1 on the noisy latents with the CFG-combined noise prediction.  All fp32 [1,4,h,w].
int mi3d_sd_ddim_step(const float* noise_pred, const float* latents_noisy, const long long* t, const float* alphas_cumprod, float* prev_sample,
                      int n, mi3d_stream_t stream) {
    if (!noise_pred || !latents_noisy || !t || !alphas_cumprod || !prev_sample || n <= 0) return MI3D_ERR_ARG;
    sd::k_ddim_step<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(noise_pred, latents_noisy, alphas_cumprod, t, prev_sample, n);
    return (int)cudaGetLastError();
}

// nerf/sd.py:201-210 decode_latents: imgs = (vae.decode(latents / 0.18215).sample / 2 + 0.5).clamp(0, 1); latents fp32 [1,4,h,w] -> imgs fp32 [1,3,S,S]
int mi3d_sd_decode(mi3d_engine_t h, const float* latents, float* imgs, mi3d_stream_t stream) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep || ep->vcfg.n_levels == 0 || !ep->vcfg.decoder || !latents || !imgs) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream; sd::Engine& e = *ep;
    const int pix = (int)e.dec_in.rows(), S = e.vcfg.image_hw;
    const float* qw = (const float*)e.params[e.pindex["post_quant_conv.weight"]].dst; const float* qb = (const float*)e.params[e.pindex["post_quant_conv.bias"]].dst;
    sd::k_dec_in<<<(pix + 127) / 128, 128, 0, st>>>(latents, qw, qb, e.dec_in.p, pix);
    int r = e.run(e.dec_ops, st); if (r) return r;
    sd::k_dec_out<<<(S * S + 127) / 128, 128, 0, st>>>(e.dec_out, imgs, S * S);
    return (int)cudaGetLastError();
}

// nerf/sd.py:138-171 : add_noise -> U-Net on [uncond_0..uncond_{G-1}, text_0..text_{G-1}] -> CFG -> SDS gradient, G = batch / 2 views at one
// timestep.  t: device int64 scalar; alphas: device [1000] fp32
int mi3d_sd_unet_sds(mi3d_engine_t h, const float* latents, const float* noise, const long long* t, const float* alphas_cumprod,
                     const float* text_embeddings, float guidance_scale, float* noise_pred, float* grad, mi3d_stream_t stream) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep || ep->ucfg.n_levels == 0) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream; sd::Engine& e = *ep;
    const int pix = e.ucfg.latent_hw * e.ucfg.latent_hw, B = e.ucfg.batch;
    if (B < 2 || B % 2 || e.ucfg.in_ch != 4) return MI3D_ERR_ARG;
    const int G = B / 2;
    MI3D_CHECK(cudaMemcpyAsync(e.t_dev, t, sizeof(long long), cudaMemcpyDeviceToDevice, st));
    int r = sd::add_noise(latents, noise, alphas_cumprod, e.t_dev, e.unet_in.p, pix, G, st); if (r) return r;
    sd::k_ctx_pad<<<sd::Engine::blocks_for((size_t)B * e.ctx_pad * e.ucfg.cross_dim), 256, 0, st>>>(text_embeddings, e.ctx16, B, e.ucfg.ctx_len, e.ctx_pad, e.ucfg.cross_dim);
    r = e.run(e.unet_ops, st); if (r) return r;
    return sd::cfg_sds(e.unet_out, noise, alphas_cumprod, e.t_dev, guidance_scale, noise_pred, grad, pix, G, st);
}

// nerf/sd.py:176-199 produce_latents: n DDIM steps with CFG on the device; the text context is padded once, before the loop
int mi3d_sd_sample(mi3d_engine_t h, float* latents, const mi3d_sd_schedule* sched, int n, int prediction_type, const float* text_embeddings,
                   float guidance_scale, mi3d_stream_t stream) {
    sd::Engine* ep = plan::engine_of<sd::Engine>(h);
    if (!ep || ep->sample_ops.empty() || !latents || !sched || !text_embeddings || n < 1 || n > sd::kMaxSampleSteps ||
        (prediction_type != 0 && prediction_type != 1))
        return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream; sd::Engine& e = *ep;
    const int count = 4 * e.ucfg.latent_hw * e.ucfg.latent_hw, B = e.ucfg.batch;
    sd::k_sample_begin<<<sd::Engine::blocks_for((size_t)std::max(count, n)), 256, 0, st>>>(sched, n, latents, e.sample_sched, e.sample_lat,
                                                                                          count, e.sample_state, prediction_type, guidance_scale);
    sd::k_ctx_pad<<<sd::Engine::blocks_for((size_t)B * e.ctx_pad * e.ucfg.cross_dim), 256, 0, st>>>(text_embeddings, e.ctx16, B, e.ucfg.ctx_len, e.ctx_pad, e.ucfg.cross_dim);
    for (int i = 0; i < n; i++) { int r = e.run(e.sample_ops, st); if (r) return r; }
    MI3D_CHECK(cudaMemcpyAsync(latents, e.sample_lat, (size_t)count * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// Test entry points: one kernel of this engine with the launch geometry the engine plans (include/mi3d.h, the mi3d_op_* section)
// ------------------------------------------------------------------------------------------------------------
static int sms_of_device() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}

int mi3d_op_groupnorm(const void* x, void* y, double* stats, const float* gamma, const float* beta, int N, int HW, int C, int G, float eps,
                      int silu, int* geom, mi3d_stream_t stream) {
    sdk::GnGrid q;
    if (!x || !y || !stats || !gamma || !beta || !sdk::gn_grid(N, HW, C, G, sms_of_device(), &q)) return MI3D_ERR_ARG;
    if (geom) { geom[0] = q.chunks; geom[1] = q.ppc; geom[2] = q.PL; }
    return sdk::gn_forward(q, (const __half*)x, (__half*)y, stats, gamma, beta, N, HW, C, G, eps, silu, (cudaStream_t)stream);
}

int mi3d_op_groupnorm_bwd(const void* x, const void* dy, const double* stats, double* bstats, const float* gamma, const float* beta,
                          const void* add, void* dx, int N, int HW, int C, int G, float eps, int silu, int* geom, mi3d_stream_t stream) {
    sdk::GnGrid q;
    if (!x || !dy || !stats || !bstats || !gamma || !beta || !dx || !sdk::gn_grid(N, HW, C, G, sms_of_device(), &q)) return MI3D_ERR_ARG;
    if (geom) { geom[0] = q.chunks; geom[1] = q.ppc; geom[2] = q.PL; }
    return sdk::gn_backward(q, (const __half*)x, (const __half*)dy, stats, bstats, gamma, beta, (const __half*)add, (__half*)dx, N, HW, C, G,
                            eps, silu, (cudaStream_t)stream);
}

int mi3d_op_col2im_s2(const void* dcol, void* dx, int N, int H, int W, int C, int Ho, int Wo, int pad_lo, mi3d_stream_t stream) {
    if (N < 1 || H < 1 || W < 1 || C % 8 || Ho < 1 || Wo < 1 || (pad_lo != 0 && pad_lo != 1)) return MI3D_ERR_ARG;
    return sd::col2im_s2((const __half*)dcol, (__half*)dx, N, H, W, C, Ho, Wo, pad_lo, (cudaStream_t)stream);
}

int mi3d_op_linear_small(const float* x, const void* const* w, const float* const* bias, float* const* y, const int* N, int layers, int B, int K,
                         int silu_in, int silu_out, int grouped, mi3d_stream_t stream) {
    if (!x || !w || !bias || !y || !N || layers < 1 || layers > 64 || B < 1 || K < 8 || K % 8) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (!grouped) {
        if (layers != 1 || N[0] < 1) return MI3D_ERR_ARG;
        return sdk::linear_small(x, (const __half*)w[0], bias[0], y[0], B, N[0], K, silu_in, silu_out, st);
    }
    if (!silu_in || silu_out) return MI3D_ERR_ARG;          // the grouped kernel applies SiLU to x and nothing to y
    sdk::SmallLinearJob jobs[64]; int max_n = 0;
    for (int i = 0; i < layers; i++) {
        if (N[i] < 1) return MI3D_ERR_ARG;
        jobs[i] = {(const __half*)w[i], bias[i], y[i], N[i]}; max_n = std::max(max_n, N[i]);
    }
    sdk::SmallLinearJob* dev = nullptr;
    MI3D_CHECK(cudaMallocAsync((void**)&dev, layers * sizeof(sdk::SmallLinearJob), st));
    MI3D_CHECK(cudaMemcpyAsync(dev, jobs, layers * sizeof(sdk::SmallLinearJob), cudaMemcpyHostToDevice, st));
    const int r = sdk::linear_small_grouped(x, dev, layers, max_n, B, K, st);
    const int f = (int)cudaFreeAsync(dev, st);
    MI3D_CHECK(cudaStreamSynchronize(st));                   // the job table is host memory of this frame
    return r ? r : f;
}

int mi3d_op_interp_in(const float* rgb, int H, int W, void* out, int S, int G, mi3d_stream_t stream) {
    if (!rgb || !out || H < 1 || W < 1 || S < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::interp_in(rgb, H, W, (__half*)out, S, G, (cudaStream_t)stream);
}

int mi3d_op_interp_bwd(const float* g, int S, float* grad_rgb, int H, int W, int G, mi3d_stream_t stream) {
    if (!g || !grad_rgb || H < 1 || W < 1 || S < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::interp_bwd(g, S, grad_rgb, H, W, G, (cudaStream_t)stream);
}

int mi3d_op_sample_latents(const float* conv_out, const float* qw, const float* qb, const float* eps, float* latents, int pix, int G,
                           mi3d_stream_t stream) {
    if (!conv_out || !qw || !qb || !eps || !latents || pix < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::sample_latents(conv_out, qw, qb, eps, latents, pix, G, (cudaStream_t)stream);
}

int mi3d_op_sample_latents_bwd(const float* conv_out, const float* qw, const float* qb, const float* eps, const float* g_lat, float* g_conv_out,
                               int pix, int G, mi3d_stream_t stream) {
    if (!conv_out || !qw || !qb || !eps || !g_lat || !g_conv_out || pix < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::sample_latents_bwd(conv_out, qw, qb, eps, g_lat, g_conv_out, pix, G, (cudaStream_t)stream);
}

int mi3d_op_add_noise(const float* latents, const float* noise, const float* alphas_cumprod, const long long* t, void* xin, int pix, int G,
                      mi3d_stream_t stream) {
    if (!latents || !noise || !alphas_cumprod || !t || !xin || pix < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::add_noise(latents, noise, alphas_cumprod, t, (__half*)xin, pix, G, (cudaStream_t)stream);
}

int mi3d_op_cfg_sds(const float* unet_out, const float* noise, const float* alphas_cumprod, const long long* t, float guidance_scale,
                    float* noise_pred, float* grad, int pix, int G, mi3d_stream_t stream) {
    if (!unet_out || !noise || !alphas_cumprod || !t || pix < 1 || G < 1) return MI3D_ERR_ARG;
    return sd::cfg_sds(unet_out, noise, alphas_cumprod, t, guidance_scale, noise_pred, grad, pix, G, (cudaStream_t)stream);
}

}  // extern "C"
