// clip_engine.cu -- CLIP ViT image tower (with input gradient) and text tower (C ABI: include/mi3d.h, section B4).
//
// Replaces what openai CLIP's encode_image / encode_text run for the per-step CLIP losses of the training step
// (nerf/utils.py:436-453, nerf/sd.py:97-114): a statically planned list of launches over the tile GEMM (tc_gemm.cuh) and the fused
// attention (attn.cuh), built with the op builders shared with the SD engine (engine_plan.cuh) and the transformer block shared with
// the SD-2 text encoder (transformer_plan.cuh), plus the kernels of clip_kernels.cuh.
// Token rows: every image / prompt owns Tpad = roundup(T, 64) rows (197 -> 256 image tokens, 77 -> 128 text tokens); rows past T are
// zero at the embedding, carry finite values through the blocks, are masked out as keys and never reach a valid row, so every
// attention product of the input-gradient pass has K a multiple of 64.  Activations fp16, statistics and accumulation fp32, weights
// fp16 copies (plus transposed copies for the input-gradient GEMMs) of the fp32 openai parameters.  The CLIP weights are frozen: the
// backward computes the input gradient only.  No split-K and no atomics: results are bit-reproducible run to run and under graph replay.
#include "transformer_plan.cuh"

namespace clip {

using namespace plan;

// scratch of the reverse walk, shared by all blocks (they run one after the other)
struct BwdA { __half *dpre, *dln2, *dh, *dao, *daoT, *dS, *PT, *dST, *dqkv, *dln1; };

struct Engine : TowerBuilder {
    mi3d_clip_cfg cfg;
    explicit Engine(const mi3d_clip_cfg& c) : cfg(c) {}
    Tower vt, tt;
    int np = 0, G = 0, KP = 0;
    std::vector<BlockW> vw, tw;
    std::vector<BlockA> va, ta;
    BwdA bw;
    // image tower I/O and fixed buffers
    __half *patches = nullptr, *pe = nullptr, *x0 = nullptr, *cls = nullptr, *clsn = nullptr;
    float* img_feats = nullptr;
    float* gscale = nullptr;                        // power-of-two scale of the input-gradient pass (k_grad_in)
    __half *dfeat16 = nullptr, *dcls = nullptr, *dclsx = nullptr, *dx0 = nullptr, *dpe = nullptr, *dpatch = nullptr;
    std::vector<__half*> dres;                      // gradient of the residual stream after block i (index L: after the last block)
    // text tower
    long long* tokens = nullptr; __half *tx0 = nullptr, *eot = nullptr, *eotn = nullptr; float* txt_feats = nullptr;
    // launch lists: [b - 1]
    std::vector<std::vector<Op>> img_fwd, img_fwd_tape, img_bwd, txt_fwd;
    // the tape of the last image forward
    bool tape_valid = false; int tape_B = 0, tape_H = 0, tape_W = 0, tape_aug = 0;

    void block_params(const std::string& pre, int C, bool both, BlockW& w) {
        const PKind k = both ? PK_LINEAR_BOTH : PK_LINEAR;
        auto lin = [&](const std::string& n, int o, int i, const __half** fw, const __half** bw_) {
            Param& P = param(pre + n, {o, i}, k); *fw = (const __half*)P.dst; *bw_ = (const __half*)P.dst2;
        };
        w.ln1 = pf(pre + ".ln_1.weight", {C}); w.ln1_b = pf(pre + ".ln_1.bias", {C});
        lin(".attn.in_proj_weight", 3 * C, C, &w.w_in, &w.t_in); w.b_in = pf(pre + ".attn.in_proj_bias", {3 * C});
        lin(".attn.out_proj.weight", C, C, &w.w_out, &w.t_out); w.b_out = pf(pre + ".attn.out_proj.bias", {C});
        w.ln2 = pf(pre + ".ln_2.weight", {C}); w.ln2_b = pf(pre + ".ln_2.bias", {C});
        lin(".mlp.c_fc.weight", 4 * C, C, &w.w_fc, &w.t_fc); w.b_fc = pf(pre + ".mlp.c_fc.bias", {4 * C});
        lin(".mlp.c_proj.weight", C, 4 * C, &w.w_proj, &w.t_proj); w.b_proj = pf(pre + ".mlp.c_proj.bias", {C});
    }
    // one block's activations, sized for max_batch; every launch list of the tower (any batch) uses the same buffers
    BlockA block_bufs(const Tower& t, __half* x) {
        const size_t M = (size_t)cfg.max_batch * t.Tpad, C = t.C;
        BlockA a; a.x = x;
        a.ln1 = alloc16(M * C); a.qkv = alloc16(M * 3 * C); a.qkvT = alloc16(M * 3 * C);
        a.S = alloc16((size_t)cfg.max_batch * t.heads * t.Tpad * t.Tpad); a.ao = alloc16(M * C); a.h = alloc16(M * C);
        a.ln2 = alloc16(M * C); a.pre = alloc16(M * 4 * C); a.act = alloc16(M * 4 * C); a.out = alloc16(M * C);
        return a;
    }

    // dx = LayerNorm input gradient of dy (+ add)
    void layernorm_bwd(const __half* x, const __half* dy, const float* gamma, const __half* add, __half* dx, long long rows, int C) {
        push([=](cudaStream_t st) {
            clipk::k_layernorm_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, dy, gamma, add, dx, (int)rows, C, 1e-5f);
            return (int)cudaGetLastError();
        });
    }
    void block_bwd(const Tower& t, const BlockW& w, const BlockA& a, int n, const __half* dout, __half* dx) {
        const int C = t.C, Tp = t.Tpad; const long long M = (long long)n * Tp;
        {   // c_proj input gradient, times QuickGELU'(pre-activation)
            Mat x{dout, C, M, C}; Mat wm{w.t_proj, C, 4 * C, C};
            Out o; o.p16 = bw.dpre; o.ldc = 4 * C;
            Epi e; e.mode = tc::EPI_QUICKGELU_BWD; e.aux = a.pre;
            gemm(x, wm, 4 * C, o, e);
        }
        linear(bw.dpre, M, 4 * C, w.t_fc, C, bw.dln2);
        layernorm_bwd(a.h, bw.dln2, w.ln2, dout, bw.dh, M, C);
        linear(bw.dh, M, C, w.t_out, C, bw.dao);
        // attention: dP = dO V^T ; dV = P^T dO ; dS = softmax'(P, dP) / 8 ; dQ = dS K ; dK = dS^T Q  -> dqkv [M][3C]
        transpose(bw.dao, bw.daoT, n, Tp, C);
        bgemm(heads_rows(bw.dao, C, t), heads_rows(a.qkv + 2 * C, 3 * C, t), Tp, bw.dS, Tp, 0, (long long)Tp * Tp, 1, n, t);
        transpose(a.S, bw.PT, n * t.heads, Tp, Tp);
        bgemm(scores(bw.PT, t), heads_cols(bw.daoT, C, t), 64, bw.dqkv + 2 * C, 3 * C, 64, (long long)Tp * 3 * C, t.heads, n, t);
        {
            const __half* P = a.S; __half* dS = bw.dS; const size_t rows = (size_t)n * t.heads * Tp;
            push([=](cudaStream_t st) {
                sdk::k_softmax_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(P, dS, rows, Tp, 0.125f);
                return (int)cudaGetLastError();
            });
        }
        bgemm(scores(bw.dS, t), heads_cols(a.qkvT + (long long)C * Tp, 3 * C, t), 64, bw.dqkv, 3 * C, 64, (long long)Tp * 3 * C, t.heads, n, t);
        transpose(bw.dS, bw.dST, n * t.heads, Tp, Tp);
        bgemm(scores(bw.dST, t), heads_cols(a.qkvT, 3 * C, t), 64, bw.dqkv + C, 3 * C, 64, (long long)Tp * 3 * C, t.heads, n, t);
        linear(bw.dqkv, M, 3 * C, w.t_in, C, bw.dln1);
        layernorm_bwd(a.x, bw.dln1, w.ln1, bw.dh, dx, M, C);
    }

    const float* ln_param(const std::string& pre, int C) { const float* w = pf(pre + ".weight", {C}); pf(pre + ".bias", {C}); return w; }

    void plan_image() {
        const mi3d_clip_cfg& c = cfg; Tower& t = vt;
        const int C = c.width, Bm = c.max_batch;
        G = c.image_res / c.patch; np = G * G; KP = 3 * c.patch * c.patch;
        t.C = C; t.L = c.layers; t.heads = c.heads; t.T = np + 1; t.Tpad = pad64(t.T);
        const Param& conv1 = param("visual.conv1.weight", {C, 3, c.patch, c.patch}, PK_LINEAR_BOTH);
        const __half *w_patch = (const __half*)conv1.dst, *t_patch = (const __half*)conv1.dst2;
        const float* cls_emb = pf("visual.class_embedding", {C});
        const float* pos = pf("visual.positional_embedding", {t.T, C});
        const float* ln_pre = ln_param("visual.ln_pre", C);
        vw.assign(t.L, BlockW());
        for (int i = 0; i < t.L; i++) {
            const std::string pre = "visual.transformer.resblocks." + std::to_string(i);
            block_params(pre, C, true, vw[i]);
        }
        const float* ln_post = ln_param("visual.ln_post", C);
        const __half* w_proj = (const __half*)param("visual.proj", {C, c.embed_dim}, PK_LINEAR_T).dst;
        const __half* t_proj = (const __half*)param("visual.proj#dgrad", {C, c.embed_dim}, PK_LINEAR).dst;
        // buffers
        const long long Mm = (long long)Bm * t.Tpad;
        patches = alloc16((size_t)Bm * np * KP); pe = alloc16((size_t)Bm * np * C); x0 = alloc16(Mm * C);
        __half* r0 = alloc16(Mm * C);
        va.clear();
        __half* x = r0;
        for (int i = 0; i < t.L; i++) { va.push_back(block_bufs(t, x)); x = va.back().out; }
        __half* r_last = x;
        cls = alloc16((size_t)Bm * C); clsn = alloc16((size_t)Bm * C); img_feats = alloc32((size_t)Bm * c.embed_dim);
        bw.dpre = alloc16(Mm * 4 * C); bw.dln2 = alloc16(Mm * C); bw.dh = alloc16(Mm * C); bw.dao = alloc16(Mm * C); bw.daoT = alloc16(Mm * C);
        const size_t sc = (size_t)Bm * t.heads * t.Tpad * t.Tpad;
        bw.dS = alloc16(sc); bw.PT = alloc16(sc); bw.dST = alloc16(sc); bw.dqkv = alloc16(Mm * 3 * C); bw.dln1 = alloc16(Mm * C);
        dres.assign(t.L + 1, nullptr);
        for (int i = 0; i <= t.L; i++) dres[i] = alloc16(Mm * C);
        gscale = alloc32(1); dfeat16 = alloc16((size_t)Bm * c.embed_dim); dcls = alloc16((size_t)Bm * C); dclsx = alloc16((size_t)Bm * C);
        dx0 = alloc16(Mm * C); dpe = alloc16((size_t)Bm * np * C); dpatch = alloc16((size_t)Bm * np * KP);
        if (dry) return;
        img_fwd.assign(Bm, {}); img_fwd_tape.assign(Bm, {}); img_bwd.assign(Bm, {});
        for (int B = 1; B <= Bm; B++) {
            for (int tape = 0; tape < 2; tape++) {
                cur = tape ? &img_fwd_tape[B - 1] : &img_fwd[B - 1];
                const long long M = (long long)B * t.Tpad;
                linear(patches, (long long)B * np, KP, w_patch, C, pe);
                { const __half* p = pe; __half* xx = x0; const int Tp = t.Tpad, npp = np;
                  push([=](cudaStream_t st) {
                      clipk::k_image_embed<<<blocks_for((size_t)B * Tp * C / 8), 256, 0, st>>>(p, cls_emb, pos, xx, B, npp, Tp, C);
                      return (int)cudaGetLastError();
                  }); }
                layernorm(x0, M, C, "visual.ln_pre", r0);
                for (int i = 0; i < t.L; i++) block_fwd(t, vw[i], va[i], B, tape, tc::EPI_QUICKGELU);
                gather_rows(r_last, (size_t)t.Tpad * C, cls, C, C, B);
                layernorm(cls, B, C, "visual.ln_post", clsn);
                Mat a{clsn, C, B, C}; Mat wm{w_proj, C, c.embed_dim, C};
                Out o; o.p32 = img_feats; o.ldc = c.embed_dim; Epi e;
                gemm(a, wm, c.embed_dim, o, e);
            }
            // input gradient of the first B images of the last taped forward
            cur = &img_bwd[B - 1];
            const int n = B; const long long M = (long long)n * t.Tpad;
            linear(dfeat16, n, c.embed_dim, t_proj, C, dcls);
            layernorm_bwd(cls, dcls, ln_post, nullptr, dclsx, n, C);
            { __half* d = dres[t.L]; push([=](cudaStream_t st) { return (int)cudaMemsetAsync(d, 0, (size_t)M * C * 2, st); }); }
            gather_rows(dclsx, C, dres[t.L], (size_t)t.Tpad * C, C, n);
            for (int i = t.L - 1; i >= 0; i--) block_bwd(t, vw[i], va[i], n, dres[i + 1], dres[i]);
            layernorm_bwd(x0, dres[0], ln_pre, nullptr, dx0, M, C);
            { // patch rows 1 .. np of every image
                const __half* s = dx0 + C; __half* d = dpe; const int Tp = t.Tpad, npp = np;
                push([=](cudaStream_t st) {
                    return (int)cudaMemcpy2DAsync(d, (size_t)npp * C * 2, s, (size_t)Tp * C * 2, (size_t)npp * C * 2, n, cudaMemcpyDeviceToDevice, st);
                });
            }
            linear(dpe, (long long)n * np, C, t_patch, KP, dpatch);
        }
        cur = nullptr;
    }

    // rows r = 0 .. count-1: dst[r * ld_dst] = src[r * ld_src] (C halves each)
    void gather_rows(const __half* src, size_t ld_src, __half* dst, size_t ld_dst, int C, int count) {
        push([=](cudaStream_t st) {
            return (int)cudaMemcpy2DAsync(dst, ld_dst * 2, src, ld_src * 2, (size_t)C * 2, count, cudaMemcpyDeviceToDevice, st);
        });
    }

    void plan_text() {
        const mi3d_clip_cfg& c = cfg; Tower& t = tt;
        const int C = c.text_width, Bm = c.max_batch;
        t.C = C; t.L = c.text_layers; t.heads = c.text_heads; t.T = c.context_len; t.Tpad = pad64(t.T);
        const float* tok = pf("token_embedding.weight", {c.vocab, C});
        const float* pos = pf("positional_embedding", {t.T, C});
        tw.assign(t.L, BlockW());
        for (int i = 0; i < t.L; i++) {
            const std::string pre = "transformer.resblocks." + std::to_string(i);
            block_params(pre, C, false, tw[i]);
        }
        ln_param("ln_final", C);
        const __half* w_proj = (const __half*)param("text_projection", {C, c.embed_dim}, PK_LINEAR_T).dst;
        const long long Mm = (long long)Bm * t.Tpad;
        tokens = (long long*)alloc((size_t)Bm * t.T * sizeof(long long));
        tx0 = alloc16(Mm * C);
        ta.clear();
        __half* x = tx0;
        for (int i = 0; i < t.L; i++) { ta.push_back(block_bufs(t, x)); x = ta.back().out; }
        __half* r_last = x;
        eot = alloc16((size_t)Bm * C); eotn = alloc16((size_t)Bm * C); txt_feats = alloc32((size_t)Bm * c.embed_dim);
        if (dry) return;
        txt_fwd.assign(Bm, {});
        for (int B = 1; B <= Bm; B++) {
            cur = &txt_fwd[B - 1];
            const long long* tk = tokens; __half* xx = tx0; const int Tp = t.Tpad, T = t.T, V = c.vocab;
            push([=](cudaStream_t st) {
                clipk::k_text_embed<<<blocks_for((size_t)B * Tp * C / 8), 256, 0, st>>>(tk, tok, pos, xx, B, T, Tp, C, V);
                return (int)cudaGetLastError();
            });
            for (int i = 0; i < t.L; i++) block_fwd(t, tw[i], ta[i], B, 2, tc::EPI_QUICKGELU);
            __half* rows = eot;
            push([=](cudaStream_t st) {
                clipk::k_text_eot_rows<<<B, 128, 0, st>>>(tk, r_last, rows, T, Tp, C);
                return (int)cudaGetLastError();
            });
            layernorm(eot, B, C, "ln_final", eotn);
            Mat a{eotn, C, B, C}; Mat wm{w_proj, C, c.embed_dim, C};
            Out o; o.p32 = txt_feats; o.ldc = c.embed_dim; Epi e;
            gemm(a, wm, c.embed_dim, o, e);
        }
        cur = nullptr;
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); named.clear();
        splitk_elems = 0;                         // no split-K: its fp32 RED order would make results vary run to run
        if (cfg.layers > 0) plan_image();
        if (cfg.text_layers > 0) plan_text();
        pf("logit_scale", {});
        return err;
    }
};

bool valid_cfg(const mi3d_clip_cfg& c) {
    if (c.max_batch < 1 || c.max_batch > 8 || c.embed_dim < 64 || c.embed_dim % 64) return false;
    if (c.layers < 0 || c.text_layers < 0 || (c.layers == 0 && c.text_layers == 0)) return false;
    if (c.layers > 0 && (c.width % 64 || c.heads * 64 != c.width || c.patch < 8 || c.patch % 8 || c.image_res % c.patch ||
                         (3 * c.patch * c.patch) % 64)) return false;
    if (c.text_layers > 0 && (c.text_width % 64 || c.text_heads * 64 != c.text_width || c.context_len < 1 || c.vocab < 1)) return false;
    return true;
}

}  // namespace clip

extern "C" {

size_t mi3d_clip_workspace_bytes(const mi3d_clip_cfg* cfg) {
    return cfg && clip::valid_cfg(*cfg) ? plan::workspace_bytes<clip::Engine>(*cfg) : 0;
}

mi3d_engine_t mi3d_clip_create(const mi3d_clip_cfg* cfg, void* workspace, size_t workspace_bytes) {
    return cfg && clip::valid_cfg(*cfg) ? plan::create<clip::Engine>(workspace, workspace_bytes, *cfg) : nullptr;
}

int mi3d_clip_encode_image(mi3d_engine_t h, const float* img, int B, int H, int W, int aug, int need_grad, float* feats, mi3d_stream_t stream) {
    clip::Engine* ep = plan::engine_of<clip::Engine>(h);
    if (!ep || ep->cfg.layers == 0 || !img || !feats) return MI3D_ERR_ARG;
    clip::Engine& e = *ep; const mi3d_clip_cfg& c = e.cfg;
    if (B < 1 || B > c.max_batch || H < 1 || W < 1 || (!aug && (H != c.image_res || W != c.image_res))) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    e.tape_valid = false;
    const size_t work = (size_t)B * e.np * e.KP / 8;
    clipk::k_preprocess<<<plan::Builder::blocks_for(work), 256, 0, st>>>(img, B, H, W, c.image_res, c.patch, aug ? 1 : 0, e.patches);
    MI3D_CHECK(cudaGetLastError());
    int r = e.run(need_grad ? e.img_fwd_tape[B - 1] : e.img_fwd[B - 1], st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(feats, e.img_feats, (size_t)B * c.embed_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (need_grad) { e.tape_valid = true; e.tape_B = B; e.tape_H = H; e.tape_W = W; e.tape_aug = aug ? 1 : 0; }
    return MI3D_OK;
}

int mi3d_clip_encode_image_backward(mi3d_engine_t h, const float* dfeats, int n_grad, float* dimg, mi3d_stream_t stream) {
    clip::Engine* ep = plan::engine_of<clip::Engine>(h);
    if (!ep || !dfeats || !dimg) return MI3D_ERR_ARG;
    clip::Engine& e = *ep; const mi3d_clip_cfg& c = e.cfg;
    if (!e.tape_valid || n_grad < 1 || n_grad > e.tape_B) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    clipk::k_grad_in<<<1, 256, 0, st>>>(dfeats, n_grad * c.embed_dim, e.dfeat16, e.gscale);
    MI3D_CHECK(cudaGetLastError());
    int r = e.run(e.img_bwd[n_grad - 1], st); if (r) return r;
    const size_t total = (size_t)n_grad * 3 * e.tape_H * e.tape_W;
    clipk::k_preprocess_bwd<<<plan::Builder::blocks_for(total), 256, 0, st>>>(e.dpatch, n_grad, e.tape_H, e.tape_W, c.image_res, c.patch, e.tape_aug, e.gscale, dimg);
    return (int)cudaGetLastError();
}

int mi3d_clip_encode_text(mi3d_engine_t h, const long long* tokens, int B, float* feats, mi3d_stream_t stream) {
    clip::Engine* ep = plan::engine_of<clip::Engine>(h);
    if (!ep || ep->cfg.text_layers == 0 || !tokens || !feats) return MI3D_ERR_ARG;
    clip::Engine& e = *ep; const mi3d_clip_cfg& c = e.cfg;
    if (B < 1 || B > c.max_batch) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemcpyAsync(e.tokens, tokens, (size_t)B * c.context_len * sizeof(long long), cudaMemcpyDeviceToDevice, st));
    int r = e.run(e.txt_fwd[B - 1], st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(feats, e.txt_feats, (size_t)B * c.embed_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return MI3D_OK;
}

}  // extern "C"
