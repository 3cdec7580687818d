// blip2_engine.cu -- the BLIP-2 captioner (C ABI: include/mi3d.h, section B9).
//
// What `Blip2ForConditionalGeneration.generate(pixel_values)` computes for Salesforce/blip2-opt-2.7b with a default GenerationConfig
// (main.py:158-172): EVA ViT-g/14 (pre-LN, head_dim 88, exact GELU, LN eps 1e-6, post_layernorm on every token), the Q-Former (32
// learned queries, layernorm eps 1e-12, post-LN BERT layers with cross-attention to the image on every cross_attention_frequency-th
// layer and a query-only FFN), language_projection, and a greedy OPT decode (pre-LN, head_dim 80, ReLU FFN, learned positions with
// offset 2, final LayerNorm, lm_head tied to embed_tokens).
//
// Two static launch lists: `enc` (pixels -> language_model_inputs) on the tile GEMM, and per step count n `dec[n]`: the prompt, then n
// greedy steps.  A step is a causal pass over a fixed 64-row window (the prompt's num_query_tokens + 1 rows and the tokens generated so
// far; causal masking keeps the rows past the filled length away from the filled ones), so every step has the same shapes and the whole
// decode replays as one CUDA graph with no host round trip per token.  All decoder linears and lm_head run on the weight-streaming GEMM
// of blip2_kernels.cuh (a decode step is a read of OPT's 5.3 GB of weights); lm_head reads only the last filled row; the argmax, the
// append and the eos stop happen on the device.  Activations fp16, statistics and accumulation fp32, weights fp16.  No atomics and no
// split-K with REDs: results are bit-identical run to run and under graph replay.
#include "engine_plan.cuh"
#include "blip2_kernels.cuh"

namespace blip2 {

using namespace plan;

constexpr int kRows = 64;        // the decoder's row window

struct StreamPlan { int splits = 1, kc = 0; };
inline StreamPlan plan_stream(int N, int K, int num_sms) {
    const int tiles = (N + b2k::kStreamRows - 1) / b2k::kStreamRows, chunks = (K + b2k::kStreamChunk - 1) / b2k::kStreamChunk;
    // at most two CTAs per SM (one wave): a second, partial wave would leave most SMs idle at the end
    int s = std::max(1, std::min(chunks, (2 * num_sms) / tiles));
    const int per = (chunks + s - 1) / s;
    StreamPlan p; p.splits = (chunks + per - 1) / per; p.kc = per * b2k::kStreamChunk;
    return p;
}

inline int launch_stream(const __half* x, long long ldx, int M, const __half* w, int N, int K, const StreamPlan& sp, float* part,
                         const float* bias, const __half* residual, long long ld_res, int act, __half* y, float* y32, long long ldy, cudaStream_t st) {
    b2k::k_stream_gemm<<<dim3((unsigned)((N + b2k::kStreamRows - 1) / b2k::kStreamRows), (unsigned)sp.splits), 256, 0, st>>>(x, ldx, M, w, N, K, sp.kc, part);
    const size_t n = (size_t)M * N;
    b2k::k_stream_reduce<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, sp.splits, M, N, bias, residual, ld_res, act, y, y32, ldy);
    return (int)cudaGetLastError();
}

struct VisionW { const float *ln1, *ln1_b, *ln2, *ln2_b, *b_qkv, *b_proj, *b_fc1, *b_fc2; const __half *w_qkv, *w_proj, *w_fc1, *w_fc2; };
struct QLayerW {
    const __half *w_qkv, *w_out, *w_cq, *w_ckv, *w_cout, *w_fc1, *w_fc2;
    const float *b_qkv, *b_out, *ln1, *ln1_b, *b_cq, *b_ckv, *b_cout, *lnc, *lnc_b, *b_fc1, *b_fc2, *ln2, *ln2_b;
    bool cross = false;
};
struct OptW { const __half *w_qkv, *w_out, *w_fc1, *w_fc2; const float *b_qkv, *b_out, *b_fc1, *b_fc2, *ln1, *ln1_b, *ln2, *ln2_b; };

struct Engine : Builder {
    mi3d_blip2_cfg cfg;
    int Tv = 0, Tvp = 0, np = 0, Kpatch = 0, Vpad = 0, max_new = 0;
    std::map<int, int> padk;                 // param index -> padded K (the patch conv's weight)
    // device buffers
    float* pixels = nullptr; long long* ids = nullptr; int* state = nullptr; long long* eos = nullptr; long long* forced = nullptr;
    int* use_forced = nullptr; float* logits = nullptr; float* all_logits = nullptr; float* part = nullptr; size_t part_elems = 0;
    __half *img = nullptr, *qout = nullptr, *proj = nullptr;
    std::vector<Op> enc;
    std::map<int, std::vector<Op>> dec;
    // decoder plan (kept to build dec[n] on demand)
    std::vector<OptW> ow;
    const __half *tok16 = nullptr, *pos16 = nullptr; const float *lnf = nullptr, *lnf_b = nullptr;
    __half *dx[2] = {nullptr, nullptr}, *dln = nullptr, *dqkv = nullptr, *dao = nullptr, *dh = nullptr, *dact = nullptr, *dlast = nullptr;

    const __half* lin(const std::string& n, int N, int K) { return (const __half*)param(n, {N, K}, PK_LINEAR).dst; }

    void stream_linear(const __half* x, long long ldx, int M, const __half* w, int N, int K, const float* bias, const __half* residual,
                       int act, __half* y, float* y32 = nullptr) {
        const StreamPlan sp = plan_stream(N, K, num_sms);
        const size_t need = (size_t)sp.splits * M * N;
        if (need > part_elems) part_elems = need;
        if (dry) return;
        if (K % 32 || M > 64 || need > part_elems) { err = MI3D_ERR_ARG; return; }
        float* pt = part;
        push([=](cudaStream_t st) { return launch_stream(x, ldx, M, w, N, K, sp, pt, bias, residual, N, act, y, y32, N, st); });
    }
    void attn(const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv, __half* o, long long ldo,
              int T, int Tk, int kv_valid, int heads, int d, bool causal) {
        const float scale = 1.f / sqrtf((float)d);
        push([=](cudaStream_t st) {
            b2k::k_attn_rows<<<dim3((unsigned)((T + 7) / 8), (unsigned)heads, 1), 256, 0, st>>>(q, ldq, k, ldk, v, ldv, o, ldo, T, Tk, kv_valid, d,
                                                                                             scale, causal ? 1 : 0);
            return (int)cudaGetLastError();
        });
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); named.clear(); padk.clear();
        splitk_elems = 0;                                 // the tile GEMM runs without split-K (its fp32 RED order varies run to run)
        const mi3d_blip2_cfg& c = cfg;
        const int Cv = c.vision_width, Cq = c.qformer_width, Co = c.opt_width, nq = c.num_query_tokens;
        const int g = c.image_size / c.patch; np = g * g; Tv = np + 1; Tvp = (Tv + 63) / 64 * 64;
        Kpatch = (3 * c.patch * c.patch + 63) / 64 * 64;
        Vpad = (c.vocab + 63) / 64 * 64;
        max_new = kRows - nq - 1;
        // ---- parameters, in transformers' state_dict order
        const __half* query16 = (const __half*)param("query_tokens", {1, nq, Cq}, PK_LINEAR).dst;
        const float* cls = pf("vision_model.embeddings.class_embedding", {1, 1, Cv});
        const float* vpos = pf("vision_model.embeddings.position_embedding", {1, Tv, Cv});
        __half* wpatch = alloc16((size_t)Cv * Kpatch);
        param_view("vision_model.embeddings.patch_embedding.weight", {Cv, 3, c.patch, c.patch}, PK_LINEAR, wpatch);
        padk[pindex["vision_model.embeddings.patch_embedding.weight"]] = Kpatch;
        const float* bpatch = pf("vision_model.embeddings.patch_embedding.bias", {Cv});
        std::vector<VisionW> vw(c.vision_layers);
        for (int i = 0; i < c.vision_layers; i++) {
            const std::string p = "vision_model.encoder.layers." + std::to_string(i);
            VisionW& w = vw[i];
            w.w_qkv = lin(p + ".self_attn.qkv.weight", 3 * Cv, Cv); w.b_qkv = pf(p + ".self_attn.qkv.bias", {3 * Cv});
            w.w_proj = lin(p + ".self_attn.projection.weight", Cv, Cv); w.b_proj = pf(p + ".self_attn.projection.bias", {Cv});
            w.ln1 = pf(p + ".layer_norm1.weight", {Cv}); w.ln1_b = pf(p + ".layer_norm1.bias", {Cv});
            w.w_fc1 = lin(p + ".mlp.fc1.weight", c.vision_mlp, Cv); w.b_fc1 = pf(p + ".mlp.fc1.bias", {c.vision_mlp});
            w.w_fc2 = lin(p + ".mlp.fc2.weight", Cv, c.vision_mlp); w.b_fc2 = pf(p + ".mlp.fc2.bias", {Cv});
            w.ln2 = pf(p + ".layer_norm2.weight", {Cv}); w.ln2_b = pf(p + ".layer_norm2.bias", {Cv});
        }
        const float* vpost = pf("vision_model.post_layernorm.weight", {Cv}); const float* vpost_b = pf("vision_model.post_layernorm.bias", {Cv});
        const float* qln = pf("qformer.layernorm.weight", {Cq}); const float* qln_b = pf("qformer.layernorm.bias", {Cq});
        std::vector<QLayerW> qw(c.qformer_layers);
        for (int i = 0; i < c.qformer_layers; i++) {
            const std::string p = "qformer.encoder.layer." + std::to_string(i);
            QLayerW& w = qw[i];
            __half* wqkv = alloc16((size_t)3 * Cq * Cq); float* bqkv = alloc32((size_t)3 * Cq);
            for (int s = 0; s < 3; s++) {
                const std::string n = p + ".attention.attention." + (s == 0 ? "query" : s == 1 ? "key" : "value");
                param_view(n + ".weight", {Cq, Cq}, PK_LINEAR, wqkv + (size_t)s * Cq * Cq);
                param_view(n + ".bias", {Cq}, PK_F32, bqkv + (size_t)s * Cq);
            }
            w.w_qkv = wqkv; w.b_qkv = bqkv;
            w.w_out = lin(p + ".attention.output.dense.weight", Cq, Cq); w.b_out = pf(p + ".attention.output.dense.bias", {Cq});
            w.ln1 = pf(p + ".attention.output.LayerNorm.weight", {Cq}); w.ln1_b = pf(p + ".attention.output.LayerNorm.bias", {Cq});
            w.cross = i % c.cross_attention_frequency == 0;
            if (w.cross) {
                w.w_cq = lin(p + ".crossattention.attention.query.weight", Cq, Cq); w.b_cq = pf(p + ".crossattention.attention.query.bias", {Cq});
                __half* wkv = alloc16((size_t)2 * Cq * Cv); float* bkv = alloc32((size_t)2 * Cq);
                for (int s = 0; s < 2; s++) {
                    const std::string n = p + ".crossattention.attention." + (s == 0 ? "key" : "value");
                    param_view(n + ".weight", {Cq, Cv}, PK_LINEAR, wkv + (size_t)s * Cq * Cv);
                    param_view(n + ".bias", {Cq}, PK_F32, bkv + (size_t)s * Cq);
                }
                w.w_ckv = wkv; w.b_ckv = bkv;
                w.w_cout = lin(p + ".crossattention.output.dense.weight", Cq, Cq); w.b_cout = pf(p + ".crossattention.output.dense.bias", {Cq});
                w.lnc = pf(p + ".crossattention.output.LayerNorm.weight", {Cq}); w.lnc_b = pf(p + ".crossattention.output.LayerNorm.bias", {Cq});
            }
            w.w_fc1 = lin(p + ".intermediate_query.dense.weight", c.qformer_ffn, Cq); w.b_fc1 = pf(p + ".intermediate_query.dense.bias", {c.qformer_ffn});
            w.w_fc2 = lin(p + ".output_query.dense.weight", Cq, c.qformer_ffn); w.b_fc2 = pf(p + ".output_query.dense.bias", {Cq});
            w.ln2 = pf(p + ".output_query.LayerNorm.weight", {Cq}); w.ln2_b = pf(p + ".output_query.LayerNorm.bias", {Cq});
        }
        const __half* wlp = lin("language_projection.weight", Co, Cq); const float* blp = pf("language_projection.bias", {Co});
        const std::string d = "language_model.model.decoder.";
        __half* tok = alloc16((size_t)Vpad * Co);                      // rows >= vocab stay zero (the workspace is zero-filled)
        param_view(d + "embed_tokens.weight", {c.vocab, Co}, PK_LINEAR, tok);
        tok16 = tok;
        pos16 = lin(d + "embed_positions.weight", c.max_positions + 2, Co);
        lnf = pf(d + "final_layer_norm.weight", {Co}); lnf_b = pf(d + "final_layer_norm.bias", {Co});
        ow.assign(c.opt_layers, OptW());
        for (int i = 0; i < c.opt_layers; i++) {
            const std::string p = d + "layers." + std::to_string(i);
            OptW& w = ow[i];
            __half* wqkv = alloc16((size_t)3 * Co * Co); float* bqkv = alloc32((size_t)3 * Co);
            for (int s : {1, 2, 0}) {                              // state_dict order k, v, q; packed q, k, v
                const std::string n = p + ".self_attn." + "qkv"[s] + "_proj";
                param_view(n + ".weight", {Co, Co}, PK_LINEAR, wqkv + (size_t)s * Co * Co);
                param_view(n + ".bias", {Co}, PK_F32, bqkv + (size_t)s * Co);
            }
            w.w_qkv = wqkv; w.b_qkv = bqkv;
            w.w_out = lin(p + ".self_attn.out_proj.weight", Co, Co); w.b_out = pf(p + ".self_attn.out_proj.bias", {Co});
            w.ln1 = pf(p + ".self_attn_layer_norm.weight", {Co}); w.ln1_b = pf(p + ".self_attn_layer_norm.bias", {Co});
            w.w_fc1 = lin(p + ".fc1.weight", c.opt_ffn, Co); w.b_fc1 = pf(p + ".fc1.bias", {c.opt_ffn});
            w.w_fc2 = lin(p + ".fc2.weight", Co, c.opt_ffn); w.b_fc2 = pf(p + ".fc2.bias", {Co});
            w.ln2 = pf(p + ".final_layer_norm.weight", {Co}); w.ln2_b = pf(p + ".final_layer_norm.bias", {Co});
        }
        // ---- activations and state
        pixels = alloc32((size_t)3 * c.image_size * c.image_size);
        __half* col = alloc16((size_t)Tvp * Kpatch);
        __half* pe = alloc16((size_t)Tvp * Cv);
        __half* vx[2] = {alloc16((size_t)Tvp * Cv), alloc16((size_t)Tvp * Cv)};
        __half* vln = alloc16((size_t)Tvp * Cv); __half* vqkv = alloc16((size_t)Tvp * 3 * Cv); __half* vao = alloc16((size_t)Tvp * Cv);
        __half* vh = alloc16((size_t)Tvp * Cv); __half* vact = alloc16((size_t)Tvp * c.vision_mlp);
        img = alloc16((size_t)Tvp * Cv);
        __half* q0 = alloc16((size_t)nq * Cq); __half* qx[2] = {alloc16((size_t)nq * Cq), alloc16((size_t)nq * Cq)};
        __half* qqkv = alloc16((size_t)nq * 3 * Cq); __half* qao = alloc16((size_t)nq * Cq); __half* qt = alloc16((size_t)nq * Cq);
        __half* qh1 = alloc16((size_t)nq * Cq); __half* qh2 = alloc16((size_t)nq * Cq); __half* qcq = alloc16((size_t)nq * Cq);
        __half* qckv = alloc16((size_t)Tvp * 2 * Cq); __half* qact = alloc16((size_t)nq * c.qformer_ffn);
        proj = alloc16((size_t)nq * Co);
        ids = (long long*)alloc(kRows * sizeof(long long));
        state = (int*)alloc(16 * sizeof(int));
        eos = (long long*)alloc(sizeof(long long));
        use_forced = (int*)alloc(sizeof(int));
        forced = (long long*)alloc(kRows * sizeof(long long));
        dx[0] = alloc16((size_t)kRows * Co); dx[1] = alloc16((size_t)kRows * Co);
        dln = alloc16((size_t)kRows * Co); dqkv = alloc16((size_t)kRows * 3 * Co); dao = alloc16((size_t)kRows * Co);
        dh = alloc16((size_t)kRows * Co); dact = alloc16((size_t)kRows * c.opt_ffn); dlast = alloc16((size_t)Co);
        logits = alloc32((size_t)Vpad);
        all_logits = alloc32((size_t)max_new * c.vocab);
        // the streaming GEMM's partial sums: sized by a dry pass over the decoder's shapes
        part_elems = 0;
        {
            const bool was = dry; dry = true;
            stream_linear(nullptr, Co, kRows, nullptr, 3 * Co, Co, nullptr, nullptr, 0, nullptr);
            stream_linear(nullptr, Co, kRows, nullptr, Co, Co, nullptr, nullptr, 0, nullptr);
            stream_linear(nullptr, Co, kRows, nullptr, c.opt_ffn, Co, nullptr, nullptr, 0, nullptr);
            stream_linear(nullptr, c.opt_ffn, kRows, nullptr, Co, c.opt_ffn, nullptr, nullptr, 0, nullptr);
            stream_linear(nullptr, Co, 1, nullptr, c.vocab, Co, nullptr, nullptr, 0, nullptr);
            dry = was;
        }
        part = alloc32(part_elems);
        tap("image_embeds", img, (size_t)Tv * Cv * 2);
        tap("query_output", qx[c.qformer_layers & 1], (size_t)nq * Cq * 2);
        tap("language_model_inputs", proj, (size_t)nq * Co * 2);
        if (dry) return err;

        // ================= encode: pixels -> language_model_inputs =================
        enc.clear(); cur = &enc;
        {
            const float* px = pixels; const int S = c.image_size, P = c.patch, Kp = Kpatch, npp = np;
            push([=](cudaStream_t st) {
                b2k::k_patch_cols<<<blocks_for((size_t)npp * Kp), 256, 0, st>>>(px, S, P, Kp, col);
                return (int)cudaGetLastError();
            });
            linear(col, np, Kpatch, wpatch, Cv, pe, bpatch);
            __half* x0 = vx[0];
            push([=](cudaStream_t st) {
                b2k::k_vision_embed<<<blocks_for((size_t)(npp + 1) * Cv), 256, 0, st>>>(pe, cls, vpos, x0, npp, Cv);
                return (int)cudaGetLastError();
            });
        }
        const long long Mv = Tvp;
        const int dv = Cv / c.vision_heads;
        for (int i = 0; i < c.vision_layers; i++) {
            const VisionW& w = vw[i];
            __half* x = vx[i & 1]; __half* y = vx[(i + 1) & 1];
            layernorm(x, Mv, Cv, w.ln1, w.ln1_b, vln, 1e-6f);
            linear(vln, Mv, Cv, w.w_qkv, 3 * Cv, vqkv, w.b_qkv);
            attn(vqkv, 3 * Cv, vqkv + Cv, 3 * Cv, vqkv + 2 * Cv, 3 * Cv, vao, Cv, Tv, Tvp, Tv, c.vision_heads, dv, false);
            linear(vao, Mv, Cv, w.w_proj, Cv, vh, w.b_proj, x);
            layernorm(vh, Mv, Cv, w.ln2, w.ln2_b, vln, 1e-6f);
            {
                Mat a{vln, Cv, Mv, Cv}; Mat b{w.w_fc1, Cv, c.vision_mlp, Cv};
                Out o; o.p16 = vact; o.ldc = c.vision_mlp;
                Epi e; e.bias = w.b_fc1; e.mode = tc::EPI_GELU;
                gemm(a, b, c.vision_mlp, o, e);
            }
            linear(vact, Mv, c.vision_mlp, w.w_fc2, Cv, y, w.b_fc2, vh);
        }
        layernorm(vx[c.vision_layers & 1], Mv, Cv, vpost, vpost_b, img, 1e-6f);
        // Q-Former over the learned queries
        layernorm(query16, nq, Cq, qln, qln_b, q0, 1e-12f);
        const int dq = Cq / c.qformer_heads;
        for (int i = 0; i < c.qformer_layers; i++) {
            const QLayerW& w = qw[i];
            const __half* x = i == 0 ? q0 : qx[i & 1];
            __half* y = qx[(i + 1) & 1];
            linear(x, nq, Cq, w.w_qkv, 3 * Cq, qqkv, w.b_qkv);
            attn(qqkv, 3 * Cq, qqkv + Cq, 3 * Cq, qqkv + 2 * Cq, 3 * Cq, qao, Cq, nq, nq, nq, c.qformer_heads, dq, false);
            linear(qao, nq, Cq, w.w_out, Cq, qt, w.b_out, x);
            layernorm(qt, nq, Cq, w.ln1, w.ln1_b, qh1, 1e-12f);
            const __half* h = qh1;
            if (w.cross) {
                linear(qh1, nq, Cq, w.w_cq, Cq, qcq, w.b_cq);
                linear(img, Tvp, Cv, w.w_ckv, 2 * Cq, qckv, w.b_ckv);
                attn(qcq, Cq, qckv, 2 * Cq, qckv + Cq, 2 * Cq, qao, Cq, nq, Tvp, Tv, c.qformer_heads, dq, false);
                linear(qao, nq, Cq, w.w_cout, Cq, qt, w.b_cout, qh1);
                layernorm(qt, nq, Cq, w.lnc, w.lnc_b, qh2, 1e-12f);
                h = qh2;
            }
            {
                Mat a{h, Cq, nq, Cq}; Mat b{w.w_fc1, Cq, c.qformer_ffn, Cq};
                Out o; o.p16 = qact; o.ldc = c.qformer_ffn;
                Epi e; e.bias = w.b_fc1; e.mode = tc::EPI_GELU;
                gemm(a, b, c.qformer_ffn, o, e);
            }
            linear(qact, nq, c.qformer_ffn, w.w_fc2, Cq, qt, w.b_fc2, h);
            layernorm(qt, nq, Cq, w.ln2, w.ln2_b, y, 1e-12f);
        }
        linear(qx[c.qformer_layers & 1], nq, Cq, wlp, Co, proj, blp);
        cur = nullptr;
        return err;
    }

    // dec[n]: the prompt, then n greedy steps over the 64-row window
    std::vector<Op>* decode_list(int n) {
        auto it = dec.find(n);
        if (it != dec.end()) return &it->second;
        std::vector<Op>& L = dec[n];
        cur = &L; err = 0;
        const mi3d_blip2_cfg& c = cfg;
        const int Co = c.opt_width, nq = c.num_query_tokens, V = c.vocab, dh_ = Co / c.opt_heads;
        {
            long long* id = ids; int* stp = state; const long long it_ = c.image_token_index, bos = c.bos_token_id;
            push([=](cudaStream_t st) {
                b2k::k_decoder_start<<<1, 64, 0, st>>>(id, stp, kRows, nq, it_, bos);
                return (int)cudaGetLastError();
            });
        }
        for (int s = 0; s < n; s++) {
            {
                long long* id = ids; const __half* pr = proj; const __half* tk = tok16; const __half* ps = pos16; __half* x0 = dx[0];
                push([=](cudaStream_t st) {
                    b2k::k_decoder_embed<<<blocks_for((size_t)kRows * Co), 256, 0, st>>>(id, pr, tk, ps, x0, kRows, nq, Co, V);
                    return (int)cudaGetLastError();
                });
            }
            for (int i = 0; i < c.opt_layers; i++) {
                const OptW& w = ow[i];
                __half* x = dx[i & 1]; __half* y = dx[(i + 1) & 1];
                layernorm(x, kRows, Co, w.ln1, w.ln1_b, dln, 1e-5f);
                stream_linear(dln, Co, kRows, w.w_qkv, 3 * Co, Co, w.b_qkv, nullptr, 0, dqkv);
                attn(dqkv, 3 * Co, dqkv + Co, 3 * Co, dqkv + 2 * Co, 3 * Co, dao, Co, kRows, kRows, kRows, c.opt_heads, dh_, true);
                stream_linear(dao, Co, kRows, w.w_out, Co, Co, w.b_out, x, 0, dh);
                layernorm(dh, kRows, Co, w.ln2, w.ln2_b, dln, 1e-5f);
                stream_linear(dln, Co, kRows, w.w_fc1, c.opt_ffn, Co, w.b_fc1, nullptr, 1, dact);
                stream_linear(dact, c.opt_ffn, kRows, w.w_fc2, Co, c.opt_ffn, w.b_fc2, dh, 0, y);
            }
            {
                const __half* xl = dx[c.opt_layers & 1]; const int* stp = state; __half* last = dlast;
                push([=](cudaStream_t st) {
                    b2k::k_last_row<<<1, 256, 0, st>>>(xl, stp, last, Co);
                    return (int)cudaGetLastError();
                });
            }
            layernorm(dlast, 1, Co, lnf, lnf_b, dln, 1e-5f);
            stream_linear(dln, Co, 1, tok16, V, Co, nullptr, nullptr, 0, nullptr, logits);
            {
                const float* lg = logits; long long* id = ids; int* stp = state; const long long* eo = eos; const long long* fo = forced;
                const int* uf = use_forced; float* al = all_logits;
                push([=](cudaStream_t st) {
                    b2k::k_greedy_pick<<<1, 1024, 0, st>>>(lg, V, id, stp, eo, fo, uf, al);
                    return (int)cudaGetLastError();
                });
            }
        }
        cur = nullptr;
        if (err) { dec.erase(n); return nullptr; }
        return &L;
    }
};

bool valid_cfg(const mi3d_blip2_cfg& c) {
    auto heads_ok = [](int w, int h) { return h >= 1 && w % h == 0 && (w / h) % 8 == 0 && w / h <= 128; };
    if (c.patch < 1 || c.image_size < c.patch || c.image_size % c.patch) return false;
    const int g = c.image_size / c.patch, Tv = g * g + 1;
    return Tv <= b2k::kAttnMaxKeys && c.vision_width % 64 == 0 && c.vision_layers >= 1 && heads_ok(c.vision_width, c.vision_heads) &&
           c.vision_mlp % 64 == 0 && c.qformer_width % 64 == 0 && c.qformer_layers >= 1 && heads_ok(c.qformer_width, c.qformer_heads) &&
           c.qformer_ffn % 64 == 0 && c.cross_attention_frequency >= 1 && c.num_query_tokens >= 1 && c.num_query_tokens <= kRows - 2 &&
           c.opt_width % 64 == 0 && c.opt_layers >= 1 && heads_ok(c.opt_width, c.opt_heads) && c.opt_ffn % 32 == 0 && c.vocab >= 1 &&
           c.max_positions >= kRows && c.image_token_index >= 0 && c.image_token_index < c.vocab && c.bos_token_id >= 0 && c.bos_token_id < c.vocab;
}

}  // namespace blip2

struct mi3d_blip2 { blip2::Engine e; };

extern "C" {

size_t mi3d_blip2_workspace_bytes(const mi3d_blip2_cfg* cfg) {
    if (!cfg || !blip2::valid_cfg(*cfg)) return 0;
    blip2::Engine e; e.cfg = *cfg;
    if (e.build(true)) return 0;
    return e.off + (1 << 20);
}

mi3d_blip2_t mi3d_blip2_create(const mi3d_blip2_cfg* cfg, void* workspace, size_t workspace_bytes) {
    if (!cfg || !workspace || !blip2::valid_cfg(*cfg)) return nullptr;
    mi3d_blip2* h = new mi3d_blip2();
    h->e.cfg = *cfg; h->e.base = (uint8_t*)workspace; h->e.cap = workspace_bytes;
    int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&h->e.num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (h->e.build(false) != 0) { delete h; return nullptr; }
    return h;
}

void mi3d_blip2_destroy(mi3d_blip2_t h) { delete h; }

int mi3d_blip2_num_params(mi3d_blip2_t h) { return h ? (int)h->e.params.size() : 0; }
const char* mi3d_blip2_param_name(mi3d_blip2_t h, int i) {
    if (!h || i < 0 || i >= (int)h->e.params.size()) return nullptr;
    return h->e.params[i].name.c_str();
}
int mi3d_blip2_param_shape(mi3d_blip2_t h, int i, int* shape4) {
    if (!h || !shape4 || i < 0 || i >= (int)h->e.params.size()) return -1;
    const auto& s = h->e.params[i].shape;
    for (int k = 0; k < 4; k++) shape4[k] = k < (int)s.size() ? s[k] : 0;
    return (int)s.size();
}

int mi3d_blip2_load_param(mi3d_blip2_t h, int i, const float* src, mi3d_stream_t stream) {
    if (!h || i < 0 || i >= (int)h->e.params.size() || !src) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const plan::Param& P = h->e.params[i];
    auto pk = h->e.padk.find(i);
    if (pk != h->e.padk.end()) {
        const int N = P.shape[0], K = (int)(P.numel / N);
        b2k::k_f32_to_f16_padk<<<plan::Builder::blocks_for((size_t)N * pk->second), 256, 0, st>>>(src, (__half*)P.dst, N, K, pk->second);
        return (int)cudaGetLastError();
    }
    switch (P.kind) {
        case plan::PK_F32: MI3D_CHECK(cudaMemcpyAsync(P.dst, src, P.numel * 4, cudaMemcpyDeviceToDevice, st)); break;
        case plan::PK_LINEAR: sdk::k_f32_to_f16<<<plan::Builder::blocks_for(P.numel), 256, 0, st>>>(src, (__half*)P.dst, P.numel); break;
        default: return MI3D_ERR_ARG;
    }
    return (int)cudaGetLastError();
}

int mi3d_blip2_set_graph_replay(mi3d_blip2_t h, int enable) {
    if (!h) return MI3D_ERR_ARG;
    h->e.use_graph = enable != 0;
    return MI3D_OK;
}

int mi3d_blip2_graph_replays(mi3d_blip2_t h) { return h ? h->e.graph_replays() : -1; }

int mi3d_blip2_encode(mi3d_blip2_t h, const float* pixel_values, float* out, mi3d_stream_t stream) {
    if (!h || !pixel_values) return MI3D_ERR_ARG;
    blip2::Engine& e = h->e; const mi3d_blip2_cfg& c = e.cfg;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemcpyAsync(e.pixels, pixel_values, (size_t)3 * c.image_size * c.image_size * 4, cudaMemcpyDeviceToDevice, st));
    int r = e.run(e.enc, st); if (r) return r;
    if (out) {
        const size_t n = (size_t)c.num_query_tokens * c.opt_width;
        b2k::k_f16_to_f32<<<plan::Builder::blocks_for(n), 256, 0, st>>>(e.proj, out, n);
        return (int)cudaGetLastError();
    }
    return MI3D_OK;
}

int mi3d_blip2_generate(mi3d_blip2_t h, const float* pixel_values, int max_new_tokens, long long eos_token_id, const long long* forced_ids,
                        long long* ids, int* count, float* step_logits, mi3d_stream_t stream) {
    if (!h || !pixel_values || !ids || !count) return MI3D_ERR_ARG;
    blip2::Engine& e = h->e; const mi3d_blip2_cfg& c = e.cfg;
    if (max_new_tokens < 1 || max_new_tokens > e.max_new) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<plan::Op>* L = e.decode_list(max_new_tokens);
    if (!L) return MI3D_ERR_ARG;
    // per-call scalars live in the workspace, so the launch lists (and their graphs) do not depend on them
    static thread_local long long eos_h; static thread_local int uf_h;
    eos_h = eos_token_id; uf_h = forced_ids ? 1 : 0;
    MI3D_CHECK(cudaMemcpyAsync(e.eos, &eos_h, sizeof(long long), cudaMemcpyHostToDevice, st));
    MI3D_CHECK(cudaMemcpyAsync(e.use_forced, &uf_h, sizeof(int), cudaMemcpyHostToDevice, st));
    if (forced_ids) MI3D_CHECK(cudaMemcpyAsync(e.forced, forced_ids, (size_t)max_new_tokens * sizeof(long long), cudaMemcpyDeviceToDevice, st));
    int r = mi3d_blip2_encode(h, pixel_values, nullptr, stream); if (r) return r;
    r = e.run(*L, st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(ids, e.ids, blip2::kRows * sizeof(long long), cudaMemcpyDeviceToDevice, st));
    MI3D_CHECK(cudaMemcpyAsync(count, e.state, sizeof(int), cudaMemcpyDeviceToDevice, st));
    if (step_logits) MI3D_CHECK(cudaMemcpyAsync(step_logits, e.all_logits, (size_t)max_new_tokens * c.vocab * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return MI3D_OK;
}

int mi3d_blip2_tap(mi3d_blip2_t h, const char* name, float* dst, mi3d_stream_t stream) {
    if (!h || !name || !dst) return MI3D_ERR_ARG;
    auto it = h->e.named.find(name);
    if (it == h->e.named.end()) return MI3D_ERR_ARG;
    const size_t n = it->second.second / 2;
    b2k::k_f16_to_f32<<<plan::Builder::blocks_for(n), 256, 0, (cudaStream_t)stream>>>((const __half*)it->second.first, dst, n);
    return (int)cudaGetLastError();
}

size_t mi3d_stream_gemm_workspace_bytes(int M, int N, int K) {
    if (M < 1 || M > 64 || N < 1 || K < 32 || K % 32) return 0;
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaGetLastError();
    const blip2::StreamPlan p = blip2::plan_stream(N, K, sms);
    return (size_t)p.splits * M * N * sizeof(float);
}

int mi3d_stream_gemm_f16(const void* x, const void* w, const float* bias, const void* residual, int relu, void* y, int M, int N, int K,
                         void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    if (!x || !w || !y || !workspace || M < 1 || M > 64 || N < 1 || K < 32 || K % 32) return MI3D_ERR_ARG;
    int dev = 0, sms = 132;
    MI3D_CHECK(cudaGetDevice(&dev)); MI3D_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const blip2::StreamPlan p = blip2::plan_stream(N, K, sms);
    if (workspace_bytes < (size_t)p.splits * M * N * sizeof(float)) return MI3D_ERR_ARG;
    return blip2::launch_stream((const __half*)x, K, M, (const __half*)w, N, K, p, (float*)workspace, bias, (const __half*)residual, N,
                                relu ? 1 : 0, (__half*)y, nullptr, N, (cudaStream_t)stream);
}

}  // extern "C"
