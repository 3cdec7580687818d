// sd_text_engine.cu -- the Stable Diffusion text encoder (C ABI: include/mi3d.h, section B3').
//
// What `CLIPTextModel(input_ids)[0]` computes for SD-2.x (nerf/sd.py:68-85): OpenCLIP ViT-H/14's text tower truncated to 23 layers
// (width 1024, 16 heads of 64, MLP 4096 with exact GELU, causal attention, no padding mask), then final_layer_norm over every one of
// the 77 positions (last_hidden_state; no EOT pooling, no projection).  SD-1.x ships OpenAI CLIP ViT-L/14's text tower instead (12
// layers, width 768, 12 heads of 64, quick-GELU; act = 1), otherwise the same computation.  A statically planned list of
// launches: the token embedding (Builder::text_embed), the pre-LN blocks of transformer_plan.cuh with the tile GEMM's EPI_GELU or
// EPI_QUICKGELU epilogue, and a final LayerNorm that writes fp32.  Activations fp16, statistics and accumulation fp32, weights fp16 (the embeddings and LayerNorms fp32).  Forward only
// (the encoder is frozen), so all blocks share one set of activation buffers.  No split-K and no atomics: results are bit-identical
// run to run, under graph replay, and for a sequence whether it is encoded alone or in a batch.
#include "transformer_plan.cuh"
#include "warp_reduce.cuh"

namespace sdtext {

using namespace plan;

// out[b, t] = LayerNorm(x[b * Tpad + t]) in fp32 for t < T (statistics as sdk::k_layernorm).  One warp per output row.
__global__ void k_layernorm_rows_f32(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                     float* __restrict__ out, int B, int T, int Tpad, int C, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= B * T) return;
    const __half* xr = x + ((size_t)(row / T) * Tpad + row % T) * C;
    float mean, rstd;
    row_stats(xr, C, eps, lane, mean, rstd);
    float* yr = out + (size_t)row * C;
    for (int c = lane * 8; c < C; c += 256) {
        const uint4 raw = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        float o[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) o[k] = (__half2float(h[k]) - mean) * rstd * gamma[c + k] + beta[c + k];
        *reinterpret_cast<float4*>(yr + c) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(yr + c + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
}

struct Engine : TowerBuilder {
    mi3d_sd_text_cfg cfg;
    int act;                                  // 0: exact GELU, 1: quick-GELU (the MLP epilogue)
    Engine(const mi3d_sd_text_cfg& c, int a) : cfg(c), act(a) {}
    Tower t;
    std::vector<BlockW> w;
    std::vector<BlockA> a;
    long long* tokens = nullptr;
    float* out = nullptr;
    std::vector<std::vector<Op>> fwd;       // [B - 1]

    // transformers' CLIPEncoderLayer, in its state_dict order; q / k / v land in the row slices of the packed [3C][C] weight and [3C] bias
    void layer_params(const std::string& pre, int C, BlockW& bw) {
        __half* w_in = alloc16((size_t)3 * C * C);
        float* b_in = alloc32((size_t)3 * C);
        for (int s : {1, 2, 0}) {
            const std::string n = pre + ".self_attn." + "qkv"[s] + "_proj";
            param_view(n + ".weight", {C, C}, PK_LINEAR, w_in + (size_t)s * C * C);
            param_view(n + ".bias", {C}, PK_F32, b_in + (size_t)s * C);
        }
        bw.w_in = w_in; bw.b_in = b_in;
        bw.w_out = (const __half*)param(pre + ".self_attn.out_proj.weight", {C, C}, PK_LINEAR).dst;
        bw.b_out = pf(pre + ".self_attn.out_proj.bias", {C});
        bw.ln1 = pf(pre + ".layer_norm1.weight", {C}); bw.ln1_b = pf(pre + ".layer_norm1.bias", {C});
        bw.w_fc = (const __half*)param(pre + ".mlp.fc1.weight", {4 * C, C}, PK_LINEAR).dst;
        bw.b_fc = pf(pre + ".mlp.fc1.bias", {4 * C});
        bw.w_proj = (const __half*)param(pre + ".mlp.fc2.weight", {C, 4 * C}, PK_LINEAR).dst;
        bw.b_proj = pf(pre + ".mlp.fc2.bias", {C});
        bw.ln2 = pf(pre + ".layer_norm2.weight", {C}); bw.ln2_b = pf(pre + ".layer_norm2.bias", {C});
        bw.t_in = bw.t_out = bw.t_fc = bw.t_proj = nullptr;
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); named.clear();
        splitk_elems = 0;                         // no split-K: its fp32 RED order would make results vary run to run
        const mi3d_sd_text_cfg& c = cfg;
        const int C = c.width, Bm = c.max_batch;
        t.C = C; t.L = c.layers; t.heads = c.heads; t.T = c.context_len; t.Tpad = pad64(t.T);
        const float* tok = pf("text_model.embeddings.token_embedding.weight", {c.vocab, C});
        const float* pos = pf("text_model.embeddings.position_embedding.weight", {t.T, C});
        w.assign(t.L, BlockW());
        for (int i = 0; i < t.L; i++) layer_params("text_model.encoder.layers." + std::to_string(i), C, w[i]);
        const float* lnf = pf("text_model.final_layer_norm.weight", {C});
        const float* lnf_b = pf("text_model.final_layer_norm.bias", {C});
        // activations: the residual stream ping-pongs between r[0] and r[1]; the rest is scratch shared by all blocks
        const size_t M = (size_t)Bm * t.Tpad;
        tokens = (long long*)alloc((size_t)Bm * t.T * sizeof(long long));
        __half* r[2] = {alloc16(M * C), alloc16(M * C)};
        BlockA s;
        s.ln1 = alloc16(M * C); s.qkv = alloc16(M * 3 * C); s.qkvT = alloc16(M * 3 * C);
        s.S = alloc16((size_t)Bm * t.heads * t.Tpad * t.Tpad); s.ao = alloc16(M * C); s.h = alloc16(M * C);
        s.ln2 = alloc16(M * C); s.pre = nullptr; s.act = alloc16(M * 4 * C);
        a.assign(t.L, s);
        for (int i = 0; i < t.L; i++) { a[i].x = r[i & 1]; a[i].out = r[(i + 1) & 1]; }
        const __half* r_last = r[t.L & 1];
        out = alloc32((size_t)Bm * t.T * C);
        if (dry) return err;
        fwd.assign(Bm, {});
        for (int B = 1; B <= Bm; B++) {
            cur = &fwd[B - 1];
            text_embed(tokens, tok, pos, r[0], B, t.T, t.Tpad, C, c.vocab);
            float* o = out; const int Tp = t.Tpad, T = t.T;
            for (int i = 0; i < t.L; i++) block_fwd(t, w[i], a[i], B, 2, act ? tc::EPI_QUICKGELU : tc::EPI_GELU);
            push([=](cudaStream_t st) {
                k_layernorm_rows_f32<<<(unsigned)((B * T + 7) / 8), 256, 0, st>>>(r_last, lnf, lnf_b, o, B, T, Tp, C, 1e-5f);
                return (int)cudaGetLastError();
            });
        }
        cur = nullptr;
        return err;
    }
};

bool valid_cfg(const mi3d_sd_text_cfg& c) {
    return c.max_batch >= 1 && c.max_batch <= 8 && c.layers >= 1 && c.width >= 64 && c.width % 64 == 0 && c.heads * 64 == c.width &&
           c.context_len >= 1 && c.context_len <= 512 && c.vocab >= 1;
}

}  // namespace sdtext

extern "C" {

size_t mi3d_sd_text_act_workspace_bytes(const mi3d_sd_text_cfg* cfg, int act) {
    return cfg && sdtext::valid_cfg(*cfg) && (act == 0 || act == 1) ? plan::workspace_bytes<sdtext::Engine>(*cfg, act) : 0;
}

mi3d_engine_t mi3d_sd_text_act_create(const mi3d_sd_text_cfg* cfg, int act, void* workspace, size_t workspace_bytes) {
    return cfg && sdtext::valid_cfg(*cfg) && (act == 0 || act == 1) ? plan::create<sdtext::Engine>(workspace, workspace_bytes, *cfg, act)
                                                                      : nullptr;
}

size_t mi3d_sd_text_workspace_bytes(const mi3d_sd_text_cfg* cfg) { return mi3d_sd_text_act_workspace_bytes(cfg, 0); }

mi3d_engine_t mi3d_sd_text_create(const mi3d_sd_text_cfg* cfg, void* workspace, size_t workspace_bytes) {
    return mi3d_sd_text_act_create(cfg, 0, workspace, workspace_bytes);
}

int mi3d_sd_text_encode(mi3d_engine_t h, const long long* ids, int B, float* out, mi3d_stream_t stream) {
    sdtext::Engine* ep = plan::engine_of<sdtext::Engine>(h);
    if (!ep || !ids || !out) return MI3D_ERR_ARG;
    sdtext::Engine& e = *ep; const mi3d_sd_text_cfg& c = e.cfg;
    if (B < 1 || B > c.max_batch) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemcpyAsync(e.tokens, ids, (size_t)B * c.context_len * sizeof(long long), cudaMemcpyDeviceToDevice, st));
    int r = e.run(e.fwd[B - 1], st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(out, e.out, (size_t)B * c.context_len * c.width * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return MI3D_OK;
}

}  // extern "C"
