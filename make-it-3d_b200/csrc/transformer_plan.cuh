// transformer_plan.cuh -- the pre-LN transformer block shared by the CLIP towers (clip_engine.cu), the SD-2 text encoder
// (sd_text_engine.cu) and DPT's ViT-B/16 (dpt_engine.cu), built on the op builders of engine_plan.cuh.
//
// Token rows: every sequence owns Tpad = roundup(T, 64) rows; rows past T carry finite values, are masked out as keys and never reach a
// valid row.  Per-head products run as batched tile GEMMs over z = b * heads + h; head_dim is 64.
#pragma once
#include "engine_plan.cuh"

namespace plan {

struct Tower { int C = 0, L = 0, heads = 0, T = 0, Tpad = 0; float ln_eps = 1e-5f; };   // ln_eps: 1e-6 in timm's ViTs (DPT)

struct BlockW {
    const float *ln1, *ln1_b, *ln2, *ln2_b, *b_in, *b_out, *b_fc, *b_proj;
    const __half *w_in, *w_out, *w_fc, *w_proj;           // [out][in]: forward; w_in packs q, k, v as rows [3C][C]
    const __half *t_in, *t_out, *t_fc, *t_proj;           // [in][out]: input-gradient GEMMs (CLIP image tower only)
};
// one block's activations (pre: the MLP pre-activation, kept only by a taped forward)
struct BlockA { __half *x, *ln1, *qkv, *qkvT, *S, *ao, *h, *ln2, *pre, *act, *out; };

struct TowerBuilder : Builder {
    static int pad64(int t) { return (t + 63) / 64 * 64; }

    // head h of section s (0 q, 1 k, 2 v) of a [b][Tpad][ld] token matrix, K = 64 contiguous
    Mat heads_rows(const __half* p, long long ld, const Tower& t) const {
        Mat m{p, ld, t.Tpad, 64}; m.z1 = t.heads; m.sz1 = 64; m.z2 = 0; m.sz2 = (long long)t.Tpad * ld; return m;
    }
    // the same head as an operand with K = tokens: per-sequence transposed copy [b][ldT][Tpad], head rows at h*64 (+ section offset in p)
    Mat heads_cols(const __half* p, long long ldT, const Tower& t) const {
        Mat m{p, t.Tpad, 64, t.Tpad}; m.z1 = t.heads; m.sz1 = 64LL * t.Tpad; m.z2 = 0; m.sz2 = ldT * t.Tpad; return m;
    }
    // [b * heads][Tpad][Tpad] score-shaped operand
    Mat scores(const __half* p, const Tower& t) const {
        Mat m{p, t.Tpad, t.Tpad, t.Tpad}; m.z1 = t.heads; m.sz1 = (long long)t.Tpad * t.Tpad; m.z2 = 0; m.sz2 = (long long)t.heads * t.Tpad * t.Tpad; return m;
    }
    void bgemm(Mat a, Mat b, int N, __half* out, long long ldc, long long s_lo, long long s_hi, int out_z1, int B, const Tower& t) {
        a.z2 = B; b.z2 = B;
        Out o; o.p16 = out; o.ldc = ldc; o.z1 = out_z1; o.s_lo = s_lo; o.s_hi = s_hi;
        Epi e;
        gemm(a, b, N, o, e, B * t.heads, true);
    }

    // attention with the score matrix materialised: S = Q K^T, (causal) softmax, O = P V; P stays in a.S for a backward
    void attention_materialised(const Tower& t, const BlockA& a, int B, bool causal) {
        const int C = t.C, Tp = t.Tpad;
        transpose(a.qkv, a.qkvT, B, Tp, 3 * C);                                          // [b][3C][Tpad]
        bgemm(heads_rows(a.qkv, 3 * C, t), heads_rows(a.qkv + C, 3 * C, t), Tp, a.S, Tp, 0, (long long)Tp * Tp, 1, B, t);
        softmax(a.S, (size_t)B * t.heads * Tp, Tp, t.T, 0.125f, causal ? Tp : 0);
        bgemm(scores(a.S, t), heads_cols(a.qkvT + 2LL * C * Tp, 3 * C, t), 64, a.ao, C, 64, (long long)Tp * C, t.heads, B, t);
    }

    // x -> out = h + MLP(LN2(h)), h = x + Attn(LN1(x)).
    // mode 0: fused attention (no tape); 1: materialised, tape kept for the backward; 2: materialised causal (text towers).
    // act: the MLP activation epilogue of the tile GEMM (tc::EPI_QUICKGELU for CLIP, tc::EPI_GELU for the SD-2 text encoder).
    void block_fwd(const Tower& t, const BlockW& w, const BlockA& a, int B, int mode, int act) {
        const int C = t.C; const long long M = (long long)B * t.Tpad;
        layernorm(a.x, M, C, w.ln1, w.ln1_b, a.ln1, t.ln_eps);
        linear(a.ln1, M, C, w.w_in, 3 * C, a.qkv, w.b_in);
        if (mode == 0) attention_core(a.qkv, 3 * C, a.qkv + C, 3 * C, a.qkv + 2 * C, 3 * C, B, t.Tpad, t.Tpad, t.T, t.heads, 64, a.ao, C);
        else attention_materialised(t, a, B, mode == 2);
        linear(a.ao, M, C, w.w_out, C, a.h, w.b_out, a.x);
        layernorm(a.h, M, C, w.ln2, w.ln2_b, a.ln2, t.ln_eps);
        {
            Mat x{a.ln2, C, M, C}; Mat wm{w.w_fc, C, 4 * C, C};
            Out o; o.p16 = a.act; o.ldc = 4 * C;
            Epi e; e.bias = w.b_fc; e.mode = act; e.aux = mode == 1 ? a.pre : nullptr;
            gemm(x, wm, 4 * C, o, e);
        }
        linear(a.act, M, 4 * C, w.w_proj, C, a.out, w.b_proj, a.h);
    }
};

}  // namespace plan
