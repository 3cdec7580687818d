// tc_test.cu -- C-ABI entry points that run single ops of the engines' op layer (plan::Builder / plan::TowerBuilder) through the
// builder methods the engines call (the tile GEMM, both implicit convs and both attention paths planned as in production, and the row
// kernels), for the parity tests and for tools/ timing.
#include "transformer_plan.cuh"
#include "../../include/mi3d.h"

namespace {

// A builder that records into a local list (the engines' real-build state: dry = false, this device's SM count), with the tile
// kernel's launches bracketed by events so that the planned block-N / split count can be reported.
struct OneOp {
    plan::TowerBuilder b;
    std::vector<plan::Op> ops;
    OneOp(void* splitk_ws = nullptr, size_t splitk_bytes = 0) {
        b.dry = false; b.cur = &ops; b.profile = true;
        int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&b.num_sms, cudaDevAttrMultiProcessorCount, dev);
        b.splitk_ws = (float*)splitk_ws; b.splitk_elems = splitk_ws ? splitk_bytes / sizeof(float) : 0;
    }
    ~OneOp() { for (auto& e : b.prof_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); } }
    int run(mi3d_stream_t stream, int* plan = nullptr) {
        if (b.err) return b.err;
        if (ops.empty()) return MI3D_ERR_ARG;
        const int r = b.run_eager(ops, (cudaStream_t)stream);
        if (!r && plan && b.prof_used) { plan[0] = b.prof_shapes[0].bn; plan[1] = b.prof_shapes[0].splits; }
        return r;
    }
};

plan::T4 t4(const void* p, int n, int h, int w, int c) { plan::T4 t; t.p = (__half*)p; t.n = n; t.h = h; t.w = w; t.c = c; return t; }

}  // namespace

extern "C" {

int mi3d_op_gemm(const mi3d_op_gemm_args* g, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream) {
    if (!g) return MI3D_ERR_ARG;
    OneOp op(splitk_ws, splitk_bytes);
    plan::Builder::Mat a{(const __half*)g->a, g->lda, g->a_rows, g->K, g->a_z1, g->a_sz1, g->a_z2, g->a_sz2};
    plan::Builder::Mat b{(const __half*)g->b, g->ldb, g->b_rows, g->K, g->b_z1, g->b_sz1, g->b_z2, g->b_sz2};
    plan::Builder::Out o; o.p16 = (__half*)g->out16; o.p32 = (float*)g->out32; o.ldc = g->ldc; o.z1 = g->out_z1; o.s_lo = g->out_s_lo; o.s_hi = g->out_s_hi;
    plan::Builder::Epi e; e.bias = g->bias; e.row_bias = g->row_bias; e.rows_per_group = g->rows_per_group; e.residual = (const __half*)g->residual;
    e.ld_res = g->ld_res; e.mode = g->mode; e.alpha = g->alpha; e.aux = (__half*)g->aux;
    op.b.gemm(a, b, g->N, o, e, g->batch, g->b_batched != 0);
    return op.run(stream, plan);
}

int mi3d_op_conv3(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const float* bias, const float* row_bias,
                  const void* residual, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream) {
    OneOp op(splitk_ws, splitk_bytes);
    op.b.conv3(t4(x, Nimg, H, W, Cin), (const __half*)w, Cout, t4(y, Nimg, H, W, Cout), bias, row_bias, (const __half*)residual);
    return op.run(stream, plan);
}

// the im2col matrix of Builder::conv3_s2 is carved out of `col` (the builder's workspace)
int mi3d_op_conv3_s2(const void* x, const void* w, void* y, int Nimg, int H, int W, int C, int Ho, int Wo, int Cout, const float* bias, int pad_lo,
                     void* col, size_t col_bytes, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream) {
    if (!col || (pad_lo != 0 && pad_lo != 1) || C % 8 || Ho < 1 || Wo < 1) return MI3D_ERR_ARG;
    OneOp op(splitk_ws, splitk_bytes);
    op.b.base = (uint8_t*)col; op.b.cap = col_bytes;
    op.b.conv3_s2(t4(x, Nimg, H, W, C), (const __half*)w, t4(y, Nimg, Ho, Wo, Cout), bias, pad_lo);
    return op.run(stream, plan);
}

int mi3d_op_conv_small_cin(const void* x, const float* w, const float* bias, void* y, int Nimg, int H, int W, int Cin, int Cout, mi3d_stream_t stream) {
    OneOp op;
    op.b.conv_small_cin(t4(x, Nimg, H, W, Cin), w, bias, t4(y, Nimg, H, W, Cout));
    return op.run(stream);
}

int mi3d_op_conv_small_cout(const void* x, const void* w, const float* bias, float* y, int Nimg, int H, int W, int Cin, int Cout,
                            mi3d_stream_t stream) {
    OneOp op;
    op.b.conv_small_cout(t4(x, Nimg, H, W, Cin), (const __half*)w, bias, y, Cout);
    return op.run(stream);
}

int mi3d_op_conv3_block(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const float* bias, int mode,
                        const void* aux, const void* residual, int* plan, mi3d_stream_t stream) {
    OneOp op;
    op.b.conv3_block(t4(x, Nimg, H, W, Cin), (const __half*)w, Cout, t4(y, Nimg, H, W, Cout), bias, mode, (const __half*)aux,
                     (const __half*)residual);
    return op.run(stream, plan);
}

int mi3d_op_attention_core(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                           int B, int T, int Tk, int Tk_valid, int heads, int head_dim, mi3d_stream_t stream) {
    if (B < 1 || T < 1 || Tk < 1 || Tk_valid < 1 || Tk_valid > Tk || heads < 1 || (ldq | ldk | ldv | ldo) % 8) return MI3D_ERR_ARG;
    OneOp op;
    op.b.attention_core((const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, B, T, Tk, Tk_valid, heads, head_dim, (__half*)o, (int)ldo);
    return op.run(stream);
}

int mi3d_op_attention(const void* qkv, void* qkvT, void* S, void* o, int B, int T, int Tpad, int heads, int mode, mi3d_stream_t stream) {
    if (B < 1 || heads < 1 || T < 1 || T > Tpad || Tpad % 64 || mode < 0 || mode > 2) return MI3D_ERR_ARG;
    OneOp op;
    plan::Tower t; t.C = 64 * heads; t.heads = heads; t.T = T; t.Tpad = Tpad; t.L = 1;
    plan::BlockA a = {};
    a.qkv = (__half*)qkv; a.qkvT = (__half*)qkvT; a.S = (__half*)S; a.ao = (__half*)o;
    if (mode == 0) op.b.attention_core(a.qkv, 3 * t.C, a.qkv + t.C, 3 * t.C, a.qkv + 2 * t.C, 3 * t.C, B, Tpad, Tpad, T, heads, 64, a.ao, t.C);
    else op.b.attention_materialised(t, a, B, mode == 2);
    return op.run(stream);
}

int mi3d_op_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, int C, float eps, mi3d_stream_t stream) {
    if (rows < 1 || C % 8) return MI3D_ERR_ARG;
    OneOp op;
    op.b.layernorm((const __half*)x, rows, C, gamma, beta, (__half*)y, eps);
    return op.run(stream);
}

int mi3d_op_layernorm_bwd(const void* x, const void* dy, const float* gamma, const void* add, void* dx, int rows, int C, float eps,
                          mi3d_stream_t stream) {
    if (rows < 1 || C % 8) return MI3D_ERR_ARG;
    OneOp op;
    op.b.layernorm_bwd((const __half*)x, (const __half*)dy, gamma, (const __half*)add, (__half*)dx, rows, C, eps);
    return op.run(stream);
}

int mi3d_op_softmax(void* s, size_t rows, int cols, int valid, int causal_tq, float scale, mi3d_stream_t stream) {
    if (rows < 1 || cols % 8 || valid < 1 || valid > cols) return MI3D_ERR_ARG;
    OneOp op;
    op.b.softmax((__half*)s, rows, cols, valid, scale, causal_tq);
    return op.run(stream);
}

int mi3d_op_softmax_bwd(const void* p, void* dp, size_t rows, int cols, float scale, mi3d_stream_t stream) {
    if (rows < 1 || cols % 8) return MI3D_ERR_ARG;
    OneOp op;
    op.b.softmax_bwd((const __half*)p, (__half*)dp, rows, cols, scale);
    return op.run(stream);
}

int mi3d_op_transpose(const void* in, void* out, int Z, int R, int C, mi3d_stream_t stream) {
    if (Z < 1 || R < 1 || C < 1) return MI3D_ERR_ARG;
    OneOp op;
    op.b.transpose((const __half*)in, (__half*)out, Z, R, C);
    return op.run(stream);
}

}  // extern "C"
