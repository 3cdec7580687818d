// tc_test.cu -- C-ABI entry points that expose the raw tensor-core tile kernel (used by the parity tests and by
// tools/ for roofline measurements; the SD engine calls the same tc::launch), and single ops of the engines' op layer.
#include "tc_host.cuh"
#include "attn.cuh"
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

// D[M,N] (fp16 or fp32) = alpha * A[M,K] . B[N,K]^T + bias[N] (+ residual)
static int gemm_f16_impl(const void* a, const void* b, void* out, int out_is_f32, int M, int N, int K, int block_n, float alpha,
                  const float* bias, const void* residual, int epi_mode, int b_mn, mi3d_stream_t stream, int splits = 1, float* ws = nullptr) {
    if (M % 128 || K % 64) return MI3D_ERR_ARG;
    if (block_n == 0) block_n = tc::pick_block_n(N, M / 128, 132, tc::has_block_n_160(epi_mode, 0));
    if (block_n == 0 || N % block_n) return MI3D_ERR_ARG;
    CUtensorMap ma, mb;
    int r = tc::make_map_matrix(&ma, (const __half*)a, K, M, K, 128);
    if (r) return r;
    if (b_mn) {   // B given as [K][N]: boxes of [64 k rows][64 n]
        const uint64_t dims[4] = {(uint64_t)N, (uint64_t)K, 1, 1};
        const uint64_t str[4] = {2, (uint64_t)N * 2, (uint64_t)N * K * 2, (uint64_t)N * K * 2};
        const uint32_t box[4] = {64, 64, 1, 1};
        r = tc::make_map_f16(&mb, b, dims, str, box);
    } else r = tc::make_map_matrix(&mb, (const __half*)b, K, N, K, block_n);
    if (r) return r;
    tc::GemmParams p = {};
    p.b_mn = b_mn; p.splits = 1;
    p.M = M; p.N = N; p.K = K; p.num_k_blocks = K / 64; p.conv = 0; p.a_z1 = 1; p.b_z1 = 1; p.b_batched = 0;
    p.out = out_is_f32 ? nullptr : (__half*)out; p.out_f32 = out_is_f32 ? (float*)out : nullptr;
    p.ldc = epi_mode == tc::EPI_GEGLU ? N / 2 : (epi_mode == tc::EPI_TRANSPOSED ? M : N);
    p.out_z1 = 1; p.out_s_lo = 0; p.out_s_hi = 0; p.bias = bias; p.row_bias = nullptr; p.rows_per_group = 1;
    p.residual = (const __half*)residual; p.ld_res = N; p.epi_mode = epi_mode; p.alpha = alpha; p.m_valid = M;
    if (splits > 1) return tc::launch_splitk(ma, mb, p, block_n, splits, ws, (cudaStream_t)stream);
    return tc::launch(ma, mb, p, block_n, 1, (cudaStream_t)stream);
}

int mi3d_gemm_f16(const void* a, const void* b, void* out, int out_is_f32, int M, int N, int K, int block_n, float alpha,
                  const float* bias, const void* residual, int epi_mode, mi3d_stream_t stream) {
    return gemm_f16_impl(a, b, out, out_is_f32, M, N, K, block_n, alpha, bias, residual, epi_mode, 0, stream);
}
// split-K variant (fp16 out, plain epilogue): K is cut into `splits` ranges whose partial sums meet in ws (fp32 [M][N])
int mi3d_gemm_f16_splitk(const void* a, const void* b, void* out, int M, int N, int K, int block_n, int splits, float alpha,
                         const float* bias, const void* residual, void* ws, mi3d_stream_t stream) {
    if (splits < 1 || splits > K / 64 || !ws) return MI3D_ERR_ARG;
    return gemm_f16_impl(a, b, out, 0, M, N, K, block_n, alpha, bias, residual, 0, 0, stream, splits, (float*)ws);
}
// test path: out[M,N] = A[M,K] . Bt[K,N]  (B consumed as an MN-major UMMA operand)
int mi3d_gemm_f16_bt(const void* a, const void* bt, void* out, int M, int N, int K, int block_n, mi3d_stream_t stream) {
    return gemm_f16_impl(a, bt, out, 1, M, N, K, block_n, 1.f, nullptr, nullptr, 0, 1, stream);
}

// fused attention on token matrices: q [B*T, ldq], k / v [B*Tk, ld] (head h at column h*64, d = 64), o [B*T, ldo]
int mi3d_flash_attn_f16(const void* q, const void* k, const void* v, void* o, int B, int T, int Tk, int Tk_valid, int heads,
                        int ldq, int ldk, int ldv, int ldo, mi3d_stream_t stream) {
    if (B < 1 || T < 1 || Tk < 1 || Tk_valid < 1 || Tk_valid > Tk || heads < 1 || (ldq | ldk | ldv | ldo) % 8) return MI3D_ERR_ARG;
    attn::Maps m;
    int r = attn::make_maps(&m, (const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, B, T, Tk, heads, 64);
    if (r) return r;
    return attn::launch(m, (__half*)o, ldo, B, T, Tk_valid, heads, (cudaStream_t)stream);
}

// 3x3 stride-1 pad-1 convolution, NHWC fp16: x [N,H,W,Cin], w [Cout][3][3][Cin], y [N,H,W,Cout]
int mi3d_conv3x3_f16(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, int block_n,
                     const float* bias, const void* residual, mi3d_stream_t stream) {
    const long long Mtot = (long long)Nimg * H * W;
    if (Mtot % 128 || Cin % 64) return MI3D_ERR_ARG;
    int bw = W < 128 ? W : 128, bh = 128 / bw; if (bh > H) bh = H; int bn = 128 / (bw * bh);
    if (bw * bh * bn != 128 || W % bw || H % bh || Nimg % bn) return MI3D_ERR_ARG;
    if (block_n == 0) block_n = tc::pick_block_n(Cout, Mtot / 128, 132);
    if (block_n == 0 || Cout % block_n) return MI3D_ERR_ARG;
    CUtensorMap ma, mb;
    int r = tc::make_map_nhwc(&ma, (const __half*)x, Cin, W, H, Nimg, bw, bh, bn);
    if (r) return r;
    r = tc::make_map_matrix(&mb, (const __half*)w, 9ull * Cin, Cout, 9ull * Cin, block_n);
    if (r) return r;
    tc::GemmParams p = {};
    p.splits = 1;
    p.M = (int)Mtot; p.N = Cout; p.K = 9 * Cin; p.num_k_blocks = 9 * (Cin / 64); p.conv = 1;
    p.conv_H = H; p.conv_W = W; p.conv_bw = bw; p.conv_bh = bh; p.cin_blocks = Cin / 64;
    p.a_z1 = 1; p.b_z1 = 1; p.b_batched = 0;
    p.out = (__half*)y; p.out_f32 = nullptr; p.ldc = Cout; p.out_z1 = 1; p.out_s_lo = 0; p.out_s_hi = 0; p.bias = bias; p.row_bias = nullptr;
    p.rows_per_group = 1; p.residual = (const __half*)residual; p.ld_res = Cout; p.epi_mode = tc::EPI_PLAIN; p.alpha = 1.f;
    p.m_valid = (int)Mtot;
    return tc::launch(ma, mb, p, block_n, 1, (cudaStream_t)stream);
}

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
    clipk::k_layernorm_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const __half*)x, (const __half*)dy, gamma,
                                                                                         (const __half*)add, (__half*)dx, rows, C, eps);
    return (int)cudaGetLastError();
}

int mi3d_op_softmax(void* s, size_t rows, int cols, int valid, int causal_tq, float scale, mi3d_stream_t stream) {
    if (rows < 1 || cols % 8 || valid < 1 || valid > cols) return MI3D_ERR_ARG;
    if (causal_tq > 0) {
        clipk::k_softmax_causal<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((__half*)s, rows, cols, valid, causal_tq, scale);
        return (int)cudaGetLastError();
    }
    OneOp op;
    op.b.softmax((__half*)s, rows, cols, valid, scale);
    return op.run(stream);
}

int mi3d_op_softmax_bwd(const void* p, void* dp, size_t rows, int cols, float scale, mi3d_stream_t stream) {
    if (rows < 1 || cols % 8) return MI3D_ERR_ARG;
    sdk::k_softmax_bwd<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const __half*)p, (__half*)dp, rows, cols, scale);
    return (int)cudaGetLastError();
}

int mi3d_op_transpose(const void* in, void* out, int Z, int R, int C, mi3d_stream_t stream) {
    if (Z < 1 || R < 1 || C < 1) return MI3D_ERR_ARG;
    OneOp op;
    op.b.transpose((const __half*)in, (__half*)out, Z, R, C);
    return op.run(stream);
}

}  // extern "C"
