// engine_plan.cuh -- the op-builder layer shared by the planned engines (sd, sd_text, clip, cx, unet, dpt and blip2_engine.cu).
//
// An engine is built twice: a dry run sizes the caller's workspace, the real run carves parameters and activations out of it
// (bump allocation, nothing is ever freed or reused) and records one closure per launch into static launch lists.  What lives
// here: the parameter registry and its weight loading, the workspace carving, the op builders over the tile GEMM / fused
// attention / memory-bound kernels, the replay of a list as a CUDA graph, and the create / size steps every engine's C entry
// points share (the generic mi3d_engine_* functions are in engine.cu).
#pragma once
#include <functional>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mi3d.h"
#include "sd_kernels.cuh"
#include "tc_host.cuh"
#include "attn.cuh"

// The opaque handle of include/mi3d.h: every planned engine is one (plan::Builder derives from it).
struct mi3d_engine { virtual ~mi3d_engine() {} };

namespace plan {

using Op = std::function<int(cudaStream_t)>;

// How a parameter is stored in the workspace; one kind is one layout in every engine.  Builder::load_param writes the kinds all
// engines share from the fp32 source tensor, an engine's override the kinds only it uses.
enum PKind { PK_F32 = 0, PK_LINEAR, PK_LINEAR_T, PK_LINEAR_BOTH, PK_CONV3, PK_CONV3_BOTH, PK_CONV1, PK_CONV1_BOTH,
             PK_CONV3_S2_BOTH,                                          // sd_engine.cu: strided 3x3 conv, dst2 = [9*I][O] (im2col dgrad)
             PK_GEGLU_W, PK_GEGLU_B, PK_CONV_F32_OHWI, PK_CONV_SMALL_COUT, PK_CONV_SMALL_COUT_BOTH,   // sd_engine.cu
             PK_CX_CONV_IN, PK_CX_CONV_IN_DGRAD,                        // cx_engine.cu: VGG conv1_1, fp32 forward and flipped fp16 copy
             PK_CONV_WS };   // weight-standardised conv (dpt_engine.cu): OIHW fp32 -> standardised [O][kh][kw][I] fp16

struct Param {
    std::string name; std::vector<int> shape; size_t numel = 0; PKind kind = PK_F32;
    void* dst = nullptr;      // primary storage
    void* dst2 = nullptr;     // secondary (transposed / flipped copy for the input-gradient pass)
    std::string partner;      // GEGLU: weight <-> bias handled together
};

struct T4 {  // NHWC fp16 activation
    __half* p = nullptr; int n = 0, h = 0, w = 0, c = 0;
    size_t numel() const { return (size_t)n * h * w * c; }
    long long rows() const { return (long long)n * h * w; }
};

struct Builder : mi3d_engine {
    uint8_t* base = nullptr; size_t cap = 0, off = 0; bool dry = true; int err = 0;
    int num_sms = 132;
    std::vector<Param> params; std::map<std::string, int> pindex;
    std::vector<Op>* cur = nullptr;
    std::map<std::string, std::pair<void*, size_t>> named;   // debug taps: name -> (ptr, bytes)
    float* splitk_ws = nullptr; size_t splitk_elems = 0;      // fp32 scratch shared by all split-K GEMMs (they run one at a time); 0 = no split-K
    // optional live timing of the tensor-core tile kernel (bench.py roofline leg): CUDA events around every k_tc_gemm launch
    bool profile = false; std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events; size_t prof_used = 0;
    struct ProfShape { int M, N, K, bn, splits, conv, batch, epi; }; std::vector<ProfShape> prof_shapes;
    int do_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st) {
        if (p.splits > 1) return tc::launch_splitk(ma, mb, p, bn, p.splits, splitk_ws, st);
        return tc::launch(ma, mb, p, bn, batch, st);
    }
    int timed_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st) {
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

    void* alloc(size_t bytes) {
        off = (off + 1023) & ~(size_t)1023;
        void* p = dry ? (void*)(uintptr_t)(0x10000 + off) : (void*)(base + off);
        off += bytes;
        if (!dry && off > cap) err = MI3D_ERR_ARG;
        return p;
    }
    __half* alloc16(size_t n) { return (__half*)alloc(n * 2); }
    float* alloc32(size_t n) { return (float*)alloc(n * 4); }
    void push(Op op) { if (!dry && cur) cur->push_back(std::move(op)); }
    void tap(const std::string& name, void* p, size_t bytes) { if (!dry) named[name] = {p, bytes}; }

    Param& param(const std::string& name, std::vector<int> shape, PKind kind) {
        auto it = pindex.find(name);
        if (it != pindex.end()) return params[it->second];
        Param P; P.name = name; P.shape = shape; P.kind = kind; P.numel = 1;
        for (int s : shape) P.numel *= (size_t)s;
        switch (kind) {
            case PK_F32: case PK_GEGLU_B: P.dst = alloc(P.numel * 4); break;
            case PK_CONV_F32_OHWI: case PK_CX_CONV_IN:                                                         // input channels padded to <= 8
                P.dst = alloc((size_t)std::max(shape[0], shape[1]) * 9 * 8 * 4); break;
            case PK_LINEAR: case PK_CONV3: case PK_CONV1: case PK_GEGLU_W: case PK_LINEAR_T: case PK_CONV_SMALL_COUT: case PK_CX_CONV_IN_DGRAD:
            case PK_CONV_WS:
                P.dst = alloc(P.numel * 2); break;
            case PK_LINEAR_BOTH: case PK_CONV3_BOTH: case PK_CONV1_BOTH: case PK_CONV3_S2_BOTH: case PK_CONV_SMALL_COUT_BOTH:
                P.dst = alloc(P.numel * 2); P.dst2 = alloc(P.numel * 2); break;
        }
        pindex[name] = (int)params.size();
        params.push_back(P);
        return params.back();
    }
    const float* pf(const std::string& name, std::vector<int> shape) { return (const float*)param(name, shape, PK_F32).dst; }
    // a parameter stored in memory the engine carved itself (a row slice of a packed weight): registered, not allocated
    Param& param_view(const std::string& name, std::vector<int> shape, PKind kind, void* dst) {
        auto it = pindex.find(name);
        if (it != pindex.end()) return params[it->second];
        Param P; P.name = name; P.shape = shape; P.kind = kind; P.numel = 1; P.dst = dst;
        for (int s : shape) P.numel *= (size_t)s;
        pindex[name] = (int)params.size();
        params.push_back(P);
        return params.back();
    }

    // Writes P from src, an fp32 device tensor in torch's layout (for a '#' entry: its base tensor).  partner: the second tensor of a
    // pair written together (SD's GEGLU weight and bias).  The base handles the kinds every engine lays out alike; an engine overrides
    // it for its own kinds and passes the rest on.
    virtual int load_param(const Param& P, const float* src, const float* partner, cudaStream_t st) {
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
            case PK_CONV3: sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.shape[0], P.shape[1], 0); break;
            case PK_CONV3_BOTH:                                                     // dst2: the flipped, transposed dgrad weights
                sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst, P.shape[0], P.shape[1], 0);
                sdk::k_conv_w<<<nb, 256, 0, st>>>(src, (__half*)P.dst2, P.shape[0], P.shape[1], 1); break;
            default: return MI3D_ERR_ARG;
        }
        return (int)cudaGetLastError();
    }

    // ------------------------------------------------------------------------------------------------------
    // op builders
    // ------------------------------------------------------------------------------------------------------
    struct Mat { const __half* p; long long ld; long long rows; int K; int z1 = 1; long long sz1 = 0; int z2 = 1; long long sz2 = 0; };
    struct Out { __half* p16 = nullptr; float* p32 = nullptr; long long ldc = 0; int z1 = 1; long long s_lo = 0, s_hi = 0; };
    struct Epi { const float* bias = nullptr; const float* row_bias = nullptr; int rows_per_group = 1; const __half* residual = nullptr;
                 long long ld_res = 0; int mode = tc::EPI_PLAIN; float alpha = 1.f; __half* aux = nullptr; };

    void gemm(const Mat& a, const Mat& b, int N, const Out& o, const Epi& e, int batch = 1, bool b_batched = false) {
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

    // y[M,N] = x[M,K] W[N,K]^T (+bias) (+residual)
    void linear(const __half* x, long long M, int K, const __half* W, int N, __half* y, const float* bias = nullptr,
                const __half* residual = nullptr, int mode = tc::EPI_PLAIN, long long ldc = -1) {
        Mat a{x, K, M, K}; Mat b{W, K, N, K};
        Out o; o.p16 = y; o.ldc = ldc >= 0 ? ldc : (mode == tc::EPI_GEGLU ? N / 2 : (mode == tc::EPI_TRANSPOSED ? M : N));
        Epi e; e.bias = bias; e.residual = residual; e.ld_res = N; e.mode = mode;
        gemm(a, b, N, o, e);
    }

    T4 act(int n, int h, int w, int c) { T4 t; t.n = n; t.h = h; t.w = w; t.c = c; t.p = alloc16(t.numel()); return t; }

    // 3x3 stride-1 pad-1 conv via implicit GEMM; w [Cout][3][3][Cin] fp16
    void conv3(const T4& x, const __half* w, int Cout, const T4& y, const float* bias, const float* row_bias = nullptr,
               const __half* residual = nullptr) {
        if (dry) return;
        const long long M = x.rows();
        int bw = x.w < 128 ? x.w : 128, bh = 128 / bw; if (bh > x.h) bh = x.h; const int bn_img = 128 / (bw * bh);
        if (M % 128 || x.c % 64 || bw * bh * bn_img != 128 || x.w % bw || x.h % bh || x.n % bn_img) { err = MI3D_ERR_ARG; return; }
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

    // dgrad of a stride-1 3x3 conv: dx = conv3(dy, W_flipped^T)  (+ residual accumulation)
    void conv3_dgrad(const T4& dy, const std::string& wname, int cin, const T4& dx, const __half* add = nullptr) {
        Param& w = params[pindex[wname]];
        conv3(dy, (const __half*)w.dst2, cin, dx, nullptr, nullptr, add);
    }

    // The same conv for any H x W (VGG's levels): each 128-row tile is a bw x bh block of one image (the shape that wastes the
    // fewest rows over the image edge), overhanging tiles load zeros and store only in-image pixels.  mode: EPI_PLAIN (optionally
    // + residual, same layout as y), EPI_RELU, or EPI_RELU_BWD with aux = the mask source.  No split-K (its fp32 RED order varies run to run).
    void conv3_block(const T4& x, const __half* w, int Cout, const T4& y, const float* bias, int mode, const __half* aux = nullptr,
                     const __half* residual = nullptr) {
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
        p.bias = bias; p.rows_per_group = 1; p.epi_mode = mode; p.alpha = 1.f; p.m_valid = (int)x.rows(); p.splits = 1; p.aux = const_cast<__half*>(aux);
        p.residual = residual; p.ld_res = Cout;
        push([this, ma, mb, p, bn](cudaStream_t st) { return timed_launch(ma, mb, p, bn, 1, st); });
    }

    void layernorm(const __half* x, long long rows, int C, const std::string& pname, __half* y) {
        const float* ga = pf(pname + ".weight", {C}); const float* be = pf(pname + ".bias", {C});
        layernorm(x, rows, C, ga, be, y);
    }
    void layernorm(const __half* x, long long rows, int C, const float* ga, const float* be, __half* y, float eps = 1e-5f) {
        push([=](cudaStream_t st) {
            sdk::k_layernorm<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, y, ga, be, (int)rows, C, eps);
            return (int)cudaGetLastError();
        });
    }
    void softmax(__half* s, size_t rows, int cols, int valid, float scale) {
        push([=](cudaStream_t st) {
            sdk::k_softmax<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(s, rows, cols, valid, scale);
            return (int)cudaGetLastError();
        });
    }
    void transpose(const __half* in, __half* out, int Z, int R, int C) {
        push([=](cudaStream_t st) {
            sdk::k_transpose<<<dim3((C + 31) / 32, (R + 31) / 32, Z), dim3(32, 8), 0, st>>>(in, out, R, C);
            return (int)cudaGetLastError();
        });
    }
    // persistent grids of the small direct convolutions: as many CTAs per SM as their weight staging area allows
    int small_cin_grid(size_t outputs, size_t smem) const { const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (200 * 1024) / std::max<size_t>(smem, 1))); return (int)std::min<size_t>((outputs / 8 + 255) / 256, (size_t)num_sms * per_sm); }
    int small_cout_grid(size_t pixels, int cin) const { const int ppw = cin <= 128 ? 2 : 1; return (int)std::min<size_t>((pixels / ppw + 7) / 8 + 1, (size_t)num_sms * 8); }
    static int blocks_for(size_t n) { return (int)std::min<size_t>((n + 255) / 256, 132 * 16); }

    // multi-head attention core on token matrices (attn.cuh).  q: [B*T, ldq] (head h at column h*d), k / v likewise
    // [B*Tk, ld]; only the first Tk_valid keys of each batch take part.  Writes o [B*T, C].  d: 40, 64, 80 or 160.
    void attention_core(const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv, int B, int T, int Tk,
                        int Tk_valid, int heads, int d, __half* o, int C) {
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

    int run_eager(std::vector<Op>& ops, cudaStream_t st) {
        for (auto& op : ops) { int r = op(st); if (r) return r; }
        return MI3D_OK;
    }
    // The launch lists are static (fixed pointers, shapes and order; every input lives in a device buffer), so a list replays as ONE
    // CUDA graph from its third call on (the lists lose their CPU launch cost and inter-kernel gaps).  Enabled per engine
    // (mi3d_engine_set_graph_replay); needs a capturable stream (torch's legacy default stream is not: the
    // Python engines run on their own stream, event-ordered against the caller's).  A list whose capture fails falls back to plain
    // launches for good.
    struct ListGraph { cudaGraphExec_t exec = nullptr; int calls = 0; bool failed = false; };
    std::map<std::vector<Op>*, ListGraph> graphs;
    bool use_graph = false;
    int run(std::vector<Op>& ops, cudaStream_t st) {
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
    int graph_replays() const {
        int n = 0;
        for (auto& kv : graphs) if (kv.second.exec) n++;
        return n;
    }
    ~Builder() override { for (auto& kv : graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec); }
};

// The create / size steps of every engine's C entry points.  E is constructed from the configuration arguments and has build(dry).
// Workspace size: the dry build's carve plus 1 MiB of slack; 0 when the dry build fails.
template <class E, class... Cfg> size_t workspace_bytes(const Cfg&... cfg) {
    E e(cfg...);
    return e.build(true) ? 0 : e.off + (1 << 20);
}
// The engine planned inside the caller's workspace (the real build, for this device's SM count); nullptr on failure.
template <class E, class... Cfg> E* create(void* workspace, size_t bytes, const Cfg&... cfg) {
    if (!workspace) return nullptr;
    E* e = new E(cfg...);
    e->base = (uint8_t*)workspace; e->cap = bytes;
    int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (e->build(false) != 0) { delete e; return nullptr; }
    return e;
}
// The engine of type E behind a handle; nullptr for NULL or another engine's handle (its entry points then return MI3D_ERR_ARG).
template <class E> E* engine_of(mi3d_engine_t h) { return dynamic_cast<E*>(h); }

}  // namespace plan
