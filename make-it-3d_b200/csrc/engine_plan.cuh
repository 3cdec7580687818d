// engine_plan.cuh -- the op-builder layer shared by the planned engines (sd, sd_text, clip, cx, unet, dpt and blip2_engine.cu).
//
// An engine is built twice: a dry run sizes the caller's workspace, the real run carves parameters and activations out of it
// (bump allocation, nothing is ever freed or reused) and records one closure per launch into static launch lists.  What lives
// here: the parameter registry and its weight loading, the workspace carving, the op builders over the tile GEMM / fused
// attention / memory-bound kernels, the replay of a list as a CUDA graph, and the create / size steps every engine's C entry
// points share (the generic mi3d_engine_* functions are in engine.cu).  This header is host code only: the op builders and the
// kernels they launch are compiled once, in plan.cu.
#pragma once
#include <functional>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mi3d.h"
#include "tc_host.cuh"

// The opaque handle of include/mi3d.h: every planned engine is one (plan::Builder derives from it).
struct mi3d_engine { virtual ~mi3d_engine() {} };

namespace plan {

using Op = std::function<int(cudaStream_t)>;

// How a parameter is stored in the workspace; one kind is one layout in every engine.  Builder::load_param writes the kinds all
// engines share from the fp32 source tensor, an engine's override the kinds only it uses.
enum PKind { PK_F32 = 0, PK_LINEAR, PK_LINEAR_T, PK_LINEAR_BOTH, PK_CONV3, PK_CONV3_BOTH, PK_CONV1, PK_CONV1_BOTH,
             PK_CONV3_S2_BOTH,                                          // Builder::conv3_s2 weight, dst2 = [9*I][O] (im2col dgrad)
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
    int do_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st);
    int timed_launch(const CUtensorMap& ma, const CUtensorMap& mb, const tc::GemmParams& p, int bn, int batch, cudaStream_t st);

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
    virtual int load_param(const Param& P, const float* src, const float* partner, cudaStream_t st);

    // ------------------------------------------------------------------------------------------------------
    // op builders
    // ------------------------------------------------------------------------------------------------------
    struct Mat { const __half* p; long long ld; long long rows; int K; int z1 = 1; long long sz1 = 0; int z2 = 1; long long sz2 = 0; };
    struct Out { __half* p16 = nullptr; float* p32 = nullptr; long long ldc = 0; int z1 = 1; long long s_lo = 0, s_hi = 0; };
    struct Epi { const float* bias = nullptr; const float* row_bias = nullptr; int rows_per_group = 1; const __half* residual = nullptr;
                 long long ld_res = 0; int mode = tc::EPI_PLAIN; float alpha = 1.f; __half* aux = nullptr; };

    void gemm(const Mat& a, const Mat& b, int N, const Out& o, const Epi& e, int batch = 1, bool b_batched = false);

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
               const __half* residual = nullptr);

    // dgrad of a stride-1 3x3 conv: dx = conv3(dy, W_flipped^T)  (+ residual accumulation)
    void conv3_dgrad(const T4& dy, const std::string& wname, int cin, const T4& dx, const __half* add = nullptr) {
        Param& w = params[pindex[wname]];
        conv3(dy, (const __half*)w.dst2, cin, dx, nullptr, nullptr, add);
    }

    // The same conv for any H x W (VGG's levels): each 128-row tile is a bw x bh block of one image (the shape that wastes the
    // fewest rows over the image edge), overhanging tiles load zeros and store only in-image pixels.  mode: EPI_PLAIN (optionally
    // + residual, same layout as y), EPI_RELU, or EPI_RELU_BWD with aux = the mask source.  No split-K (its fp32 RED order varies run to run).
    void conv3_block(const T4& x, const __half* w, int Cout, const T4& y, const float* bias, int mode, const __half* aux = nullptr,
                     const __half* residual = nullptr, const float* row_bias = nullptr);
    // 3x3 stride-2 conv as im2col + linear: w [Cout][3][3][Cin] fp16, y [x.n][Ho][Wo][Cout]; pad_lo = 1 (symmetric padding 1) or 0
    // (padding (0, 1, 0, 1)).  Returns the im2col matrix [x.n * Ho * Wo][9 * Cin] (the input of a weight-gradient or dgrad pass).
    __half* conv3_s2(const T4& x, const __half* w, const T4& y, const float* bias, int pad_lo);
    // Direct 3x3 stride-1 pad-1 convs for channel counts below the tile GEMM's 64-wide K blocks.  conv_small_cin: x fp16 with 4 or 8
    // channels, w fp32 [y.c][3][3][x.c], y fp16 (y.c % 8 == 0).  conv_small_cout: x fp16 (x.c % 8 == 0), w fp16 [cout][3][3][x.c]
    // with cout 4 or 8, out fp32 [x.rows()][cout].
    void conv_small_cin(const T4& x, const float* w, const float* bias, const T4& y);
    void conv_small_cout(const T4& x, const __half* w, const float* bias, float* out, int cout);

    void layernorm(const __half* x, long long rows, int C, const std::string& pname, __half* y) {
        const float* ga = pf(pname + ".weight", {C}); const float* be = pf(pname + ".bias", {C});
        layernorm(x, rows, C, ga, be, y);
    }
    void layernorm(const __half* x, long long rows, int C, const float* ga, const float* be, __half* y, float eps = 1e-5f);
    // dx = LayerNorm input gradient of dy (+ add), statistics recomputed from x as layernorm() computes them
    void layernorm_bwd(const __half* x, const __half* dy, const float* gamma, const __half* add, __half* dx, long long rows, int C,
                       float eps = 1e-5f);
    // row softmax in place: s = softmax(scale * s[:, :valid]), columns >= valid written as 0.  causal_tq > 0: row r (query
    // r % causal_tq) also drops the keys after its query.
    void softmax(__half* s, size_t rows, int cols, int valid, float scale, int causal_tq = 0);
    // softmax backward in place on dp: ds = scale * p * (dp - sum(dp * p))
    void softmax_bwd(const __half* p, __half* dp, size_t rows, int cols, float scale);
    // batched transpose fp16: in [Z][R][C] -> out [Z][C][R]
    void transpose(const __half* in, __half* out, int Z, int R, int C);
    void f32_to_f16(const float* src, __half* dst, size_t n);
    // x[b * Tpad + t] = tok_emb[tokens[b, t]] + pos[t] for t < L, rows L .. Tpad-1 zero; ids clamped into [0, vocab)
    void text_embed(const long long* tokens, const float* tok_emb, const float* pos, __half* x, int B, int L, int Tpad, int C, int vocab);
    static int blocks_for(size_t n) { return (int)std::min<size_t>((n + 255) / 256, 132 * 16); }

    // multi-head attention core on token matrices (attn.cuh).  q: [B*T, ldq] (head h at column h*d), k / v likewise
    // [B*Tk, ld]; only the first Tk_valid keys of each batch take part.  Writes o [B*T, C].  d: 40, 64, 80 or 160.
    void attention_core(const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv, int B, int T, int Tk,
                        int Tk_valid, int heads, int d, __half* o, int C);

    int run_eager(std::vector<Op>& ops, cudaStream_t st);
    // The launch lists are static (fixed pointers, shapes and order; every input lives in a device buffer), so a list replays as ONE
    // CUDA graph from its third call on (the lists lose their CPU launch cost and inter-kernel gaps).  Enabled per engine
    // (mi3d_engine_set_graph_replay); needs a capturable stream (torch's legacy default stream is not: the
    // Python engines run on their own stream, event-ordered against the caller's).  A list whose capture fails falls back to plain
    // launches for good.
    struct ListGraph { cudaGraphExec_t exec = nullptr; int calls = 0; bool failed = false; };
    std::map<std::vector<Op>*, ListGraph> graphs;
    bool use_graph = false;
    int run(std::vector<Op>& ops, cudaStream_t st);
    int graph_replays() const {
        int n = 0;
        for (auto& kv : graphs) if (kv.second.exec) n++;
        return n;
    }
    ~Builder() override;
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
