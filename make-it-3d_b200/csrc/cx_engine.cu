// cx_engine.cu -- the contextual loss of S-aiueo32/contextual_loss_pytorch as the refine stage builds it (C ABI: include/mi3d.h,
// section B6): ContextualLoss(band_width, loss_type='cosine', use_vgg=True, vgg_layer='relu5_4'), nerf/utils.py:455-457, 810, 882.
//
// VGG19 features[0:36] (conv1_1 .. relu5_4) run x and y as one batch of 2N images: conv1_1 (3 input channels) on the small direct
// conv, every other conv on the tile GEMM's CONV3_BLOCK mode with the ReLU in its epilogue, NHWC fp16 activations, fp32 accumulation.
// The loss itself is fp32 (cx_kernels.cuh).  The backward runs for x only: the sparse max/mean gradient, the row-normalisation and
// min backward, dXh = G Yh, the normalize backward, then the VGG input gradient (dgrad convs with the ReLU mask in the epilogue,
// max-pool gather backward) down to the image.  The feature gradient is scaled by a power of two before it goes to fp16 and the
// scale is undone at the image.  The weights are frozen.  No split-K and no atomics: bit-identical run to run and under graph replay.
#include "engine_plan.cuh"
#include "cx_kernels.cuh"

namespace cx {

using namespace plan;

// VGG19 features[0:36]: -1 = MaxPool2d(2, 2), else a 3x3 conv with that many output channels (+ ReLU)
static const int kLayers[] = {64, 64, -1, 128, 128, -1, 256, 256, 256, 256, -1, 512, 512, 512, 512, -1, 512, 512, 512, 512};

struct Layer {
    int pool = 0; T4 in, out; std::string w;     // conv: weight name; in = its (post-ReLU) input, out = its post-ReLU output
};

struct Engine : Builder {
    mi3d_cx_cfg cfg;
    explicit Engine(const mi3d_cx_cfg& c) : cfg(c) {}
    std::vector<Layer> layers;
    T4 img4, feat;
    int P = 0, C5 = 0;
    float *ymu = nullptr, *xh = nullptr, *nrm = nullptr, *S = nullptr, *cxm = nullptr, *rmin = nullptr, *cmax = nullptr, *mstat = nullptr, *loss = nullptr;
    int *rarg = nullptr, *carg = nullptr;
    float *dloss = nullptr, *G = nullptr, *dxh = nullptr, *rowmax = nullptr, *gscale = nullptr, *g4 = nullptr;
    T4 dfeat;
    float* bw_dev = nullptr;                 // band width of the current call (device scalar, so the lists stay static)
    std::vector<Op> fwd, bwd;
    bool tape_valid = false;

    // torchvision's features index of each conv -> the package's VGG19 slice (slice1: 0..3, slice2: 4..8, slice3: 9..17, slice4: 18..26, slice5: 27..35)
    static std::string conv_name(int idx) {
        const int slice = idx < 4 ? 1 : idx < 9 ? 2 : idx < 18 ? 3 : idx < 27 ? 4 : 5;
        return "vgg_model.slice" + std::to_string(slice) + "." + std::to_string(idx);
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; params.clear(); pindex.clear(); named.clear(); layers.clear(); fwd.clear(); bwd.clear();
        splitk_elems = 0;
        const int N = cfg.N, B = 2 * N;
        img4 = act(B, cfg.H, cfg.W, 4);
        // ---- forward: VGG19 up to relu5_4 on [x; y] ----
        cur = &fwd;
        T4 x = img4; int idx = 0, cin = 3;
        for (int li = 0; li < (int)(sizeof(kLayers) / sizeof(int)); li++) {
            Layer L;
            if (kLayers[li] < 0) {
                L.pool = 1; L.in = x; L.out = act(B, x.h / 2, x.w / 2, x.c);
                const T4 a = L.in, o = L.out;
                push([=](cudaStream_t st) {
                    cxk::k_maxpool2<<<blocks_for(o.numel() / 8), 256, 0, st>>>(a.p, o.p, a.n, a.h, a.w, a.c);
                    return (int)cudaGetLastError();
                });
                idx += 1;
            } else {
                const int cout = kLayers[li];
                L.w = conv_name(idx); L.in = x; L.out = act(B, x.h, x.w, cout);
                const float* bias = pf(L.w + ".bias", {cout});
                if (idx == 0) {
                    const float* w = (const float*)param(L.w + ".weight", {cout, cin, 3, 3}, PK_CX_CONV_IN).dst;
                    param(L.w + ".weight#dgrad", {4, cout, 3, 3}, PK_CX_CONV_IN_DGRAD);
                    const T4 o = L.out;
                    conv_small_cin(L.in, w, bias, o);
                    push([=](cudaStream_t st) {
                        cxk::k_relu<<<blocks_for(o.numel() / 8), 256, 0, st>>>(o.p, o.numel() / 8);
                        return (int)cudaGetLastError();
                    });
                } else {
                    const __half* w = (const __half*)param(L.w + ".weight", {cout, cin, 3, 3}, PK_CONV3_BOTH).dst;
                    conv3_block(L.in, w, cout, L.out, bias, tc::EPI_RELU);
                }
                idx += 2; cin = cout;
            }
            layers.push_back(L);
            x = L.out;
        }
        feat = x; C5 = x.c; P = x.h * x.w;
        tap("relu5_4", feat.p, feat.numel() * 2);
        // ---- contextual loss (fp32) ----
        ymu = alloc32(C5); xh = alloc32((size_t)B * P * C5); nrm = alloc32((size_t)B * P);
        S = alloc32((size_t)N * P * P); cxm = alloc32((size_t)N * P * P);
        rmin = alloc32((size_t)N * P); rarg = (int*)alloc((size_t)N * P * 4); cmax = alloc32((size_t)N * P); carg = (int*)alloc((size_t)N * P * 4);
        mstat = alloc32(N); loss = alloc32(1); bw_dev = alloc32(1);
        {
            const __half* F = feat.p; float *ym = ymu, *xhp = xh, *nr = nrm, *Sp = S, *cp = cxm, *rm = rmin, *cm = cmax, *ms = mstat, *lo = loss, *bwp = bw_dev;
            int *ra = rarg, *ca = carg; const int Pp = P, C = C5;
            push([=](cudaStream_t st) {
                cxk::k_ymu<<<C / 32, dim3(32, 8), 0, st>>>(F, N, Pp, C, ym);
                cxk::k_normalize<<<(B * Pp + 7) / 8, 256, 0, st>>>(F, ym, B * Pp, C, xhp, nr);
                // S[n] = Xh[n] Yh[n]^T
                cxk::k_sgemm<<<dim3((Pp + 63) / 64, (Pp + 63) / 64, N), 256, 0, st>>>(xhp, C, (long long)Pp * C, xhp + (size_t)N * Pp * C, C,
                                                                                   (long long)Pp * C, 1, Sp, Pp, (long long)Pp * Pp, Pp, Pp, C);
                return (int)cudaGetLastError();
            });
            push([=](cudaStream_t st) {
                cxk::k_cx_rows<<<N * Pp, 256, 0, st>>>(Sp, Pp, bwp, cp, rm, ra);
                cxk::k_cx_cols<<<dim3((Pp + 127) / 128, N), 128, 0, st>>>(cp, Pp, cm, ca);
                cxk::k_cx_loss<<<1, 256, 0, st>>>(cm, N, Pp, ms, lo);
                return (int)cudaGetLastError();
            });
        }
        // ---- backward, x images only ----
        cur = &bwd;
        dloss = alloc32(1); G = alloc32((size_t)N * P * P); dxh = alloc32((size_t)N * P * C5); rowmax = alloc32((size_t)N * P); gscale = alloc32(1);
        dfeat = act(N, feat.h, feat.w, C5);
        {
            const __half* F = feat.p; float *Sp = S, *cp = cxm, *rm = rmin, *ms = mstat, *dl = dloss, *Gp = G, *dx = dxh, *xhp = xh, *nr = nrm, *rmx = rowmax,
                  *gs = gscale, *bwp = bw_dev; int *ra = rarg, *ca = carg; const int Pp = P, C = C5; __half* df = dfeat.p;
            push([=](cudaStream_t st) {
                cxk::k_cx_rows_bwd<<<N * Pp, 256, 0, st>>>(Sp, cp, rm, ra, ca, ms, dl, N, Pp, bwp, Gp);
                // dXh[n] = G[n] Yh[n]
                cxk::k_sgemm<<<dim3((C + 63) / 64, (Pp + 63) / 64, N), 256, 0, st>>>(Gp, Pp, (long long)Pp * Pp, xhp + (size_t)N * Pp * C, C,
                                                                                  (long long)Pp * C, 0, dx, C, (long long)Pp * C, Pp, C, Pp);
                cxk::k_normalize_bwd<<<(N * Pp + 7) / 8, 256, 0, st>>>(dx, xhp, nr, F, N * Pp, C, rmx);
                cxk::k_grad_scale<<<1, 256, 0, st>>>(rmx, N * Pp, gs);
                cxk::k_scale_to_f16<<<blocks_for((size_t)N * Pp * C), 256, 0, st>>>(dx, gs, df, (size_t)N * Pp * C);
                return (int)cudaGetLastError();
            });
        }
        T4 dy = dfeat;               // gradient w.r.t. the current layer's pre-ReLU output (masked already), or a pool's output
        for (int li = (int)layers.size() - 1; li >= 0; li--) {
            const Layer& L = layers[li];
            const T4 in{L.in.p, N, L.in.h, L.in.w, L.in.c};          // the first N images of the batch are the x images
            if (L.pool) {
                T4 dx = act(N, in.h, in.w, in.c);
                const T4 d = dy;
                push([=](cudaStream_t st) {
                    cxk::k_maxpool2_bwd<<<blocks_for(dx.numel() / 8), 256, 0, st>>>(d.p, in.p, dx.p, N, in.h, in.w, in.c);
                    return (int)cudaGetLastError();
                });
                dy = dx;
            } else if (li > 0) {
                // dgrad; the conv's input is a pool output (mask applied by the pool backward) or a ReLU output (mask in the epilogue)
                T4 dx = act(N, in.h, in.w, in.c);
                const bool relu_in = !layers[li - 1].pool;
                conv3_block(dy, (const __half*)params[pindex[L.w + ".weight"]].dst2, in.c, dx, nullptr,
                            relu_in ? tc::EPI_RELU_BWD : tc::EPI_PLAIN, relu_in ? in.p : nullptr);
                dy = dx;
            } else {
                g4 = alloc32((size_t)N * cfg.H * cfg.W * 4);
                const __half* w = (const __half*)params[pindex[L.w + ".weight#dgrad"]].dst;
                conv_small_cout(dy, w, nullptr, g4, 4);
            }
        }
        cur = nullptr;
        return err;
    }

    int load_param(const Param& P, const float* src, const float* partner, cudaStream_t st) override {
        switch (P.kind) {
            case PK_CX_CONV_IN: {
                // conv1_1: the fp32 forward weights and, in the same pass, the flipped fp16 copy of its '#dgrad' entry
                const Param& D = params[pindex[P.name + "#dgrad"]];
                cxk::k_conv1_w<<<1, 256, 0, st>>>(src, (float*)P.dst, (__half*)D.dst, P.shape[0]);
                return (int)cudaGetLastError();
            }
            case PK_CX_CONV_IN_DGRAD: return MI3D_OK;      // written with its base tensor
            default: return Builder::load_param(P, src, partner, st);
        }
    }
};

bool valid_cfg(const mi3d_cx_cfg& c) { return c.N >= 1 && c.N <= 16 && c.H >= 16 && c.W >= 16 && c.H <= 4096 && c.W <= 4096; }

}  // namespace cx

extern "C" {

size_t mi3d_cx_workspace_bytes(const mi3d_cx_cfg* cfg) {
    return cfg && cx::valid_cfg(*cfg) ? plan::workspace_bytes<cx::Engine>(*cfg) : 0;
}

mi3d_engine_t mi3d_cx_create(const mi3d_cx_cfg* cfg, void* workspace, size_t workspace_bytes) {
    return cfg && cx::valid_cfg(*cfg) ? plan::create<cx::Engine>(workspace, workspace_bytes, *cfg) : nullptr;
}

int mi3d_cx_forward(mi3d_engine_t h, const float* x, const float* y, float band_width, int need_grad, float* loss, mi3d_stream_t stream) {
    cx::Engine* ep = plan::engine_of<cx::Engine>(h);
    if (!ep || !x || !y || !loss || !(band_width > 0.f)) return MI3D_ERR_ARG;
    cx::Engine& e = *ep; const mi3d_cx_cfg& c = e.cfg;
    cudaStream_t st = (cudaStream_t)stream;
    e.tape_valid = false;
    cxk::k_prep<<<plan::Builder::blocks_for((size_t)2 * c.N * c.H * c.W), 256, 0, st>>>(x, y, c.N, c.H, c.W, e.img4.p);
    MI3D_CHECK(cudaGetLastError());
    cxk::k_set<<<1, 1, 0, st>>>(e.bw_dev, band_width);
    int r = e.run(e.fwd, st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(loss, e.loss, sizeof(float), cudaMemcpyDeviceToDevice, st));
    e.tape_valid = need_grad != 0;
    return MI3D_OK;
}

int mi3d_cx_backward(mi3d_engine_t h, const float* dloss, float* dx, mi3d_stream_t stream) {
    cx::Engine* ep = plan::engine_of<cx::Engine>(h);
    if (!ep || !dloss || !dx) return MI3D_ERR_ARG;
    cx::Engine& e = *ep; const mi3d_cx_cfg& c = e.cfg;
    if (!e.tape_valid) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemcpyAsync(e.dloss, dloss, sizeof(float), cudaMemcpyDeviceToDevice, st));
    int r = e.run(e.bwd, st); if (r) return r;
    cxk::k_img_grad<<<plan::Builder::blocks_for((size_t)c.N * 3 * c.H * c.W), 256, 0, st>>>(e.g4, e.gscale, c.N, c.H, c.W, dx);
    return (int)cudaGetLastError();
}

}  // extern "C"
