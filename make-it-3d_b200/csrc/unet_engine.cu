// unet_engine.cu -- the refine stage's gated U-Net (C ABI: include/mi3d.h, section B7): UNet(num_input_channels=19) of the
// reference's nerf/unet.py with its defaults (feature_scale 4, bilinear upsampling, sigmoid output, gated blocks), nerf/utils.py:808, 863.
//
//   start  G(19->16) on x0 -> in64                                  (H)
//   down1  avgpool 2x2 -> G(16->13) ; cat x1 -> d1 (32)              (H/2)
//   down2  avgpool 2x2 -> G(32->45) ; cat x2 -> d2 (64)              (H/4)
//   up2    bilinear x2 -> conv3 64->32 ; cat d1 -> G(64->32, no BN)  (H/2)
//   up1    bilinear x2 -> conv3 32->16 ; cat in64 -> G(32->16, no BN) (H)
//   final  conv1x1 16->3 -> sigmoid
// G(cin->c) = BN(ELU(conv_f x) * sigmoid(conv_m x)); conv_f and conv_m run as one conv with 2c outputs (their weights sit side by
// side in the workspace).  Activations are NCHW fp32; the concatenations cost nothing: d1 and in64 live inside the buffers the up
// blocks read (cat2, cat1) and their producers write channel slices.  BatchNorm uses batch statistics in train mode (and the caller's
// running statistics are updated once per forward) or the running statistics in eval mode.  The backward gives the input gradients
// of x0, x1, x2 and every parameter's gradient.  Weight gradients are split over a fixed set of CTAs with fp32 partials and a
// fixed-order sum; there are no atomics, so every output is bit-identical run to run and under graph replay.
#include "engine_plan.cuh"
#include "unet_kernels.cuh"

namespace unet {

using namespace plan;

// an NCHW fp32 tensor view: channel c of image n at p + n * ns + c * H * W
struct V { float* p = nullptr; long long ns = 0; };

enum EKind { E_PARAM = 0, E_RMEAN = 1, E_RVAR = 2, E_COUNT = 3 };
struct Entry { std::string name; std::vector<int> shape; int kind = E_PARAM; float* slot = nullptr; float* grad = nullptr; size_t numel = 1; };

struct Gated {            // one gated block's storage
    int cin = 0, c = 0, bn = 0;
    float *w = nullptr, *b = nullptr, *dw = nullptr, *db = nullptr;      // [2c][cin][3][3], [2c] and their gradients
    float *wt = nullptr;                                                 // [cin][2c][3][3]: the input-gradient weights
    float *gamma = nullptr, *beta = nullptr, *dgamma = nullptr, *dbeta = nullptr, *rmean = nullptr, *rvar = nullptr;
    float *mean = nullptr, *var = nullptr, *rstd = nullptr, *sdy = nullptr, *sdyx = nullptr;
    float *fm = nullptr, *g = nullptr;                                   // [N][2c][HW] pre-activations, [N][c][HW] gate output
    int e_rmean = -1, e_rvar = -1, e_count = -1;                         // registry indices of the BatchNorm buffers
};
struct Conv { int cin = 0, cout = 0; float *w = nullptr, *b = nullptr, *dw = nullptr, *db = nullptr, *wt = nullptr; };

constexpr int kWgradCtas = 528;                 // CTAs per weight-gradient launch (4 per SM): the pixel split is a function of the shape only
constexpr int kMaxWgradElems = kWgradCtas * unk::WOB * unk::WCB * 9;   // S x Cout x Cin x 9 <= 528 x (32 x 16 x 9) per (o, c) block

struct Engine : Builder {
    mi3d_unet_shape cfg;
    std::vector<Entry> entries;
    Gated gs, gd1, gd2, gu2, gu1;
    Conv cu2, cu1, fin;
    int H[3], Wd[3]; size_t HW[3];
    float *x0 = nullptr, *cat1 = nullptr, *p1 = nullptr, *cat2 = nullptr, *p2 = nullptr, *d2 = nullptr, *u2 = nullptr, *u1 = nullptr, *y = nullptr;
    float *dout = nullptr, *dz = nullptr, *dg4 = nullptr, *dfm4 = nullptr, *dcat1 = nullptr, *du1 = nullptr, *dg3 = nullptr, *dfm3 = nullptr,
          *dcat2 = nullptr, *du2 = nullptr, *dd2 = nullptr, *dfm2 = nullptr, *dp2 = nullptr, *dfm1 = nullptr, *dp1 = nullptr, *dfm0 = nullptr, *dx0 = nullptr;
    float *wpart = nullptr, *bpart = nullptr, *fpart = nullptr; double* cpart = nullptr;
    std::vector<Op> fwd_train, fwd_eval, bwd_train, bwd_eval;
    int tape = 0;                                 // 0 none, 1 train-mode tape, 2 eval-mode tape

    static constexpr int kFinalCtas = 264;
    static constexpr int kChanChunks = 64;

    void add(const std::string& name, std::vector<int> shape, int kind, float* slot, float* grad) {
        Entry e; e.name = name; e.shape = shape; e.kind = kind; e.slot = slot; e.grad = grad;
        for (int s : shape) e.numel *= (size_t)s;
        entries.push_back(e);
    }

    void gated(Gated& G, const std::string& pre, int cin, int c, int bn, int lvl) {
        const int N = cfg.N;
        G.cin = cin; G.c = c; G.bn = bn;
        const size_t wn = (size_t)c * cin * 9;
        G.w = alloc32(2 * wn); G.b = alloc32(2 * c); G.dw = alloc32(2 * wn); G.db = alloc32(2 * c); G.wt = alloc32(2 * wn);
        add(pre + "conv_f.weight", {c, cin, 3, 3}, E_PARAM, G.w, G.dw);
        add(pre + "conv_f.bias", {c}, E_PARAM, G.b, G.db);
        add(pre + "conv_m.weight", {c, cin, 3, 3}, E_PARAM, G.w + wn, G.dw + wn);
        add(pre + "conv_m.bias", {c}, E_PARAM, G.b + c, G.db + c);
        if (bn) {
            G.gamma = alloc32(c); G.beta = alloc32(c); G.dgamma = alloc32(c); G.dbeta = alloc32(c); G.rmean = alloc32(c); G.rvar = alloc32(c);
            G.mean = alloc32(c); G.var = alloc32(c); G.rstd = alloc32(c); G.sdy = alloc32(c); G.sdyx = alloc32(c);
            add(pre + "norm.weight", {c}, E_PARAM, G.gamma, G.dgamma);
            add(pre + "norm.bias", {c}, E_PARAM, G.beta, G.dbeta);
            G.e_rmean = (int)entries.size(); G.e_rvar = G.e_rmean + 1; G.e_count = G.e_rmean + 2;
            add(pre + "norm.running_mean", {c}, E_RMEAN, G.rmean, nullptr);
            add(pre + "norm.running_var", {c}, E_RVAR, G.rvar, nullptr);
            add(pre + "norm.num_batches_tracked", {}, E_COUNT, nullptr, nullptr);
            G.g = alloc32((size_t)N * c * HW[lvl]);
        }
        G.fm = alloc32((size_t)N * 2 * c * HW[lvl]);
    }
    void conv(Conv& Cv, const std::string& name, int cin, int cout, int k) {
        Cv.cin = cin; Cv.cout = cout;
        const size_t wn = (size_t)cout * cin * k * k;
        Cv.w = alloc32(wn); Cv.b = alloc32(cout); Cv.dw = alloc32(wn); Cv.db = alloc32(cout); Cv.wt = alloc32(wn);
        if (k == 3) add(name + ".weight", {cout, cin, 3, 3}, E_PARAM, Cv.w, Cv.dw);
        else add(name + ".weight", {cout, cin, 1, 1}, E_PARAM, Cv.w, Cv.dw);
        add(name + ".bias", {cout}, E_PARAM, Cv.b, Cv.db);
    }

    // ---- op emitters ----
    void conv3(V in, int Cin, const float* w, const float* bias, V out, int Cout, int lvl) {
        const int h = H[lvl], wd = Wd[lvl], N = cfg.N;
        const dim3 grid(((wd + unk::CT - 1) / unk::CT) * ((h + unk::CT - 1) / unk::CT), (Cout + unk::COB - 1) / unk::COB, N);
        push([=](cudaStream_t st) {
            unk::k_conv3<<<grid, 256, 0, st>>>(in.p, in.ns, Cin, w, bias, out.p, out.ns, Cout, h, wd);
            return (int)cudaGetLastError();
        });
    }
    void flip(const float* w, int co, int ci, float* wt) {
        push([=](cudaStream_t st) {
            unk::k_flip_w<<<blocks_for((size_t)co * ci * 9), 256, 0, st>>>(w, co, ci, wt);
            return (int)cudaGetLastError();
        });
    }
    static int wgrad_chunks(int N, int h, int w, int Cin, int Cout) {
        const int tiles = N * ((w + unk::WTX - 1) / unk::WTX) * ((h + unk::WTY - 1) / unk::WTY);
        const int blocks = ((Cout + unk::WOB - 1) / unk::WOB) * ((Cin + unk::WCB - 1) / unk::WCB);
        return std::max(1, std::min(tiles, kWgradCtas / blocks));
    }
    void wgrad(V in, int Cin, V dy, int Cout, int lvl, float* dw, float* db) {
        const int h = H[lvl], wd = Wd[lvl], N = cfg.N;
        const int S = wgrad_chunks(N, h, wd, Cin, Cout);
        const dim3 grid(S, (Cout + unk::WOB - 1) / unk::WOB, (Cin + unk::WCB - 1) / unk::WCB);
        float *wp = wpart, *bp = bpart;
        const size_t E = (size_t)Cout * Cin * 9;
        if ((size_t)S * E > (size_t)kMaxWgradElems) { err = MI3D_ERR_ARG; return; }
        push([=](cudaStream_t st) {
            unk::k_conv3_wgrad<<<grid, 128, 0, st>>>(in.p, in.ns, Cin, dy.p, dy.ns, Cout, N, h, wd, wp, bp);
            unk::k_sum_chunks<<<blocks_for(E), 256, 0, st>>>(wp, S, E, dw);
            unk::k_sum_chunks<<<1, 256, 0, st>>>(bp, S, (size_t)Cout, db);
            return (int)cudaGetLastError();
        });
    }
    int chan_chunks(int lvl) const { return (int)std::max<size_t>(1, std::min<size_t>(kChanChunks, ((size_t)cfg.N * HW[lvl] + 4095) / 4096)); }

    // forward of a gated block: in (Cin channels) -> out view
    void gated_fwd(Gated& G, V in, V out, int lvl, bool train) {
        const int N = cfg.N, c = G.c; const size_t hw = HW[lvl];
        conv3(in, G.cin, G.w, G.b, V{G.fm, (long long)(2 * c * hw)}, 2 * c, lvl);
        const size_t n = (size_t)N * c * hw;
        if (!G.bn) {
            Gated g = G;
            push([=](cudaStream_t st) {
                unk::k_gate<<<blocks_for(n), 256, 0, st>>>(g.fm, c, N, hw, out.p, out.ns);
                return (int)cudaGetLastError();
            });
            return;
        }
        const int S = chan_chunks(lvl);
        Gated g = G; double* cp = cpart;
        push([=](cudaStream_t st) {
            unk::k_gate<<<blocks_for(n), 256, 0, st>>>(g.fm, c, N, hw, g.g, (long long)(c * hw));
            if (train) {
                unk::k_chan_partial<<<dim3(c, S), 256, 0, st>>>(g.g, (long long)(c * hw), nullptr, 0, nullptr, nullptr, N, hw, 0, cp);
                unk::k_bn_stats<<<1, 64, 0, st>>>(cp, c, S, (double)N * hw, 1e-5f, g.mean, g.var, g.rstd);
            } else {
                unk::k_bn_eval_stats<<<1, 64, 0, st>>>(g.rmean, g.rvar, c, 1e-5f, g.mean, g.rstd);
            }
            unk::k_bn_apply<<<blocks_for(n), 256, 0, st>>>(g.g, g.mean, g.rstd, g.gamma, g.beta, c, N, hw, out.p, out.ns);
            return (int)cudaGetLastError();
        });
    }
    // backward of a gated block: dy (gradient of its output view) -> d[f|m] (dfm) -> weight grads and, if din, the input gradient
    void gated_bwd(Gated& G, V in, V dy, float* dfm, V din, int lvl, bool train) {
        const int N = cfg.N, c = G.c; const size_t hw = HW[lvl], n = (size_t)N * c * hw;
        const int S = chan_chunks(lvl);
        Gated g = G; double* cp = cpart;
        const int bn = G.bn ? (train ? 1 : 2) : 0;
        push([=](cudaStream_t st) {
            if (bn) {
                unk::k_chan_partial<<<dim3(c, S), 256, 0, st>>>(g.g, (long long)(c * hw), dy.p, dy.ns, g.mean, g.rstd, N, hw, 1, cp);
                unk::k_bn_bwd_stats<<<1, 64, 0, st>>>(cp, c, S, g.dgamma, g.dbeta, g.sdy, g.sdyx);
            }
            unk::k_gate_bwd<<<blocks_for(n), 256, 0, st>>>(dy.p, dy.ns, g.fm, g.g, g.mean, g.rstd, g.gamma, g.sdy, g.sdyx, bn, c, N, hw, dfm);
            return (int)cudaGetLastError();
        });
        const V dv{dfm, (long long)(2 * c * hw)};
        wgrad(in, G.cin, dv, 2 * c, lvl, G.dw, G.db);
        if (din.p) conv3(dv, 2 * c, G.wt, nullptr, din, G.cin, lvl);
    }

    void emit_forward(bool train) {
        const int N = cfg.N;
        const long long s0 = 32 * (long long)HW[0], s1 = 64 * (long long)HW[1], s2 = 64 * (long long)HW[2];
        const V vx0{x0, 19 * (long long)HW[0]}, in64{cat1 + 16 * HW[0], s0}, d1{cat2 + 32 * HW[1], s1}, vd2{d2, s2};
        gated_fwd(gs, vx0, in64, 0, train);
        {
            const V a = in64; float* o = p1; const int h = H[0], w = Wd[0];
            push([=](cudaStream_t st) {
                unk::k_avgpool<<<blocks_for((size_t)N * 16 * HW[1]), 256, 0, st>>>(a.p, a.ns, 16, N, h, w, o, 16 * (long long)HW[1]);
                return (int)cudaGetLastError();
            });
        }
        gated_fwd(gd1, V{p1, 16 * (long long)HW[1]}, d1, 1, train);
        {
            const V a = d1; float* o = p2; const int h = H[1], w = Wd[1];
            push([=](cudaStream_t st) {
                unk::k_avgpool<<<blocks_for((size_t)N * 32 * HW[2]), 256, 0, st>>>(a.p, a.ns, 32, N, h, w, o, 32 * (long long)HW[2]);
                return (int)cudaGetLastError();
            });
        }
        gated_fwd(gd2, V{p2, 32 * (long long)HW[2]}, vd2, 2, train);
        {
            const V a = vd2; float* o = u2; const int h = H[2], w = Wd[2];
            push([=](cudaStream_t st) {
                unk::k_upsample2<<<blocks_for((size_t)N * 64 * HW[1]), 256, 0, st>>>(a.p, a.ns, 64, N, h, w, o, s1);
                return (int)cudaGetLastError();
            });
        }
        conv3(V{u2, s1}, 64, cu2.w, cu2.b, V{cat2, s1}, 32, 1);
        gated_fwd(gu2, V{cat2, s1}, V{g3, 32 * (long long)HW[1]}, 1, train);
        {
            const float* a = g3; float* o = u1; const int h = H[1], w = Wd[1];
            push([=](cudaStream_t st) {
                unk::k_upsample2<<<blocks_for((size_t)N * 32 * HW[0]), 256, 0, st>>>(a, 32 * (long long)HW[1], 32, N, h, w, o, s0);
                return (int)cudaGetLastError();
            });
        }
        conv3(V{u1, s0}, 32, cu1.w, cu1.b, V{cat1, s0}, 16, 0);
        gated_fwd(gu1, V{cat1, s0}, V{g4, 16 * (long long)HW[0]}, 0, train);
        {
            const float *a = g4, *w = fin.w, *b = fin.b; float* o = y; const size_t hw = HW[0];
            push([=](cudaStream_t st) {
                unk::k_final<<<blocks_for((size_t)N * hw), 256, 0, st>>>(a, w, b, N, hw, o);
                return (int)cudaGetLastError();
            });
        }
    }
    float* g3 = nullptr; float* g4 = nullptr;     // outputs of the two norm-free gated blocks

    void emit_backward(bool train) {
        const int N = cfg.N;
        const long long s0 = 32 * (long long)HW[0], s1 = 64 * (long long)HW[1], s2 = 64 * (long long)HW[2];
        // input-gradient weights of this tape's forward weights
        for (const Gated* G : {&gs, &gd1, &gd2, &gu2, &gu1}) flip(G->w, 2 * G->c, G->cin, G->wt);
        flip(cu2.w, cu2.cout, cu2.cin, cu2.wt);
        flip(cu1.w, cu1.cout, cu1.cin, cu1.wt);
        {
            const float *d = dout, *yy = y, *w = fin.w, *a = g4; float *z = dz, *dg = dg4, *fp = fpart, *dw = fin.dw, *db = fin.db; const size_t hw = HW[0];
            push([=](cudaStream_t st) {
                unk::k_final_bwd<<<blocks_for((size_t)N * hw), 256, 0, st>>>(d, yy, w, N, hw, z, dg);
                unk::k_final_wgrad<<<kFinalCtas, 256, 0, st>>>(z, a, N, hw, fp);
                unk::k_final_wgrad_sum<<<1, 64, 0, st>>>(fp, kFinalCtas, dw, db);
                return (int)cudaGetLastError();
            });
        }
        // up1: G(32->16) over cat1, then the 32->16 conv over u1 and the upsample of g3
        gated_bwd(gu1, V{cat1, s0}, V{dg4, 16 * (long long)HW[0]}, dfm4, V{dcat1, s0}, 0, train);
        wgrad(V{u1, s0}, 32, V{dcat1, s0}, 16, 0, cu1.dw, cu1.db);
        conv3(V{dcat1, s0}, 16, cu1.wt, nullptr, V{du1, s0}, 32, 0);
        {
            const float* d = du1; float* o = dg3; const int h = H[1], w = Wd[1];
            push([=](cudaStream_t st) {
                unk::k_upsample2_bwd<<<blocks_for((size_t)N * 32 * HW[1]), 256, 0, st>>>(d, s0, 32, N, h, w, o, 32 * (long long)HW[1]);
                return (int)cudaGetLastError();
            });
        }
        // up2: G(64->32) over cat2, then the 64->32 conv over u2 and the upsample of d2
        gated_bwd(gu2, V{cat2, s1}, V{dg3, 32 * (long long)HW[1]}, dfm3, V{dcat2, s1}, 1, train);
        wgrad(V{u2, s1}, 64, V{dcat2, s1}, 32, 1, cu2.dw, cu2.db);
        conv3(V{dcat2, s1}, 32, cu2.wt, nullptr, V{du2, s1}, 64, 1);
        {
            const float* d = du2; float* o = dd2; const int h = H[2], w = Wd[2];
            push([=](cudaStream_t st) {
                unk::k_upsample2_bwd<<<blocks_for((size_t)N * 64 * HW[2]), 256, 0, st>>>(d, s1, 64, N, h, w, o, s2);
                return (int)cudaGetLastError();
            });
        }
        // down2: dd2[0:45] -> G(32->45) over p2 -> dp2 -> avgpool backward into d1's gradient (dcat2[32:64])
        gated_bwd(gd2, V{p2, 32 * (long long)HW[2]}, V{dd2, s2}, dfm2, V{dp2, 32 * (long long)HW[2]}, 2, train);
        {
            const float* d = dp2; float* o = dcat2 + 32 * HW[1]; const int h = H[1], w = Wd[1];
            push([=](cudaStream_t st) {
                unk::k_avgpool_bwd_add<<<blocks_for((size_t)N * 32 * HW[1]), 256, 0, st>>>(d, 32 * (long long)HW[2], 32, N, h, w, o, s1);
                return (int)cudaGetLastError();
            });
        }
        // down1: dd1[0:13] -> G(16->13) over p1 -> dp1 -> avgpool backward into in64's gradient (dcat1[16:32])
        gated_bwd(gd1, V{p1, 16 * (long long)HW[1]}, V{dcat2 + 32 * HW[1], s1}, dfm1, V{dp1, 16 * (long long)HW[1]}, 1, train);
        {
            const float* d = dp1; float* o = dcat1 + 16 * HW[0]; const int h = H[0], w = Wd[0];
            push([=](cudaStream_t st) {
                unk::k_avgpool_bwd_add<<<blocks_for((size_t)N * 16 * HW[0]), 256, 0, st>>>(d, 16 * (long long)HW[1], 16, N, h, w, o, s0);
                return (int)cudaGetLastError();
            });
        }
        // start: d in64 -> G(19->16) over x0 -> dx0
        gated_bwd(gs, V{x0, 19 * (long long)HW[0]}, V{dcat1 + 16 * HW[0], s0}, dfm0, V{dx0, 19 * (long long)HW[0]}, 0, train);
    }

    int build(bool dry_run) {
        dry = dry_run; off = 0; err = 0; entries.clear(); named.clear();
        fwd_train.clear(); fwd_eval.clear(); bwd_train.clear(); bwd_eval.clear();
        const int N = cfg.N;
        for (int l = 0; l < 3; l++) { H[l] = cfg.H >> l; Wd[l] = cfg.W >> l; HW[l] = (size_t)H[l] * Wd[l]; }
        // parameters and buffers, in the reference's state_dict order
        gated(gs, "start.block.", 19, 16, 1, 0);
        gated(gd1, "down1.conv.block.", 16, 13, 1, 1);
        gated(gd2, "down2.conv.block.", 32, 45, 1, 2);
        conv(cu2, "up2.up.1.0", 64, 32, 3);
        gated(gu2, "up2.conv.block.", 64, 32, 0, 1);
        conv(cu1, "up1.up.1.0", 32, 16, 3);
        gated(gu1, "up1.conv.block.", 32, 16, 0, 0);
        conv(fin, "final.0.0", 16, 3, 1);
        // activations
        x0 = alloc32((size_t)N * 19 * HW[0]);
        cat1 = alloc32((size_t)N * 32 * HW[0]); p1 = alloc32((size_t)N * 16 * HW[1]);
        cat2 = alloc32((size_t)N * 64 * HW[1]); p2 = alloc32((size_t)N * 32 * HW[2]); d2 = alloc32((size_t)N * 64 * HW[2]);
        u2 = alloc32((size_t)N * 64 * HW[1]); g3 = alloc32((size_t)N * 32 * HW[1]); u1 = alloc32((size_t)N * 32 * HW[0]);
        g4 = alloc32((size_t)N * 16 * HW[0]); y = alloc32((size_t)N * 3 * HW[0]);
        // backward
        dout = alloc32((size_t)N * 3 * HW[0]); dz = alloc32((size_t)N * 3 * HW[0]); dg4 = alloc32((size_t)N * 16 * HW[0]);
        dfm4 = alloc32((size_t)N * 32 * HW[0]); dcat1 = alloc32((size_t)N * 32 * HW[0]); du1 = alloc32((size_t)N * 32 * HW[0]);
        dg3 = alloc32((size_t)N * 32 * HW[1]); dfm3 = alloc32((size_t)N * 64 * HW[1]); dcat2 = alloc32((size_t)N * 64 * HW[1]);
        du2 = alloc32((size_t)N * 64 * HW[1]); dd2 = alloc32((size_t)N * 64 * HW[2]); dfm2 = alloc32((size_t)N * 90 * HW[2]);
        dp2 = alloc32((size_t)N * 32 * HW[2]); dfm1 = alloc32((size_t)N * 26 * HW[1]); dp1 = alloc32((size_t)N * 16 * HW[1]);
        dfm0 = alloc32((size_t)N * 32 * HW[0]); dx0 = alloc32((size_t)N * 19 * HW[0]);
        // reduction scratch (the ops run one at a time on one stream)
        wpart = alloc32(kMaxWgradElems); bpart = alloc32((size_t)kWgradCtas * 64); fpart = alloc32((size_t)kFinalCtas * 51);
        cpart = (double*)alloc((size_t)64 * kChanChunks * 2 * sizeof(double));
        cur = &fwd_train; emit_forward(true);
        cur = &fwd_eval; emit_forward(false);
        cur = &bwd_train; emit_backward(true);
        cur = &bwd_eval; emit_backward(false);
        cur = nullptr;
        tap("in64", cat1 + 16 * HW[0], (size_t)N * 16 * HW[0] * 4);   // per-image stride 32 * H * W
        tap("cat1", cat1, (size_t)N * 32 * HW[0] * 4);
        tap("cat2", cat2, (size_t)N * 64 * HW[1] * 4);
        tap("d2", d2, (size_t)N * 64 * HW[2] * 4);
        tap("up2", g3, (size_t)N * 32 * HW[1] * 4);
        tap("up1", g4, (size_t)N * 16 * HW[0] * 4);
        tap("out", y, (size_t)N * 3 * HW[0] * 4);
        return err;
    }
};

bool valid_cfg(const mi3d_unet_shape& c) { return c.N >= 1 && c.N <= 16 && c.H >= 4 && c.W >= 4 && c.H % 4 == 0 && c.W % 4 == 0 && c.H <= 4096 && c.W <= 4096; }

// copy n images of `ch` channels (each image's channels contiguous) between views with different per-image strides
cudaError_t copy_slice(float* dst, long long dst_ns, const float* src, long long src_ns, int n, size_t elems, cudaStream_t st) {
    return cudaMemcpy2DAsync(dst, dst_ns * 4, src, src_ns * 4, elems * 4, n, cudaMemcpyDeviceToDevice, st);
}

}  // namespace unet

struct mi3d_unet { unet::Engine e; };

extern "C" {

size_t mi3d_unet_workspace_bytes(const mi3d_unet_shape* cfg) {
    if (!cfg || !unet::valid_cfg(*cfg)) return 0;
    unet::Engine e; e.cfg = *cfg;
    e.build(true);
    return e.off + (1 << 20);
}

mi3d_unet_t mi3d_unet_create(const mi3d_unet_shape* cfg, void* workspace, size_t workspace_bytes) {
    if (!cfg || !workspace || !unet::valid_cfg(*cfg)) return nullptr;
    mi3d_unet* h = new mi3d_unet();
    h->e.cfg = *cfg; h->e.base = (uint8_t*)workspace; h->e.cap = workspace_bytes;
    int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&h->e.num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (h->e.build(false) != 0) { delete h; return nullptr; }
    return h;
}

void mi3d_unet_destroy(mi3d_unet_t h) { delete h; }

int mi3d_unet_num_params(mi3d_unet_t h) { return h ? (int)h->e.entries.size() : 0; }
const char* mi3d_unet_param_name(mi3d_unet_t h, int i) {
    if (!h || i < 0 || i >= (int)h->e.entries.size()) return nullptr;
    return h->e.entries[i].name.c_str();
}
int mi3d_unet_param_shape(mi3d_unet_t h, int i, int* shape4) {
    if (!h || !shape4 || i < 0 || i >= (int)h->e.entries.size()) return -1;
    const auto& s = h->e.entries[i].shape;
    for (int k = 0; k < 4; k++) shape4[k] = k < (int)s.size() ? s[k] : 0;
    return (int)s.size();
}

int mi3d_unet_set_graph_replay(mi3d_unet_t h, int enable) {
    if (!h) return MI3D_ERR_ARG;
    h->e.use_graph = enable != 0;
    return MI3D_OK;
}

int mi3d_unet_graph_replays(mi3d_unet_t h) { return h ? h->e.graph_replays() : -1; }

int mi3d_unet_forward(mi3d_unet_t h, const float* x0, const float* x1, const float* x2, void* const* state, int train, int need_grad, float* out,
                      mi3d_stream_t stream) {
    if (!h || !x0 || !x1 || !x2 || !state || !out) return MI3D_ERR_ARG;
    unet::Engine& e = h->e; const int N = e.cfg.N;
    // batch statistics need more than one value per channel (H/4 x W/4 is the smallest level), as in torch's BatchNorm
    if (train && (size_t)N * e.HW[2] < 2) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    e.tape = 0;
    // the current parameter values (and, in eval mode, running statistics) into the workspace
    unk::CopyList cl = {}; int nt = 0;
    for (size_t i = 0; i < e.entries.size(); i++) {
        const unet::Entry& en = e.entries[i];
        if (en.kind == unet::E_COUNT) continue;
        if (!state[i]) { if (en.kind == unet::E_PARAM || !train) return MI3D_ERR_ARG; continue; }
        if (nt == 48) return MI3D_ERR_ARG;
        cl.src[nt] = (const float*)state[i]; cl.dst[nt] = en.slot; cl.n[nt] = (int)en.numel; nt++;
    }
    cl.count = nt;
    unk::k_copy_list<<<dim3(32, nt), 256, 0, st>>>(cl);
    MI3D_CHECK(cudaGetLastError());
    const size_t* HW = e.HW;
    MI3D_CHECK(cudaMemcpyAsync(e.x0, x0, (size_t)N * 19 * HW[0] * 4, cudaMemcpyDeviceToDevice, st));
    MI3D_CHECK(unet::copy_slice(e.cat2 + 45 * HW[1], 64 * (long long)HW[1], x1, 19 * (long long)HW[1], N, 19 * HW[1], st));
    MI3D_CHECK(unet::copy_slice(e.d2 + 45 * HW[2], 64 * (long long)HW[2], x2, 19 * (long long)HW[2], N, 19 * HW[2], st));
    int r = e.run(train ? e.fwd_train : e.fwd_eval, st); if (r) return r;
    if (train) {
        // running statistics: each layer normalised over N x its own H x W
        const unet::Gated* gl[3] = {&e.gs, &e.gd1, &e.gd2};
        unk::RunningList rl = {};
        for (int l = 0; l < 3; l++) {
            rl.rmean[l] = (float*)state[gl[l]->e_rmean]; rl.rvar[l] = (float*)state[gl[l]->e_rvar]; rl.nbt[l] = (long long*)state[gl[l]->e_count];
            rl.mean[l] = gl[l]->mean; rl.var[l] = gl[l]->var; rl.C[l] = gl[l]->c; rl.M[l] = (double)N * HW[l];
        }
        rl.momentum = 0.1f;
        unk::k_bn_running<<<3, 64, 0, st>>>(rl);
        MI3D_CHECK(cudaGetLastError());
    }
    MI3D_CHECK(cudaMemcpyAsync(out, e.y, (size_t)N * 3 * HW[0] * 4, cudaMemcpyDeviceToDevice, st));
    e.tape = need_grad ? (train ? 1 : 2) : 0;
    return MI3D_OK;
}

int mi3d_unet_backward(mi3d_unet_t h, const float* dout, float* dx0, float* dx1, float* dx2, float* const* grads, mi3d_stream_t stream) {
    if (!h || !dout || !dx0 || !dx1 || !dx2 || !grads) return MI3D_ERR_ARG;
    unet::Engine& e = h->e; const int N = e.cfg.N;
    if (!e.tape) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t* HW = e.HW;
    MI3D_CHECK(cudaMemcpyAsync(e.dout, dout, (size_t)N * 3 * HW[0] * 4, cudaMemcpyDeviceToDevice, st));
    int r = e.run(e.tape == 1 ? e.bwd_train : e.bwd_eval, st); if (r) return r;
    MI3D_CHECK(cudaMemcpyAsync(dx0, e.dx0, (size_t)N * 19 * HW[0] * 4, cudaMemcpyDeviceToDevice, st));
    MI3D_CHECK(unet::copy_slice(dx1, 19 * (long long)HW[1], e.dcat2 + 45 * HW[1], 64 * (long long)HW[1], N, 19 * HW[1], st));
    MI3D_CHECK(unet::copy_slice(dx2, 19 * (long long)HW[2], e.dd2 + 45 * HW[2], 64 * (long long)HW[2], N, 19 * HW[2], st));
    unk::CopyList cl = {}; int nt = 0;
    for (size_t i = 0; i < e.entries.size(); i++) {
        const unet::Entry& en = e.entries[i];
        if (en.kind != unet::E_PARAM || !grads[i]) continue;
        if (nt == 48) return MI3D_ERR_ARG;
        cl.src[nt] = en.grad; cl.dst[nt] = grads[i]; cl.n[nt] = (int)en.numel; nt++;
    }
    cl.count = nt;
    if (nt) unk::k_copy_list<<<dim3(32, nt), 256, 0, st>>>(cl);
    return (int)cudaGetLastError();
}

int mi3d_unet_debug_tensor(mi3d_unet_t h, const char* name, void** ptr, size_t* bytes) {
    if (!h || !name || !ptr || !bytes) return MI3D_ERR_ARG;
    auto it = h->e.named.find(name);
    if (it == h->e.named.end()) return MI3D_ERR_ARG;
    *ptr = it->second.first; *bytes = it->second.second;
    return MI3D_OK;
}

}  // extern "C"
