// coarse.cu -- B12: the per-iteration losses of the coarse loop (nerf/utils.py:491-493, :519-533, :551-556), for sm_90a
// (C ABI: include/mi3d.h)
//
// Forward (no atomics; every reduction is per-CTA fp64 partials folded by one CTA in a fixed order):
//   1. k_coarse_up            one CTA per 512-row: the align_corners=True bilinear upsample of the [h*w,3] ray-major image
//                             (pred512) and, on front views, of the depth (kept raw in the workspace); the gt composite (gt512);
//                             partial sums of |pred512 - gt512|, of x = nan_to_num(up(depth)) and of the prior over the mask, and of
//                             the opacity / entropy terms of the low-res weights_sum
//   2. k_coarse_finish_means  one CTA: opacity, entropy, l1; the masked pixel count and the two means (kept on the device)
//   3. k_coarse_centred       (front only) one CTA per 512-row: centred sums (x - mx)^2, (y - my)^2, (x - mx)(y - my)
//   4. k_coarse_finish_corr   (front only) one CTA: the Pearson coefficient, clamped to [-1, 1] (NaN stays NaN)
// so 4 launches on front views and 2 on the others.
// Backward: k_coarse_grad, one CTA per low-res row and one launch.  dL/dpred512 (the L1 sign term plus the caller's incoming
// gradient) and dL/dx512 (the Pearson term) are formed on the fly and gathered through the upsample's adjoint: the row pass sums the
// 512-rows whose bilinear stencil holds this low-res row into shared memory, the column pass sums the 512-columns holding each
// low-res pixel; both in ascending order, in fp64, with no atomics, so the result is bitwise repeatable.  The weights_sum gradient
// (opacity, entropy) is element-wise in the same launch.
//
// Compiled with -fmad=false: every element-wise op rounds once, like torch's separate kernels.
#include <math.h>
#include <float.h>

#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kOut = 512;                  // F.interpolate(., (512, 512)) and the reference image size
constexpr int kPix = kOut * kOut;
constexpr int kThreads = 512;              // one thread per 512-column
constexpr int kPart = 8;                   // doubles per CTA partial
constexpr float kLo = 1e-5f;               // clamp(ws, 1e-5, 1 - 1e-5): the Python scalars as torch converts them for fp32
constexpr float kHi = (float)(1.0 - 1e-5);

// stats block of the workspace
enum { ST_N, ST_MX, ST_MY, ST_R, ST_INV, ST_R_SXX, kStats = 8 };

struct Tap {
    int i0, i1;
    float l0, l1;
};

// torch's upsample_bilinear2d (align_corners=True) source taps of output index o for an input of size n, in fp32
__device__ __forceinline__ Tap tap(int n, int o) {
    const float scale = (float)(n - 1) / (float)(kOut - 1);
    const float src = scale * (float)o;
    const int i0 = (int)src;
    Tap t;
    t.i0 = i0;
    t.i1 = i0 + (i0 < n - 1 ? 1 : 0);
    t.l1 = src - (float)i0;
    t.l0 = 1.0f - t.l1;
    return t;
}

__device__ __forceinline__ float bilerp(const float* src, int stride, int ld, const Tap& ty, const Tap& tx) {
    const float a00 = src[((size_t)ty.i0 * ld + tx.i0) * stride], a01 = src[((size_t)ty.i0 * ld + tx.i1) * stride];
    const float a10 = src[((size_t)ty.i1 * ld + tx.i0) * stride], a11 = src[((size_t)ty.i1 * ld + tx.i1) * stride];
    return ty.l0 * (tx.l0 * a00 + tx.l1 * a01) + ty.l1 * (tx.l0 * a10 + tx.l1 * a11);
}

__device__ __forceinline__ float nan_to_num(float v) {
    if (isnan(v)) return 0.0f;
    if (isinf(v)) return v > 0.0f ? FLT_MAX : -FLT_MAX;
    return v;
}

// clamp(v, lo, hi) as torch computes it: NaN passes through
__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// fixed-order block sum of K doubles (warp shuffle tree, then the warp totals in warp order); thread 0 gets the result
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    #pragma unroll
    for (int k = 0; k < K; k++)
        #pragma unroll
        for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], off);
    if (lane == 0)
        #pragma unroll
        for (int k = 0; k < K; k++) sh[warp * K + k] = v[k];
    __syncthreads();
    if (warp == 0) {
        #pragma unroll
        for (int k = 0; k < K; k++) {
            v[k] = lane < nw ? sh[lane * K + k] : 0.0;
            #pragma unroll
            for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], off);
        }
    }
    __syncthreads();
}

struct FwdArgs {
    const float* image;        // [h*w,3]
    const float* depth;        // [h*w]
    const float* ws;           // [h*w]
    int h, w;
    const float* ref;          // [1,4,512,512]
    const float* bg;           // [3]
    const double* prior;       // [512,512]
    const uint8_t* mask;       // [512,512]
    int front;
    float* pred512;            // [1,3,512,512]
    float* gt512;              // [1,3,512,512]
    float* raw512;             // [512,512] up(depth) before nan_to_num (workspace)
    double* partials;          // [512][kPart] (workspace)
};

__global__ void __launch_bounds__(kThreads) k_coarse_up(FwdArgs a) {
    __shared__ double sh[32 * 6];
    const int oy = blockIdx.x, ox = threadIdx.x;
    const size_t pix = (size_t)oy * kOut + ox;
    const Tap ty = tap(a.h, oy), tx = tap(a.w, ox);
    double l1 = 0.0, sx = 0.0, sy = 0.0, n = 0.0, op = 0.0, en = 0.0;
    const float alpha = a.ref[3 * (size_t)kPix + pix];
    #pragma unroll
    for (int c = 0; c < 3; c++) {
        const float p = bilerp(a.image + c, 3, a.w, ty, tx);
        const float g = a.ref[c * (size_t)kPix + pix] * alpha + a.bg[c] * (1.0f - alpha);
        a.pred512[c * (size_t)kPix + pix] = p;
        a.gt512[c * (size_t)kPix + pix] = g;
        if (a.front) l1 += (double)fabsf(p - g);
    }
    if (a.front) {
        const float raw = bilerp(a.depth, 1, a.w, ty, tx);
        a.raw512[pix] = raw;
        if (a.mask[pix]) {
            sx += (double)nan_to_num(raw);
            sy += a.prior[pix];
            n += 1.0;
        }
    }
    const int hw = a.h * a.w;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < hw; i += kOut * kThreads) {
        const float v = a.ws[i];
        op += (double)(v * v);
        const float al = clamp_nan(v, kLo, kHi);
        en += (double)((-al) * log2f(al) - (1.0f - al) * log2f(1.0f - al));
    }
    double v[6] = {l1, sx, sy, n, op, en};
    block_sum<6>(v, sh);
    if (threadIdx.x == 0)
        #pragma unroll
        for (int k = 0; k < 6; k++) a.partials[blockIdx.x * kPart + k] = v[k];
}

// terms[0..2] = opacity, entropy, l1 (0 off the front); stats: masked count and means
__global__ void __launch_bounds__(kThreads) k_coarse_finish_means(const double* __restrict__ partials, int hw, int front,
                                                                  float* __restrict__ terms, double* __restrict__ st) {
    __shared__ double sh[32 * 6];
    double v[6];
    #pragma unroll
    for (int k = 0; k < 6; k++) v[k] = partials[threadIdx.x * kPart + k];
    block_sum<6>(v, sh);
    if (threadIdx.x == 0) {
        terms[0] = (float)(v[4] / (double)hw);
        terms[1] = (float)(v[5] / (double)hw);
        terms[2] = front ? (float)(v[0] / (3.0 * (double)kPix)) : 0.0f;
        if (!front) terms[3] = 0.0f;
        st[ST_N] = v[3];
        st[ST_MX] = v[1] / v[3];
        st[ST_MY] = v[2] / v[3];
    }
}

__global__ void __launch_bounds__(kThreads) k_coarse_centred(const float* __restrict__ raw512, const double* __restrict__ prior,
                                                             const uint8_t* __restrict__ mask, const double* __restrict__ st,
                                                             double* __restrict__ partials) {
    __shared__ double sh[32 * 3];
    const size_t pix = (size_t)blockIdx.x * kOut + threadIdx.x;
    double v[3] = {0.0, 0.0, 0.0};
    if (mask[pix]) {
        const double dx = (double)nan_to_num(raw512[pix]) - st[ST_MX], dy = prior[pix] - st[ST_MY];
        v[0] = dx * dx;
        v[1] = dy * dy;
        v[2] = dx * dy;
    }
    block_sum<3>(v, sh);
    if (threadIdx.x == 0)
        #pragma unroll
        for (int k = 0; k < 3; k++) partials[blockIdx.x * kPart + k] = v[k];
}

// torchmetrics' PearsonCorrCoef: cov / sqrt(var_x var_y) with the (n - 1) divisions, clamped to [-1, 1]; < 2 pixels give NaN
__global__ void __launch_bounds__(kThreads) k_coarse_finish_corr(const double* __restrict__ partials, float* __restrict__ terms,
                                                                 double* __restrict__ st) {
    __shared__ double sh[32 * 3];
    double v[3];
    #pragma unroll
    for (int k = 0; k < 3; k++) v[k] = partials[threadIdx.x * kPart + k];
    block_sum<3>(v, sh);
    if (threadIdx.x == 0) {
        const double n1 = st[ST_N] - 1.0;
        const double vx = v[0] / n1, vy = v[1] / n1, cxy = v[2] / n1;
        const double r = cxy / sqrt(vx * vy);
        st[ST_R] = r;
        st[ST_INV] = 1.0 / sqrt(v[0] * v[1]);       // dr/dx_i = (y_i - my) / sqrt(Sxx Syy) - r (x_i - mx) / Sxx
        st[ST_R_SXX] = r / v[0];
        terms[3] = (float)(r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r));
    }
}

struct BwdArgs {
    const float* ws;           // [h*w]
    int h, w;
    const float* pred512;
    const float* gt512;
    const float* raw512;
    const double* prior;
    const uint8_t* mask;
    const double* st;
    int front;
    const float* g;            // [4]
    const float* gpred512;     // nullable
    float* gimage;             // [h*w,3]
    float* gdepth;             // [h*w]
    float* gws;                // [h*w]
};

// first index in [0, kOut) whose i0 >= target (kOut if none)
__device__ __forceinline__ int lower_bound_i0(const int* i0, int target) {
    int lo = 0, hi = kOut;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (i0[mid] < target) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// weight of input index i in the stencil of output tap t (both taps count when they coincide at the last row / column)
__device__ __forceinline__ double tap_weight(int i, int i0, int i1, float l0, float l1) {
    return (i0 == i ? (double)l0 : 0.0) + (i1 == i ? (double)l1 : 0.0);
}

__global__ void __launch_bounds__(kThreads) k_coarse_grad(BwdArgs a) {
    __shared__ int s_y0[kOut], s_y1[kOut], s_x0[kOut], s_x1[kOut];
    __shared__ float s_yl0[kOut], s_yl1[kOut], s_xl0[kOut], s_xl1[kOut];
    __shared__ double s_t[4][kOut];
    const int iy = blockIdx.x, t = threadIdx.x;
    {
        const Tap ty = tap(a.h, t), tx = tap(a.w, t);
        s_y0[t] = ty.i0; s_y1[t] = ty.i1; s_yl0[t] = ty.l0; s_yl1[t] = ty.l1;
        s_x0[t] = tx.i0; s_x1[t] = tx.i1; s_xl0[t] = tx.l0; s_xl1[t] = tx.l1;
    }
    __syncthreads();
    // mean backward then abs backward: (g / N) * sign(pred - gt)
    const float gl1 = a.front ? a.g[2] / (float)(3 * kPix) : 0.0f;
    // the clamp passes the gradient where -1 <= r <= 1 (inclusive; NaN passes nothing)
    const double r = a.front ? a.st[ST_R] : 0.0;
    const bool corr = a.front && r >= -1.0 && r <= 1.0;
    const double gp = corr ? (double)a.g[3] : 0.0;
    const double inv = corr ? a.st[ST_INV] : 0.0, rs = corr ? a.st[ST_R_SXX] : 0.0;
    const double mx = corr ? a.st[ST_MX] : 0.0, my = corr ? a.st[ST_MY] : 0.0;
    // row pass: 512-rows oy with i0(oy) in {iy - 1, iy}, ascending
    const int oy_lo = lower_bound_i0(s_y0, iy - 1), oy_hi = lower_bound_i0(s_y0, iy + 1);
    {
        const int ox = t;
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int oy = oy_lo; oy < oy_hi; oy++) {
            if (s_y0[oy] != iy && s_y1[oy] != iy) continue;
            const double wy = tap_weight(iy, s_y0[oy], s_y1[oy], s_yl0[oy], s_yl1[oy]);
            const size_t pix = (size_t)oy * kOut + ox;
            #pragma unroll
            for (int c = 0; c < 3; c++) {
                const size_t i = c * (size_t)kPix + pix;
                float gc = 0.0f;
                if (a.front) {
                    const float d = a.pred512[i] - a.gt512[i];
                    gc = gl1 * (d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f));
                }
                if (a.gpred512) gc = gc + a.gpred512[i];
                acc[c] += wy * (double)gc;
            }
            if (corr && a.mask[pix]) {
                const float raw = a.raw512[pix];
                if (isfinite(raw)) {                  // nan_to_num passes no gradient where its input was not finite
                    const double dx = (double)raw - mx, dy = a.prior[pix] - my;
                    acc[3] += wy * (double)(float)(gp * (dy * inv - rs * dx));
                }
            }
        }
        #pragma unroll
        for (int c = 0; c < 4; c++) s_t[c][ox] = acc[c];
    }
    __syncthreads();
    // column pass and the element-wise weights_sum gradient of this row
    const float inv_hw = 1.0f / (float)(a.h * a.w);
    const float go = a.g[0] * inv_hw, ge = a.g[1] * inv_hw;
    for (int ix = t; ix < a.w; ix += kThreads) {
        const int ox_lo = lower_bound_i0(s_x0, ix - 1), ox_hi = lower_bound_i0(s_x0, ix + 1);
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int ox = ox_lo; ox < ox_hi; ox++) {
            if (s_x0[ox] != ix && s_x1[ox] != ix) continue;
            const double wx = tap_weight(ix, s_x0[ox], s_x1[ox], s_xl0[ox], s_xl1[ox]);
            #pragma unroll
            for (int c = 0; c < 4; c++) acc[c] += wx * s_t[c][ox];
        }
        const size_t p = (size_t)iy * a.w + ix;
        #pragma unroll
        for (int c = 0; c < 3; c++) a.gimage[p * 3 + c] = (float)acc[c];
        a.gdepth[p] = (float)acc[3];
        // d/dws of mean(ws^2) and of the entropy of clamp(ws): 2 ws and log2(1 - a) - log2(a), zero outside the clamp's bounds
        const float v = a.ws[p];
        float gv = go * (2.0f * v);
        if (v >= kLo && v <= kHi) gv = gv + ge * (log2f(1.0f - v) - log2f(v));
        a.gws[p] = gv;
    }
}

constexpr size_t kPartBytes = (size_t)kOut * kPart * sizeof(double);
constexpr size_t kStatBytes = kStats * sizeof(double);
constexpr size_t kRawOffset = kPartBytes + kStatBytes;
constexpr size_t kWorkspaceBytes = kRawOffset + (size_t)kPix * sizeof(float);

inline bool dims_ok(uint32_t h, uint32_t w) { return h >= 2 && w >= 2 && h <= 16384 && w <= 16384; }

}  // namespace

extern "C" {

size_t mi3d_coarse_losses_workspace_bytes(uint32_t h, uint32_t w) { return dims_ok(h, w) ? kWorkspaceBytes : 0; }

int mi3d_coarse_losses(const float* image, const float* depth, const float* weights_sum, uint32_t h, uint32_t w, const float* ref_rgba,
                       const float* bg_color, const double* depth_prior, const uint8_t* depth_mask, int front, float* pred512, float* gt512,
                       float* terms, void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    if (!dims_ok(h, w) || !image || !weights_sum || !ref_rgba || !bg_color || !pred512 || !gt512 || !terms || !workspace) return MI3D_ERR_ARG;
    if (front && (!depth || !depth_prior || !depth_mask)) return MI3D_ERR_ARG;
    if (workspace_bytes < kWorkspaceBytes) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    double* partials = (double*)ws;
    double* stats = (double*)(ws + kPartBytes);
    FwdArgs a;
    a.image = image; a.depth = depth; a.ws = weights_sum; a.h = (int)h; a.w = (int)w;
    a.ref = ref_rgba; a.bg = bg_color; a.prior = depth_prior; a.mask = depth_mask; a.front = front ? 1 : 0;
    a.pred512 = pred512; a.gt512 = gt512; a.raw512 = (float*)(ws + kRawOffset); a.partials = partials;
    k_coarse_up<<<kOut, kThreads, 0, st>>>(a);
    k_coarse_finish_means<<<1, kThreads, 0, st>>>(partials, (int)(h * w), a.front, terms, stats);
    if (front) {
        k_coarse_centred<<<kOut, kThreads, 0, st>>>(a.raw512, depth_prior, depth_mask, stats, partials);
        k_coarse_finish_corr<<<1, kThreads, 0, st>>>(partials, terms, stats);
    }
    MI3D_RETURN_LAUNCH();
}

int mi3d_coarse_losses_backward(const float* weights_sum, uint32_t h, uint32_t w, const float* pred512, const float* gt512,
                                const double* depth_prior, const uint8_t* depth_mask, int front, const float* grad_terms,
                                const float* grad_pred512, const void* workspace, size_t workspace_bytes, float* grad_image,
                                float* grad_depth, float* grad_weights_sum, mi3d_stream_t stream) {
    if (!dims_ok(h, w) || !weights_sum || !grad_terms || !workspace || !grad_image || !grad_depth || !grad_weights_sum) return MI3D_ERR_ARG;
    if (front && (!pred512 || !gt512 || !depth_prior || !depth_mask)) return MI3D_ERR_ARG;
    if (workspace_bytes < kWorkspaceBytes) return MI3D_ERR_ARG;
    const char* ws = (const char*)workspace;
    BwdArgs a;
    a.ws = weights_sum; a.h = (int)h; a.w = (int)w; a.pred512 = pred512; a.gt512 = gt512;
    a.raw512 = (const float*)(ws + kRawOffset); a.prior = depth_prior; a.mask = depth_mask;
    a.st = (const double*)(ws + kPartBytes); a.front = front ? 1 : 0; a.g = grad_terms; a.gpred512 = grad_pred512;
    a.gimage = grad_image; a.gdepth = grad_depth; a.gws = grad_weights_sum;
    k_coarse_grad<<<h, kThreads, 0, (cudaStream_t)stream>>>(a);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
