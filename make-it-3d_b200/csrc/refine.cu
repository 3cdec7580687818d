// refine.cu -- B11: the per-iteration glue of the refine loop (nerf/utils.py:865-894), for sm_90a (C ABI: include/mi3d.h)
//
// Image losses (forward, no atomics, fixed-order reductions):
//   1. k_refine_image_losses  one CTA per 16x16 pixel tile: the coverage of the tile plus a 2-pixel halo from the scale-0 composite
//                             weights (sum over the ppp slots in slot order, starting at 0: the unit-colour render_point image, bit for
//                             bit), the 5x5 max dilation (MaxPool2d(5, 1, 2), -inf padding), then per pixel and channel the background
//                             term 1 - pred (1 - dilate) and, on front iterations, |pred m - gt m|; per-CTA partial sums in fp64
//   2. k_refine_finish        one CTA: the partial sums in a fixed order -> bg_loss = 1e-3 sum, l1 = 1000 mean
// Backward: k_refine_image_grad writes dL/dpred of both terms from pred, gt, mask and the saved dilation (torch's op order).
//
// Adam (torch.optim.Adam, foreach path, in its operation order: adam_update.cuh): one launch over the concatenation of every
// parameter tensor, a device table of segments.  Segment 0 may be the refine cloud's [P,19] buffer; its colour columns then get the
// gradient of the two MSE regularisers added on the fly, and their values are reduced like the image losses.
//
// Compiled with -fmad=false: every element-wise op rounds once, like torch's separate kernels; where torch's own kernels contract
// to an FMA (lerp, addcmul, addcdiv) the fmaf is written out.
#include <math.h>

#include "adam_update.cuh"
#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kTile = 16;
constexpr int kHalo = 2;                         // MaxPool2d(kernel 5, stride 1, padding 2)
constexpr int kSpan = kTile + 2 * kHalo;
constexpr int kFinThreads = 1024;
constexpr int kAdamThreads = 256;
constexpr int kAdamPerThread = 8;
constexpr int kAdamChunk = kAdamThreads * kAdamPerThread;
constexpr int kMaxSegs = 256;
constexpr uint32_t kCols = 19;                   // 3 colours + 16 features per point
constexpr uint32_t kColourCols = 3;

// fixed-order block sum of two doubles (blockDim.x * blockDim.y threads, a power of two); thread 0 gets the result
template <int NT>
__device__ __forceinline__ void block_sum2(double& a, double& b, double* sa, double* sb) {
    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    sa[tid] = a;
    sb[tid] = b;
    __syncthreads();
    #pragma unroll
    for (int s = NT / 2; s > 0; s >>= 1) {
        if (tid < s) { sa[tid] += sa[tid + s]; sb[tid] += sb[tid + s]; }
        __syncthreads();
    }
    a = sa[0];
    b = sb[0];
}

__global__ void __launch_bounds__(kTile * kTile)
k_refine_image_losses(const float* __restrict__ w, int S, int ppp, const float* __restrict__ pred, const float* __restrict__ gt,
                      const float* __restrict__ mask, int front, float* __restrict__ cover, float* __restrict__ dilated,
                      double2* __restrict__ partials) {
    __shared__ float s_cov[kSpan][kSpan];
    __shared__ double s_a[kTile * kTile], s_b[kTile * kTile];
    const int tid = threadIdx.y * kTile + threadIdx.x;
    const int x0 = blockIdx.x * kTile - kHalo, y0 = blockIdx.y * kTile - kHalo;
    for (int i = tid; i < kSpan * kSpan; i += kTile * kTile) {
        const int hy = y0 + i / kSpan, hx = x0 + i % kSpan;
        float acc = -INFINITY;
        if (hy >= 0 && hy < S && hx >= 0 && hx < S) {
            const float* wp = w + ((size_t)hy * S + hx) * ppp;
            acc = 0.0f;
            for (int k = 0; k < ppp; k++) acc = acc + wp[k];
        }
        s_cov[i / kSpan][i % kSpan] = acc;
    }
    __syncthreads();
    const int x = blockIdx.x * kTile + threadIdx.x, y = blockIdx.y * kTile + threadIdx.y;
    double bg = 0.0, l1 = 0.0;
    if (x < S && y < S) {
        float d = -INFINITY;
        #pragma unroll
        for (int dy = 0; dy < 5; dy++)
            #pragma unroll
            for (int dx = 0; dx < 5; dx++) d = fmaxf(d, s_cov[threadIdx.y + dy][threadIdx.x + dx]);
        const size_t pix = (size_t)y * S + x, HW = (size_t)S * S;
        if (cover) cover[pix] = s_cov[threadIdx.y + kHalo][threadIdx.x + kHalo];
        dilated[pix] = d;
        const float keep = 1.0f - d;
        const float m = front ? mask[pix] : 0.0f;
        #pragma unroll
        for (int c = 0; c < 3; c++) {
            const float p = pred[c * HW + pix];
            bg += (double)(1.0f - p * keep);
            if (front) l1 += (double)fabsf(p * m - gt[c * HW + pix] * m);
        }
    }
    block_sum2<kTile * kTile>(bg, l1, s_a, s_b);
    if (tid == 0) partials[blockIdx.y * gridDim.x + blockIdx.x] = make_double2(bg, l1);
}

// one CTA: out[0] = s0 * sum of partials[.].x, out[1] = s1 * sum of partials[.].y (each thread a strided sum, then a fixed tree)
__global__ void __launch_bounds__(kFinThreads) k_refine_finish(const double2* __restrict__ partials, int n, double s0, double s1,
                                                               float* __restrict__ out) {
    __shared__ double s_a[kFinThreads], s_b[kFinThreads];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < n; i += kFinThreads) { a += partials[i].x; b += partials[i].y; }
    block_sum2<kFinThreads>(a, b, s_a, s_b);
    if (threadIdx.x == 0) { out[0] = (float)(s0 * a); out[1] = (float)(s1 * b); }
}

// out[0] = w0 * sum0 / n0 + w1 * sum1 / n1 (the two regulariser means; an empty region contributes 0)
__global__ void __launch_bounds__(kFinThreads) k_refine_reg_finish(const double2* __restrict__ partials, int n, double w0, double n0,
                                                                   double w1, double n1, float* __restrict__ out) {
    __shared__ double s_a[kFinThreads], s_b[kFinThreads];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < n; i += kFinThreads) { a += partials[i].x; b += partials[i].y; }
    block_sum2<kFinThreads>(a, b, s_a, s_b);
    if (threadIdx.x == 0) out[0] = (float)((n0 > 0.0 ? w0 * a / n0 : 0.0) + (n1 > 0.0 ? w1 * b / n1 : 0.0));
}

// dL/dpred for L = g_bg bg_loss + g_l1 l1, in the op order of torch's autograd for
//   bg_loss = 1e-3 * (1 - pred * (1 - dilate)).sum()            -> (-(g_bg * 1e-3)) * (1 - dilate)
//   l1 = 1000 * L1Loss()(pred * m, gt * m) (mean over 3 S^2)    -> (((g_l1 * 1000) / N) * sign(pred m - gt m)) * m
__global__ void __launch_bounds__(256)
k_refine_image_grad(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ mask,
                    const float* __restrict__ dilated, uint32_t HW, int front, const float* __restrict__ g, float* __restrict__ dpred) {
    const uint32_t pix = blockIdx.x * 256 + threadIdx.x;
    if (pix >= HW) return;
    const float gb = -(g[0] * 1e-3f);
    const float keep = 1.0f - dilated[pix];
    const float gl = front ? (g[1] * 1000.0f) / (float)(3.0 * (double)HW) : 0.0f;
    const float m = front ? mask[pix] : 0.0f;
    #pragma unroll
    for (int c = 0; c < 3; c++) {
        const size_t i = (size_t)c * HW + pix;
        float v = gb * keep;
        if (front) {
            const float d = pred[i] * m - gt[i] * m;
            const float sgn = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f);
            v = v + (gl * sgn) * m;
        }
        dpred[i] = v;
    }
}

struct RegArgs {
    const float* origin;     // [P,3] colour origins (NULL: no regulariser)
    uint32_t p_cano, p_novel;
    float norm_cano, norm_novel;   // 2 / (3 p): MSELoss's mean gradient factor
    float w_cano, w_novel;
};

__global__ void __launch_bounds__(kAdamThreads)
k_refine_adam(const mi3d_adam_segment* __restrict__ segs, int n_segs, unsigned long long total, const mi3d_adam::Scalars a, RegArgs r,
              double2* __restrict__ partials) {
    __shared__ unsigned long long s_off[kMaxSegs + 1];
    __shared__ double s_a[kAdamThreads], s_b[kAdamThreads];
    for (int i = threadIdx.x; i < n_segs; i += kAdamThreads) s_off[i] = segs[i].offset;
    if (threadIdx.x == 0) s_off[n_segs] = total;
    __syncthreads();
    double rc = 0.0, rn = 0.0;
    const unsigned long long base = (unsigned long long)blockIdx.x * kAdamChunk;
    #pragma unroll 1
    for (int j = 0; j < kAdamPerThread; j++) {
        const unsigned long long e = base + (unsigned long long)j * kAdamThreads + threadIdx.x;
        if (e >= total) break;
        int lo = 0, hi = n_segs - 1;                 // last segment whose offset <= e
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (s_off[mid] <= e) lo = mid; else hi = mid - 1;
        }
        const mi3d_adam_segment& s = segs[lo];
        const unsigned long long i = e - s_off[lo];
        float p = s.param[i];
        float g = s.grad[i];
        if (lo == 0 && r.origin) {
            const uint32_t row = (uint32_t)(i / kCols), col = (uint32_t)(i % kCols);
            if (col < kColourCols) {
                const float diff = p - r.origin[(size_t)row * kColourCols + col];
                const bool cano = row < r.p_cano;
                g = g + (diff * (cano ? r.norm_cano : r.norm_novel)) * (cano ? r.w_cano : r.w_novel);
                const double sq = (double)diff * (double)diff;
                if (cano) rc += sq; else rn += sq;
            }
        }
        float m = s.exp_avg[i], v = s.exp_avg_sq[i];
        mi3d_adam::update(p, m, v, g, a);
        s.exp_avg[i] = m;
        s.exp_avg_sq[i] = v;
        s.param[i] = p;
    }
    if (partials) {
        block_sum2<kAdamThreads>(rc, rn, s_a, s_b);
        if (threadIdx.x == 0) partials[blockIdx.x] = make_double2(rc, rn);
    }
}

inline uint32_t image_blocks(uint32_t S) { const uint32_t t = mi3d_ceil_div(S, kTile); return t * t; }
inline size_t adam_blocks(unsigned long long total) { return (size_t)((total + kAdamChunk - 1) / kAdamChunk); }

}  // namespace

extern "C" {

size_t mi3d_refine_image_losses_workspace_bytes(uint32_t S) {
    if (S == 0 || S > 16384) return 0;
    return (size_t)image_blocks(S) * sizeof(double2);
}

int mi3d_refine_image_losses(const float* weights, uint32_t S, uint32_t ppp, const float* pred, const float* gt, const float* gt_mask,
                             int front, float* coverage, float* dilated, float* losses, void* workspace, size_t workspace_bytes,
                             mi3d_stream_t stream) {
    if (S == 0 || S > 16384 || ppp == 0 || ppp > 16 || !weights || !pred || !dilated || !losses || !workspace) return MI3D_ERR_ARG;
    if (front && (!gt || !gt_mask)) return MI3D_ERR_ARG;
    if (workspace_bytes < mi3d_refine_image_losses_workspace_bytes(S)) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const uint32_t t = mi3d_ceil_div(S, kTile);
    double2* partials = (double2*)workspace;
    k_refine_image_losses<<<dim3(t, t), dim3(kTile, kTile), 0, st>>>(weights, (int)S, (int)ppp, pred, gt, gt_mask, front ? 1 : 0, coverage,
                                                                     dilated, partials);
    k_refine_finish<<<1, kFinThreads, 0, st>>>(partials, (int)(t * t), 1e-3, 1000.0 / (3.0 * (double)S * (double)S), losses);
    MI3D_RETURN_LAUNCH();
}

int mi3d_refine_image_losses_backward(const float* pred, const float* gt, const float* gt_mask, const float* dilated, uint32_t S, int front,
                                      const float* grad_losses, float* grad_pred, mi3d_stream_t stream) {
    if (S == 0 || S > 16384 || !pred || !dilated || !grad_losses || !grad_pred) return MI3D_ERR_ARG;
    if (front && (!gt || !gt_mask)) return MI3D_ERR_ARG;
    const uint32_t HW = S * S;
    k_refine_image_grad<<<mi3d_ceil_div(HW, 256), 256, 0, (cudaStream_t)stream>>>(pred, gt, gt_mask, dilated, HW, front ? 1 : 0, grad_losses,
                                                                                  grad_pred);
    MI3D_RETURN_LAUNCH();
}

size_t mi3d_refine_adam_workspace_bytes(unsigned long long total) {
    if (total == 0 || adam_blocks(total) > 0x7fffffffull) return 0;
    return adam_blocks(total) * sizeof(double2);
}

int mi3d_refine_adam(const mi3d_adam_segment* segs, int n_segs, unsigned long long total, double lr, double beta1, double beta2, double eps,
                     int step, const float* origin, uint32_t p_cano, uint32_t p_novel, double w_cano, double w_novel, float* reg,
                     void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    if (!segs || n_segs < 1 || n_segs > kMaxSegs || total == 0 || step < 1) return MI3D_ERR_ARG;
    if (origin && (!reg || !workspace || workspace_bytes < mi3d_refine_adam_workspace_bytes(total))) return MI3D_ERR_ARG;
    const mi3d_adam::Scalars a = mi3d_adam::host_scalars(lr, beta1, beta2, eps, step);
    RegArgs r;
    r.origin = origin;
    r.p_cano = p_cano;
    r.p_novel = p_novel;
    r.norm_cano = p_cano ? (float)(2.0 / (3.0 * (double)p_cano)) : 0.0f;
    r.norm_novel = p_novel ? (float)(2.0 / (3.0 * (double)p_novel)) : 0.0f;
    r.w_cano = (float)w_cano;
    r.w_novel = (float)w_novel;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t blocks = adam_blocks(total);
    double2* partials = origin ? (double2*)workspace : nullptr;
    k_refine_adam<<<(unsigned)blocks, kAdamThreads, 0, st>>>(segs, n_segs, total, a, r, partials);
    if (origin)
        k_refine_reg_finish<<<1, kFinThreads, 0, st>>>(partials, (int)blocks, w_cano, 3.0 * (double)p_cano, w_novel, 3.0 * (double)p_novel,
                                                       reg);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
