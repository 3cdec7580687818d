// views.cu -- B5: the refine stage's point-cloud construction (load_views, reference nerf/refine_utils.py:61-152, :335-410), for
// sm_90a (C ABI: include/mi3d.h)
//
// The reference builds the two coloured clouds the refine stage optimises with numpy fp64 back-projection, OpenCV morphology and
// Canny, and CPU grid_sample.  These kernels reproduce that arithmetic so the selected points are the same points, in the same order:
//   * masks are uint8 images.  cv2.erode / cv2.dilate with a k x k rectangle use a +inf / -inf border, i.e. the window is clipped to
//     the image; they run as a horizontal then a vertical min / max pass over shared-memory tiles;
//   * Canny(img, t, t) has no weak pixels (low == high), so its output is the non-maximum-suppression survivors with L1 magnitude > t:
//     one fused pass over a shared-memory tile (replicated border for the 3x3 Sobel, zero magnitude outside the image, OpenCV's
//     fixed-point tan 22.5 test and its asymmetric > / >= neighbour comparisons);
//   * fp64 matrix products follow the order OpenBLAS' dgemm evaluates numpy's 3x3 products in: acc = a0 b0, acc = fma(a1, b1, acc),
//     acc = fma(a2, b2, acc), then the translation is added.  The file is compiled with -fmad=false, so every other op rounds once;
//   * grid_sample (bilinear, zeros, align_corners=False) follows ATen's vectorised CPU kernel: ix = fma(x + 1, W / 2, -0.5),
//     w = ix - floor(ix), e = 1 - w, corner weights s e, s w, n e, n w, and an fma chain over the corners nw, ne, sw, se;
//   * compaction keeps row-major pixel order: a flag pass with per-block counts, one scan of the block counts, an emit pass.
#include <limits.h>
#include <math.h>

#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kThreads = 256;              // flag / emit passes: one thread per pixel or point
constexpr int kMaxRadius = 15;             // morphology: k <= 31
constexpr int kRowSeg = 256;               // horizontal pass: outputs per block
constexpr int kColW = 32, kColH = 8;       // vertical pass: outputs per block
constexpr int kCannyT = 16;                // Canny: 16 x 16 outputs per block

// ---- morphology: separable min (erode) / max (dilate) over a window clipped to the image ----
template <bool kMax>
__device__ __forceinline__ uint8_t morph_op(uint8_t a, uint8_t b) { return kMax ? (a > b ? a : b) : (a < b ? a : b); }

template <bool kMax>
__global__ void __launch_bounds__(kRowSeg) k_morph_rows(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int H, int W, int r) {
    __shared__ uint8_t s[kRowSeg + 2 * kMaxRadius];
    const int y = blockIdx.y, x0 = blockIdx.x * kRowSeg;
    const uint8_t neutral = kMax ? 0 : 255;
    for (int t = threadIdx.x; t < kRowSeg + 2 * r; t += kRowSeg) {
        const int x = x0 - r + t;
        s[t] = (x >= 0 && x < W) ? src[(size_t)y * W + x] : neutral;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    if (x >= W) return;
    uint8_t v = s[threadIdx.x];
    for (int j = 1; j <= 2 * r; j++) v = morph_op<kMax>(v, s[threadIdx.x + j]);
    dst[(size_t)y * W + x] = v;
}

template <bool kMax>
__global__ void __launch_bounds__(kColW * kColH) k_morph_cols(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int H, int W, int r) {
    __shared__ uint8_t s[kColH + 2 * kMaxRadius][kColW];
    const int x = blockIdx.x * kColW + threadIdx.x, y0 = blockIdx.y * kColH;
    const uint8_t neutral = kMax ? 0 : 255;
    for (int t = threadIdx.y; t < kColH + 2 * r; t += kColH) {
        const int y = y0 - r + t;
        s[t][threadIdx.x] = (x < W && y >= 0 && y < H) ? src[(size_t)y * W + x] : neutral;
    }
    __syncthreads();
    const int y = y0 + threadIdx.y;
    if (x >= W || y >= H) return;
    uint8_t v = s[threadIdx.y][threadIdx.x];
    for (int j = 1; j <= 2 * r; j++) v = morph_op<kMax>(v, s[threadIdx.y + j][threadIdx.x]);
    dst[(size_t)y * W + x] = v;
}

// depth * mask * 255.0 cast to uint8 (refine_utils.py:386-387): fp64 product, truncation, then wrap modulo 256 as numpy's cast does on
// x86-64 (300.7 -> 44).  The depth is depth_u16 / 1000.0 (load_depth(...) / 1000.0).
__device__ __forceinline__ uint8_t depth_blur(const uint16_t* __restrict__ depth, const uint8_t* __restrict__ eroded, size_t i) {
    if (eroded[i] != 255) return 0;
    const double d = ((double)depth[i] / 1000.0) * 255.0;
    return (uint8_t)(unsigned)(long long)d;
}

// Canny(blur, t, t) (refine_utils.py:388): L1 magnitude of the 3x3 Sobel (replicated border), then OpenCV's non-maximum suppression
__global__ void __launch_bounds__(kCannyT * kCannyT)
k_canny(const uint16_t* __restrict__ depth, const uint8_t* __restrict__ eroded, int H, int W, int thresh, uint8_t* __restrict__ edges) {
    constexpr int TB = kCannyT + 4, TM = kCannyT + 2;
    __shared__ int16_t s_b[TB][TB];                 // blur at clamped coordinates (y0 - 2 .., x0 - 2 ..)
    __shared__ int s_m[TM][TM];                     // magnitude at (y0 - 1 .., x0 - 1 ..), 0 outside the image
    const int x0 = blockIdx.x * kCannyT, y0 = blockIdx.y * kCannyT;
    const int tid = threadIdx.y * kCannyT + threadIdx.x;
    for (int t = tid; t < TB * TB; t += kCannyT * kCannyT) {
        const int yy = min(max(y0 - 2 + t / TB, 0), H - 1), xx = min(max(x0 - 2 + t % TB, 0), W - 1);
        s_b[t / TB][t % TB] = depth_blur(depth, eroded, (size_t)yy * W + xx);
    }
    __syncthreads();
    // Sobel at tile position (a, b) of s_b (a, b >= 1): dx = right column - left column, dy = bottom row - top row, weights 1 2 1
    auto sobel = [&](int a, int b, int& dx, int& dy) {
        dx = (s_b[a - 1][b + 1] + 2 * s_b[a][b + 1] + s_b[a + 1][b + 1]) - (s_b[a - 1][b - 1] + 2 * s_b[a][b - 1] + s_b[a + 1][b - 1]);
        dy = (s_b[a + 1][b - 1] + 2 * s_b[a + 1][b] + s_b[a + 1][b + 1]) - (s_b[a - 1][b - 1] + 2 * s_b[a - 1][b] + s_b[a - 1][b + 1]);
    };
    for (int t = tid; t < TM * TM; t += kCannyT * kCannyT) {
        const int a = t / TM, b = t % TM, yy = y0 - 1 + a, xx = x0 - 1 + b;
        int m = 0;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            int dx, dy;
            sobel(a + 1, b + 1, dx, dy);
            m = abs(dx) + abs(dy);
        }
        s_m[a][b] = m;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= W || y >= H) return;
    const int a = threadIdx.y + 1, b = threadIdx.x + 1;
    const int m = s_m[a][b];
    bool edge = false;
    if (m > thresh) {
        int xs, ys;
        sobel(a + 1, b + 1, xs, ys);
        constexpr int kShift = 15;
        constexpr int kTg22 = 13573;                // (int)(tan(22.5 deg) * 2^15 + 0.5)
        const int ax = abs(xs), ay = abs(ys) << kShift;
        const int tg22x = ax * kTg22;
        if (ay < tg22x) {
            edge = m > s_m[a][b - 1] && m >= s_m[a][b + 1];
        } else {
            const int tg67x = tg22x + (ax << (kShift + 1));
            if (ay > tg67x) {
                edge = m > s_m[a - 1][b] && m >= s_m[a + 1][b];
            } else {
                const int sg = (xs ^ ys) < 0 ? -1 : 1;
                edge = m > s_m[a - 1][b - sg] && m > s_m[a + 1][b + sg];
            }
        }
    }
    edges[(size_t)y * W + x] = edge ? 255 : 0;
}

// out = (a == a_on) && (b != 255); optional masked depth float32(depth_u16 / 1000.0 * out) for the canonical occlusion test
__global__ void __launch_bounds__(kThreads)
k_mask_combine(const uint8_t* __restrict__ a, uint8_t a_on, const uint8_t* __restrict__ b, size_t n, uint8_t* __restrict__ out,
               const uint16_t* __restrict__ depth, float* __restrict__ masked_depth) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const bool m = a[i] == a_on && (b == nullptr || b[i] != 255);
    out[i] = m;
    if (masked_depth) masked_depth[i] = (float)(((double)depth[i] / 1000.0) * (m ? 1.0 : 0.0));
}

// canonical-cloud coverage (refine_utils.py:79-84): q = uint8(render * 255) (float32 product, truncation); mask / 255 > 0.9, kept as
// 255 / 0 so the 15 x 15 erosion of the thresholded image equals the threshold of the eroded one
__global__ void __launch_bounds__(kThreads)
k_cover_threshold(const float* __restrict__ render, size_t n, uint8_t* __restrict__ quant, uint8_t* __restrict__ t) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const uint8_t q = (uint8_t)(unsigned)(render[i] * 255.0f);
    if (quant) quant[i] = q;
    t[i] = ((double)q / 255.0 > 0.9) ? 255 : 0;
}

// ---- fp64 geometry in OpenBLAS' dgemm order ----
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
    return fma(a2, b2, fma(a1, b1, a0 * b0));
}

// refine_utils.py:154-158 project(): c = xyz RT[:, :3]^T + RT[:, 3], q = c K^T; returns (u, v) = q.xy / q.z and z = q.z
__device__ __forceinline__ void project(double x, double y, double z, const double* __restrict__ k, const double* __restrict__ rt, double& u,
                                        double& v, double& w) {
    double c[3], q[3];
    #pragma unroll
    for (int r = 0; r < 3; r++) c[r] = dot3(x, y, z, rt[4 * r], rt[4 * r + 1], rt[4 * r + 2]) + rt[4 * r + 3];
    #pragma unroll
    for (int r = 0; r < 3; r++) q[r] = dot3(c[0], c[1], c[2], k[3 * r], k[3 * r + 1], k[3 * r + 2]);
    u = q[0] / q[2];
    v = q[1] / q[2];
    w = q[2];
}

// world point of pixel (x, y) at depth depth_u16 / 1000 (refine_utils.py:87-99, :131-139): inv(K) [x, y, 1] * D, then v c2w[:3,:3]^T +
// c2w[:3, 3]
__device__ __forceinline__ void backproject(int x, int y, uint16_t d16, const double* __restrict__ kinv, const double* __restrict__ c2w,
                                            double p[3]) {
    const double D = (double)d16 / 1000.0;
    double v[3];
    #pragma unroll
    for (int r = 0; r < 3; r++) v[r] = dot3((double)x, (double)y, 1.0, kinv[3 * r], kinv[3 * r + 1], kinv[3 * r + 2]) * D;
    #pragma unroll
    for (int r = 0; r < 3; r++) p[r] = dot3(v[0], v[1], v[2], c2w[4 * r], c2w[4 * r + 1], c2w[4 * r + 2]) + c2w[4 * r + 3];
}

// ndarray.astype(np.int32) of a rounded double as x86-64 computes it (cvttsd2si): out of range or NaN -> INT_MIN
__device__ __forceinline__ int to_i32(double r) { return fabs(r) < 2147483648.0 ? (int)r : INT_MIN; }

// grid_sample of C interleaved channels of img [H,W,C] at normalised (gx, gy) (ATen's vectorised CPU arithmetic, see the top).
// The image is float32, or uint8 read as float32(u8 / 255.0) (imageio.imread(...) / 255. held in a float32 tensor).
__device__ __forceinline__ float texel(const float* __restrict__ f, const uint8_t* __restrict__ u8, size_t i) {
    return f ? f[i] : (float)((double)u8[i] / 255.0);
}

__device__ __forceinline__ void grid_sample(const float* __restrict__ f, const uint8_t* __restrict__ u8, int H, int W, int C, float gx,
                                            float gy, float* out) {
    const float ix = fmaf(gx + 1.0f, (float)W / 2.0f, -0.5f), iy = fmaf(gy + 1.0f, (float)H / 2.0f, -0.5f);
    const float xw = floorf(ix), yn = floorf(iy);
    const float w = ix - xw, e = 1.0f - w, n = iy - yn, s = 1.0f - n;
    const float wt[4] = {s * e, s * w, n * e, n * w};
    const float cx[4] = {xw, xw + 1.0f, xw, xw + 1.0f}, cy[4] = {yn, yn, yn + 1.0f, yn + 1.0f};
    size_t off[4];
    bool in[4];
    #pragma unroll
    for (int k = 0; k < 4; k++) {
        in[k] = cx[k] > -1.0f && cx[k] < (float)W && cy[k] > -1.0f && cy[k] < (float)H;
        off[k] = in[k] ? ((size_t)(int)cy[k] * W + (size_t)(int)cx[k]) * C : 0;
    }
    for (int c = 0; c < C; c++) {
        float acc = (in[0] ? texel(f, u8, off[0] + c) : 0.0f) * wt[0];
        #pragma unroll
        for (int k = 1; k < 4; k++) acc = fmaf(in[k] ? texel(f, u8, off[k] + c) : 0.0f, wt[k], acc);
        out[c] = acc;
    }
}

// torch.Tensor(xy) / H * 2. - 1. in float32
__device__ __forceinline__ float to_grid(float a, int S) { return (a / (float)S) * 2.0f - 1.0f; }

// ---- order-preserving compaction ----
// exclusive rank of this thread's flag among its block's flags; *total = the block's count (all threads of the block must call)
__device__ __forceinline__ uint32_t block_rank(bool flag, uint32_t* total) {
    __shared__ uint32_t s_warp[kThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t ballot = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[wid] = __popc(ballot);
    __syncthreads();
    uint32_t before = 0, tot = 0;
    #pragma unroll
    for (int k = 0; k < kThreads / 32; k++) {
        const uint32_t c = s_warp[k];
        before += k < wid ? c : 0u;
        tot += c;
    }
    __syncthreads();
    *total = tot;
    return before + __popc(ballot & ((1u << lane) - 1u));
}

// exclusive scan of n block counters by one CTA of 1024 threads: off[t] = sum of cnt[< t]; *count = the total
__global__ void __launch_bounds__(1024) k_scan_blocks(const uint32_t* __restrict__ cnt, int n, uint32_t* __restrict__ off, int* __restrict__ count) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int t = base + threadIdx.x;
        const uint32_t v = t < n ? cnt[t] : 0u;
        uint32_t inc = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
        if (lane == 31) warp_tot[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            const uint32_t w = warp_tot[lane];
            uint32_t wi = w;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += u; }
            warp_tot[lane] = wi - w;
        }
        __syncthreads();
        const uint32_t ex = carry_s + warp_tot[wid] + inc - v;
        if (t < n) off[t] = ex;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = ex + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = (int)carry_s;
}

// flag pass of the back-projection: keep = mask, and (with a canonical depth) not hidden-or-duplicated in the canonical view
// (refine_utils.py:100-107): project into the canonical camera, np.round, grid_sample the masked canonical depth d, drop the point when
// -0.2 <= z - d <= 1/H (fp64 z minus float32 d)
__global__ void __launch_bounds__(kThreads)
k_bp_flag(const uint16_t* __restrict__ depth, const uint8_t* __restrict__ mask, int H, int W, const double* __restrict__ kinv,
          const double* __restrict__ c2w, const double* __restrict__ k, const double* __restrict__ cano_w2c, const float* __restrict__ cano_depth,
          uint8_t* __restrict__ flags, uint32_t* __restrict__ block_cnt) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const size_t n = (size_t)H * W;
    bool keep = i < n && mask[i] != 0;
    if (keep && cano_depth) {
        double p[3], u, v, z;
        backproject((int)(i % W), (int)(i / W), depth[i], kinv, c2w, p);
        project(p[0], p[1], p[2], k, cano_w2c, u, v, z);
        const float gx = to_grid((float)to_i32(rint(u)), H), gy = to_grid((float)to_i32(rint(v)), H);
        float d;
        grid_sample(cano_depth, nullptr, H, W, 1, gx, gy, &d);
        const double diff = z - (double)d;
        keep = !(diff <= 1.0 / (double)H && diff >= -0.2);
    }
    if (i < n) flags[i] = keep;
    uint32_t tot;
    block_rank(keep, &tot);
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = tot;
}

// emit pass: the kept points in pixel order; rows [count, H*W) are filled with NaN, which z_buffer treats as off-image
__global__ void __launch_bounds__(kThreads)
k_bp_emit(const uint16_t* __restrict__ depth, int H, int W, const double* __restrict__ kinv, const double* __restrict__ c2w,
          const uint8_t* __restrict__ flags, const uint32_t* __restrict__ block_off, const int* __restrict__ count, double* __restrict__ points) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const size_t n = (size_t)H * W;
    const bool keep = i < n && flags[i];
    uint32_t tot;
    const uint32_t r = block_rank(keep, &tot);
    if (keep) {
        double p[3];
        backproject((int)(i % W), (int)(i / W), depth[i], kinv, c2w, p);
        double* o = points + 3 * (size_t)(block_off[blockIdx.x] + r);
        o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
    }
    if (i < n && i >= (size_t)*count) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        points[3 * i] = nan; points[3 * i + 1] = nan; points[3 * i + 2] = nan;
    }
}

__global__ void __launch_bounds__(kThreads) k_flag_count(const uint8_t* __restrict__ keep, uint32_t P, uint32_t* __restrict__ block_cnt) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    uint32_t tot;
    block_rank(i < P && keep[i], &tot);
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = tot;
}

// v = v[keep]; colour = grid_sample(img, project(v, K, w2c) / H * 2 - 1) (refine_utils.py:109-114, :144-151)
__global__ void __launch_bounds__(kThreads)
k_compact_colour(const double* __restrict__ points, uint32_t P, const uint8_t* __restrict__ keep, const double* __restrict__ k,
                 const double* __restrict__ w2c, const float* __restrict__ img_f32, const uint8_t* __restrict__ img_u8, int H, int W,
                 const uint32_t* __restrict__ block_off, double* __restrict__ points_out, float* __restrict__ colours) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    const bool kp = i < P && keep[i];
    uint32_t tot;
    const uint32_t r = block_rank(kp, &tot);
    if (!kp) return;
    const double x = points[3 * (size_t)i], y = points[3 * (size_t)i + 1], z = points[3 * (size_t)i + 2];
    double u, v, w;
    project(x, y, z, k, w2c, u, v, w);
    float c[3];
    grid_sample(img_f32, img_u8, H, W, 3, to_grid((float)u, H), to_grid((float)v, H), c);
    const size_t o = block_off[blockIdx.x] + r;
    points_out[3 * o] = x; points_out[3 * o + 1] = y; points_out[3 * o + 2] = z;
    colours[3 * o] = c[0]; colours[3 * o + 1] = c[1]; colours[3 * o + 2] = c[2];
}

struct ViewsWs {
    uint8_t *t0, *t1, *t2, *t3;            // H*W each: morphology / Canny scratch, then the compaction flags (t0)
    uint32_t *block_cnt, *block_off;
    size_t bytes;
};

bool carve(void* base, uint32_t H, uint32_t W, ViewsWs* ws) {
    if (H == 0 || W == 0 || H != W || H > 16384) return false;
    const size_t n = (size_t)H * W, nb = mi3d_ceil_div((uint32_t)n, kThreads);
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    char* p = (char*)base;
    size_t o = 0;
    ws->t0 = (uint8_t*)(p + o); o += al(n);
    ws->t1 = (uint8_t*)(p + o); o += al(n);
    ws->t2 = (uint8_t*)(p + o); o += al(n);
    ws->t3 = (uint8_t*)(p + o); o += al(n);
    ws->block_cnt = (uint32_t*)(p + o); o += al(nb * 4);
    ws->block_off = (uint32_t*)(p + o); o += al(nb * 4);
    ws->bytes = o;
    return true;
}

template <bool kMax>
void morph(const uint8_t* src, uint8_t* tmp, uint8_t* dst, int H, int W, int r, cudaStream_t st) {
    k_morph_rows<kMax><<<dim3(mi3d_ceil_div(W, kRowSeg), H), kRowSeg, 0, st>>>(src, tmp, H, W, r);
    k_morph_cols<kMax><<<dim3(mi3d_ceil_div(W, kColW), mi3d_ceil_div(H, kColH)), dim3(kColW, kColH), 0, st>>>(tmp, dst, H, W, r);
}

bool odd_k(uint32_t k) { return (k & 1u) && k <= 2 * kMaxRadius + 1; }

}  // namespace

extern "C" {

size_t mi3d_views_workspace_bytes(uint32_t H, uint32_t W) {
    ViewsWs ws;
    return carve(nullptr, H, W, &ws) ? ws.bytes : 0;
}

int mi3d_views_mask(const uint16_t* depth, const uint8_t* mask, uint32_t H, uint32_t W, uint32_t erode_k, int canny_thresh, uint32_t dilate_k,
                    uint8_t* out, float* masked_depth, uint8_t* eroded, uint8_t* edges, uint8_t* dilated, void* workspace,
                    size_t workspace_bytes, mi3d_stream_t stream) {
    ViewsWs ws;
    if (!depth || !mask || !out || !workspace || !odd_k(erode_k) || (canny_thresh >= 0 && !odd_k(dilate_k)) || !carve(workspace, H, W, &ws) ||
        ws.bytes > workspace_bytes)
        return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int h = (int)H, w = (int)W;
    const size_t n = (size_t)H * W;
    uint8_t* er = eroded ? eroded : ws.t1;
    morph<false>(mask, ws.t0, er, h, w, (int)erode_k / 2, st);
    const uint8_t* dl = nullptr;
    if (canny_thresh >= 0) {
        uint8_t* ed = edges ? edges : ws.t2;
        k_canny<<<dim3(mi3d_ceil_div(W, kCannyT), mi3d_ceil_div(H, kCannyT)), dim3(kCannyT, kCannyT), 0, st>>>(depth, er, h, w, canny_thresh, ed);
        uint8_t* dd = dilated ? dilated : ws.t3;
        morph<true>(ed, ws.t0, dd, h, w, (int)dilate_k / 2, st);
        dl = dd;
    }
    k_mask_combine<<<mi3d_ceil_div((uint32_t)n, kThreads), kThreads, 0, st>>>(er, 255, dl, n, out, depth, masked_depth);
    MI3D_RETURN_LAUNCH();
}

int mi3d_views_cover_mask(const float* render, const uint8_t* alphamask, uint32_t H, uint32_t W, uint32_t erode_k, uint8_t* out, uint8_t* quant,
                          void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    ViewsWs ws;
    if (!render || !alphamask || !out || !workspace || !odd_k(erode_k) || !carve(workspace, H, W, &ws) || ws.bytes > workspace_bytes)
        return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)H * W;
    const unsigned blocks = mi3d_ceil_div((uint32_t)n, kThreads);
    k_cover_threshold<<<blocks, kThreads, 0, st>>>(render, n, quant, ws.t1);
    morph<false>(ws.t1, ws.t0, ws.t2, (int)H, (int)W, (int)erode_k / 2, st);
    k_mask_combine<<<blocks, kThreads, 0, st>>>(alphamask, 1, ws.t2, n, out, nullptr, nullptr);
    MI3D_RETURN_LAUNCH();
}

int mi3d_views_backproject(const uint16_t* depth, const uint8_t* mask, uint32_t H, uint32_t W, const double* kinv, const double* c2w,
                           const double* cam_k, const double* cano_w2c, const float* cano_depth, double* points, int* count, void* workspace,
                           size_t workspace_bytes, mi3d_stream_t stream) {
    ViewsWs ws;
    if (!depth || !mask || !kinv || !c2w || !points || !count || !workspace || !carve(workspace, H, W, &ws) || ws.bytes > workspace_bytes)
        return MI3D_ERR_ARG;
    if (cano_depth && (!cam_k || !cano_w2c)) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const uint32_t n = H * W, nb = mi3d_ceil_div(n, kThreads);
    k_bp_flag<<<nb, kThreads, 0, st>>>(depth, mask, (int)H, (int)W, kinv, c2w, cam_k, cano_w2c, cano_depth, ws.t0, ws.block_cnt);
    k_scan_blocks<<<1, 1024, 0, st>>>(ws.block_cnt, (int)nb, ws.block_off, count);
    k_bp_emit<<<nb, kThreads, 0, st>>>(depth, (int)H, (int)W, kinv, c2w, ws.t0, ws.block_off, count, points);
    MI3D_RETURN_LAUNCH();
}

int mi3d_views_compact_colour(const double* points, uint32_t P, const uint8_t* keep, const double* cam_k, const double* world2cam,
                              const float* img_f32, const uint8_t* img_u8, uint32_t H, uint32_t W, double* points_out, float* colours,
                              int* count, void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    ViewsWs ws;
    if (!keep || !cam_k || !world2cam || (!img_f32 == !img_u8) || !points_out || !colours || !count || !workspace ||
        !carve(workspace, H, W, &ws) || ws.bytes > workspace_bytes || P > H * W || (P > 0 && !points))
        return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (P == 0) {
        MI3D_CHECK(cudaMemsetAsync(count, 0, sizeof(int), st));
        return MI3D_OK;
    }
    const uint32_t nb = mi3d_ceil_div(P, kThreads);
    k_flag_count<<<nb, kThreads, 0, st>>>(keep, P, ws.block_cnt);
    k_scan_blocks<<<1, 1024, 0, st>>>(ws.block_cnt, (int)nb, ws.block_off, count);
    k_compact_colour<<<nb, kThreads, 0, st>>>(points, P, keep, cam_k, world2cam, img_f32, img_u8, (int)H, (int)W, ws.block_off, points_out,
                                              colours);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
