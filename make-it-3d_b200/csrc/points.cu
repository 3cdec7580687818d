// points.cu -- B5: the refine stage's point-splat renderer and z-buffer visibility, for sm_90a (C ABI: include/mi3d.h)
//
// Replaces pytorch3d's rasterize_points + alpha_composite as nerf/refine_utils.py:306-333 (render_point) drives them, and the
// per-point Python loop of z_buffer (refine_utils.py:167-208).  Compiled with -fmad=false: every fp32 / fp64 op rounds once, in the
// order oracle/points_ref.py restates, so the selected points and their distances are bit-identical to the CPU oracle.
//
// Forward (no host synchronisation, no atomics on anything that reaches an output):
//   1. k_points_bin_count   per point: project (R p + t, then K), cull z < 0 / non-finite, and count the 16x16 screen tiles its
//                           pixel footprint (the exact coverage range widened by one pixel) touches -> per-tile counters
//   2. k_points_tile_scan   one CTA: exclusive scan of the tile counters -> list offsets (and the emit cursors)
//   3. k_points_bin_emit    per point: append its id to every touched tile's list (order inside a list is arbitrary)
//   4. k_points_raster      one CTA per tile, one thread per pixel: streams the tile's list through shared memory, keeps the K
//                           covering points with the smallest (z, index) in registers, then writes idx / w (saved for the
//                           backward), optional zbuf / dist2 and the alpha-composited image.  The total order (z, index) makes
//                           the result independent of the list order.
// Backward: k_points_feat_grad is a gather, one thread per point: it re-projects the point, walks the same pixel footprint and
// finds itself among each pixel's K slots; dfeat[p][c] = sum g[c,pix] * w.  No atomics: bit-identical from run to run.
//
// Workspace: the list capacity is P x (a host-side bound on the tiles one footprint can touch), so it cannot overflow and no
// device count is ever read back.
#include <limits.h>
#include <math.h>

#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kTile = 16;                  // screen tile edge (pixels); one raster CTA = kTile x kTile threads
constexpr int kPtThreads = 256;
constexpr int kMaxK = 16;                  // points per pixel
constexpr int kMaxC = 32;                  // feature channels

// fused projection of refine_utils.py:307-315 in its op order: c = R p + t, q = K c, u = q.x / q.z, px = -(u / W * 2 - 1)
__device__ __forceinline__ float3 project_ndc(const float* __restrict__ cam_k, const float* __restrict__ w2c, const float* __restrict__ pts,
                                              uint32_t i, float proj_w, float proj_h) {
    const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    float c[3], q[3];
    #pragma unroll
    for (int r = 0; r < 3; r++) c[r] = ((w2c[4 * r] * x + w2c[4 * r + 1] * y) + w2c[4 * r + 2] * z) + w2c[4 * r + 3];
    #pragma unroll
    for (int r = 0; r < 3; r++) q[r] = (cam_k[3 * r] * c[0] + cam_k[3 * r + 1] * c[1]) + cam_k[3 * r + 2] * c[2];
    const float u = q[0] / q[2], v = q[1] / q[2];
    return make_float3(-((u / proj_w) * 2.0f - 1.0f), -((v / proj_h) * 2.0f - 1.0f), q[2]);
}

// Pixel range [lo, hi] (inclusive, clamped to the image) along one axis that a point at NDC coordinate `p` may cover: pixel i has
// centre 1 - (2i + 1) / S, so |centre - p| < r holds only for i in ((S (1 - p - r) - 1) / 2, (S (1 - p + r) - 1) / 2); one pixel of
// margin on each side absorbs the rounding of this estimate.  Returns false when the range misses the image.
__device__ __forceinline__ bool axis_range(float p, float r, int S, int& lo, int& hi) {
    const float a = ((float)S * (1.0f - p - r) - 1.0f) * 0.5f;
    const float b = ((float)S * (1.0f - p + r) - 1.0f) * 0.5f;
    const float flo = floorf(a) - 1.0f, fhi = ceilf(b) + 1.0f;
    if (!(fhi >= 0.0f) || !(flo <= (float)(S - 1))) return false;        // also rejects NaN
    lo = (int)fmaxf(flo, 0.0f);
    hi = (int)fminf(fhi, (float)(S - 1));
    return true;
}

// footprint of a projected point (culled: z < 0 or non-finite x / y -> empty)
__device__ __forceinline__ bool footprint(float3 q, float r, int S, int& x0, int& x1, int& y0, int& y1) {
    if (q.z < 0.0f || !isfinite(q.x) || !isfinite(q.y)) return false;
    return axis_range(q.x, r, S, x0, x1) && axis_range(q.y, r, S, y0, y1);
}

__global__ void __launch_bounds__(kPtThreads)
k_points_bin_count(const float* __restrict__ pts, uint32_t P, const float* __restrict__ cam_k, const float* __restrict__ w2c, float proj_w,
                   float proj_h, int S, float r, int n_tx, float4* __restrict__ proj, uint32_t* __restrict__ tile_cnt) {
    const uint32_t i = blockIdx.x * kPtThreads + threadIdx.x;
    if (i >= P) return;
    const float3 q = project_ndc(cam_k, w2c, pts, i, proj_w, proj_h);
    proj[i] = make_float4(q.x, q.y, q.z, 0.0f);
    int x0, x1, y0, y1;
    if (!footprint(q, r, S, x0, x1, y0, y1)) return;
    for (int ty = y0 / kTile; ty <= y1 / kTile; ty++)
        for (int tx = x0 / kTile; tx <= x1 / kTile; tx++) atomicAdd(&tile_cnt[ty * n_tx + tx], 1u);
}

// exclusive scan of n tile counters by one CTA of 1024 threads: off[t] (and cursor[t]) = sum of cnt[< t]
__global__ void __launch_bounds__(1024) k_points_tile_scan(const uint32_t* __restrict__ cnt, int n, uint32_t* __restrict__ off,
                                                          uint32_t* __restrict__ cursor) {
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
            uint32_t w = warp_tot[lane], wi = w;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += u; }
            warp_tot[lane] = wi - w;            // exclusive prefix of the warps
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        const uint32_t ex = carry + warp_tot[wid] + inc - v;
        if (t < n) { off[t] = ex; cursor[t] = ex; }
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = ex + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) off[n] = carry_s;
}

__global__ void __launch_bounds__(kPtThreads)
k_points_bin_emit(const float4* __restrict__ proj, uint32_t P, int S, float r, int n_tx, uint32_t* __restrict__ cursor,
                  uint32_t* __restrict__ list) {
    const uint32_t i = blockIdx.x * kPtThreads + threadIdx.x;
    if (i >= P) return;
    const float4 p4 = proj[i];
    int x0, x1, y0, y1;
    if (!footprint(make_float3(p4.x, p4.y, p4.z), r, S, x0, x1, y0, y1)) return;
    for (int ty = y0 / kTile; ty <= y1 / kTile; ty++)
        for (int tx = x0 / kTile; tx <= x1 / kTile; tx++) list[atomicAdd(&cursor[ty * n_tx + tx], 1u)] = i;
}

__device__ __forceinline__ bool zi_less(float za, int ia, float zb, int ib) { return za < zb || (za == zb && ia < ib); }

template <int KM>
__global__ void __launch_bounds__(kTile * kTile)
k_points_raster(const float4* __restrict__ proj, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ list, int S, int n_tx,
                float r, float r2_alpha, int K, const float* __restrict__ feats, int C, float* __restrict__ image, int* __restrict__ idx_out,
                float* __restrict__ w_out, float* __restrict__ zbuf_out, float* __restrict__ dist2_out) {
    __shared__ float4 s_pt[kTile * kTile];
    __shared__ int s_id[kTile * kTile];
    const int tid = threadIdx.y * kTile + threadIdx.x;
    const int tile = blockIdx.x, tx = tile % n_tx, ty = tile / n_tx;
    const int xi = tx * kTile + threadIdx.x, yi = ty * kTile + threadIdx.y;
    const bool inside = xi < S && yi < S;
    // pixel centre in NDC, evaluated in double and rounded once (+X points left, +Y up: pytorch3d's convention)
    const float xf = (float)(-1.0 + (2.0 * (double)(S - 1 - xi) + 1.0) / (double)S);
    const float yf = (float)(-1.0 + (2.0 * (double)(S - 1 - yi) + 1.0) / (double)S);
    const float rr = r * r;

    float zs[KM], ds[KM];
    int ids[KM];
    #pragma unroll
    for (int k = 0; k < KM; k++) { zs[k] = INFINITY; ids[k] = INT_MAX; ds[k] = -1.0f; }
    float zw = INFINITY;       // (zw, iw) = the K-th best so far: a candidate must beat it
    int iw = INT_MAX;

    const uint32_t beg = tile_off[tile], end = tile_off[tile + 1];
    for (uint32_t base = beg; base < end; base += kTile * kTile) {
        const uint32_t n = min(end - base, (uint32_t)(kTile * kTile));
        __syncthreads();
        if ((uint32_t)tid < n) { const int id = (int)list[base + tid]; s_id[tid] = id; s_pt[tid] = proj[id]; }
        __syncthreads();
        if (!inside) continue;
        for (uint32_t j = 0; j < n; j++) {
            const float4 p = s_pt[j];
            const float dx = xf - p.x, dy = yf - p.y;
            const float d2 = dx * dx + dy * dy;
            if (!(d2 < rr)) continue;
            const int id = s_id[j];
            if (!zi_less(p.z, id, zw, iw)) continue;
            float cz = p.z, cd = d2;
            int ci = id;
            #pragma unroll
            for (int k = 0; k < KM; k++) {
                if (k < K && zi_less(cz, ci, zs[k], ids[k])) {
                    const float tz = zs[k], td = ds[k];
                    const int ti = ids[k];
                    zs[k] = cz; ds[k] = cd; ids[k] = ci;
                    cz = tz; cd = td; ci = ti;
                }
            }
            #pragma unroll
            for (int k = 0; k < KM; k++) if (k == K - 1) { zw = zs[k]; iw = ids[k]; }
        }
    }
    if (!inside) return;

    // alpha = 1 - sqrt(clamp(0.1 * dist2 / r^2, 1e-3, 1)) (refine_utils.py:320-325); composite front to back (alpha_composite):
    // w_k = T alpha_k, T *= 1 - alpha_k, empty slots skipped
    const size_t pix = (size_t)yi * S + xi;
    float ws[KM];
    float T = 1.0f;
    #pragma unroll
    for (int k = 0; k < KM; k++) {
        ws[k] = 0.0f;
        if (k < K) {
            const bool full = ids[k] != INT_MAX;
            if (full) {
                const float a = 1.0f - sqrtf(fminf(fmaxf((0.1f * ds[k]) / r2_alpha, 1e-3f), 1.0f));
                ws[k] = T * a;
                T = T * (1.0f - a);
            }
            idx_out[pix * K + k] = full ? ids[k] : -1;
            if (w_out) w_out[pix * K + k] = ws[k];
            if (zbuf_out) zbuf_out[pix * K + k] = full ? zs[k] : -1.0f;
            if (dist2_out) dist2_out[pix * K + k] = full ? ds[k] : -1.0f;
        }
    }
    if (!image) return;
    const size_t HW = (size_t)S * S;
    for (int c = 0; c < C; c++) {
        float acc = 0.0f;
        #pragma unroll
        for (int k = 0; k < KM; k++)
            if (k < K && ids[k] != INT_MAX) acc = acc + ws[k] * feats[(size_t)ids[k] * C + c];
        image[c * HW + pix] = acc;
    }
}

// dfeat[p][c] = sum over (pixel, slot) holding p of g[c, pixel] * w; one thread per point walks its footprint (no atomics)
__global__ void __launch_bounds__(kPtThreads)
k_points_feat_grad(const float* __restrict__ pts, uint32_t P, const float* __restrict__ cam_k, const float* __restrict__ w2c, float proj_w,
                   float proj_h, int S, float r, int K, const int* __restrict__ idx, const float* __restrict__ w, const float* __restrict__ g,
                   int C, float* __restrict__ dfeat) {
    const uint32_t i = blockIdx.x * kPtThreads + threadIdx.x;
    if (i >= P) return;
    float acc[kMaxC];
    #pragma unroll
    for (int c = 0; c < kMaxC; c++) acc[c] = 0.0f;
    const float3 q = project_ndc(cam_k, w2c, pts, i, proj_w, proj_h);
    int x0, x1, y0, y1;
    if (footprint(q, r, S, x0, x1, y0, y1)) {
        const size_t HW = (size_t)S * S;
        for (int y = y0; y <= y1; y++)
            for (int x = x0; x <= x1; x++) {
                const size_t pix = (size_t)y * S + x;
                for (int k = 0; k < K; k++) {
                    const int id = idx[pix * K + k];
                    if (id < 0) break;
                    if (id != (int)i) continue;
                    const float wk = w[pix * K + k];
                    #pragma unroll
                    for (int c = 0; c < kMaxC; c++) if (c < C) acc[c] = acc[c] + g[c * HW + pix] * wk;
                    break;
                }
            }
    }
    #pragma unroll
    for (int c = 0; c < kMaxC; c++) if (c < C) dfeat[(size_t)i * C + c] = acc[c];
}

// ---- z_buffer (fp64): order-preserving uint64 key of a double, so atomicMin on the key is a min on the value ----
__device__ __forceinline__ unsigned long long dkey(double d) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// refine_utils.py:154-158 project() in double: c = R p + t, q = K c, (u, v) = q.xy / q.z; returns false when rint(u, v) is off-image
__device__ __forceinline__ bool zb_project(const double* __restrict__ pts, uint32_t i, const double* __restrict__ cam_k,
                                           const double* __restrict__ w2c, int H, int W, double& z, int& pix) {
    const double x = pts[3 * i], y = pts[3 * i + 1], zz = pts[3 * i + 2];
    double c[3], q[3];
    #pragma unroll
    for (int r = 0; r < 3; r++) c[r] = ((w2c[4 * r] * x + w2c[4 * r + 1] * y) + w2c[4 * r + 2] * zz) + w2c[4 * r + 3];
    #pragma unroll
    for (int r = 0; r < 3; r++) q[r] = (cam_k[3 * r] * c[0] + cam_k[3 * r + 1] * c[1]) + cam_k[3 * r + 2] * c[2];
    const double u = rint(q[0] / q[2]), v = rint(q[1] / q[2]);     // np.round: half to even
    z = q[2];
    if (!(u >= 0.0 && u <= (double)(W - 1) && v >= 0.0 && v <= (double)(H - 1))) return false;
    pix = (int)v * W + (int)u;
    return true;
}

__global__ void __launch_bounds__(kPtThreads)
k_zbuffer_min(const double* __restrict__ pts, uint32_t P, const double* __restrict__ cam_k, const double* __restrict__ w2c, int H, int W,
              unsigned long long* __restrict__ zbuf) {
    const uint32_t i = blockIdx.x * kPtThreads + threadIdx.x;
    if (i >= P) return;
    double z;
    int pix;
    if (zb_project(pts, i, cam_k, w2c, H, W, z, pix)) atomicMin(&zbuf[pix], dkey(z));
}

__global__ void __launch_bounds__(kPtThreads)
k_zbuffer_mask(const double* __restrict__ pts, uint32_t P, const double* __restrict__ cam_k, const double* __restrict__ w2c, int H, int W,
               const unsigned long long* __restrict__ zbuf, uint8_t* __restrict__ mask) {
    const uint32_t i = blockIdx.x * kPtThreads + threadIdx.x;
    if (i >= P) return;
    double z;
    int pix;
    const bool in = zb_project(pts, i, cam_k, w2c, H, W, z, pix);
    mask[i] = in && !((z - dkey_inv(zbuf[pix])) > 1.0 / (double)H);
}

struct PointsWs {
    float4* proj;
    uint32_t *tile_cnt, *tile_off, *cursor, *list;
    size_t bytes;
};

// tiles one footprint can touch along an axis: the footprint spans at most S r + 5 pixels (axis_range), plus slack
uint32_t tiles_per_point(uint32_t S, double radius) {
    const double px = (double)S * radius + 6.0;
    const uint32_t n_t = mi3d_ceil_div(S, kTile);
    const double t = floor(px / kTile) + 2.0;
    const uint32_t ta = t >= (double)n_t ? n_t : (uint32_t)t;
    return ta * ta;
}

bool carve(void* base, uint32_t P, uint32_t S, double radius, PointsWs* ws) {
    const uint32_t n_t = mi3d_ceil_div(S, kTile), n_tiles = n_t * n_t;
    const uint64_t cap = (uint64_t)P * tiles_per_point(S, radius);
    if (cap >= 0x80000000ull) return false;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    char* p = (char*)base;
    size_t o = 0;
    ws->proj = (float4*)(p + o); o += al((size_t)P * sizeof(float4));
    ws->tile_cnt = (uint32_t*)(p + o); o += al((size_t)n_tiles * 4);
    ws->tile_off = (uint32_t*)(p + o); o += al((size_t)(n_tiles + 1) * 4);
    ws->cursor = (uint32_t*)(p + o); o += al((size_t)n_tiles * 4);
    ws->list = (uint32_t*)(p + o); o += al((size_t)cap * 4);
    ws->bytes = o;
    return true;
}

bool valid_args(uint32_t P, uint32_t H, uint32_t W, double radius, uint32_t K, uint32_t C) {
    return P > 0 && P < 0x80000000u && H == W && H > 0 && H <= 16384 && radius > 0.0 && isfinite(radius) && K >= 1 && K <= kMaxK &&
           C >= 1 && C <= kMaxC;
}

}  // namespace

extern "C" {

size_t mi3d_points_workspace_bytes(uint32_t P, uint32_t H, uint32_t W, double radius) {
    PointsWs ws;
    if (!valid_args(P, H, W, radius, 1, 1) || !carve(nullptr, P, H, radius, &ws)) return 0;
    return ws.bytes;
}

int mi3d_points_render_forward(const float* points, const float* feats, uint32_t P, uint32_t C, const float* cam_k, const float* world2cam,
                               float proj_w, float proj_h, uint32_t H, uint32_t W, double radius, uint32_t K, float* image, int* idx,
                               float* w, float* zbuf, float* dist2, void* workspace, size_t workspace_bytes, mi3d_stream_t stream) {
    if (!valid_args(P, H, W, radius, K, image ? C : 1) || !points || !cam_k || !world2cam || !idx || !workspace) return MI3D_ERR_ARG;
    if (image && (!feats || !w)) return MI3D_ERR_ARG;
    PointsWs ws;
    if (!carve(workspace, P, H, radius, &ws) || ws.bytes > workspace_bytes) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int S = (int)H, n_t = (int)mi3d_ceil_div(H, kTile), n_tiles = n_t * n_t;
    const float r = (float)radius, r2_alpha = (float)(radius * radius);
    const unsigned pblocks = mi3d_ceil_div(P, kPtThreads);
    MI3D_CHECK(cudaMemsetAsync(ws.tile_cnt, 0, (size_t)n_tiles * 4, st));
    k_points_bin_count<<<pblocks, kPtThreads, 0, st>>>(points, P, cam_k, world2cam, proj_w, proj_h, S, r, n_t, ws.proj, ws.tile_cnt);
    k_points_tile_scan<<<1, 1024, 0, st>>>(ws.tile_cnt, n_tiles, ws.tile_off, ws.cursor);
    k_points_bin_emit<<<pblocks, kPtThreads, 0, st>>>(ws.proj, P, S, r, n_t, ws.cursor, ws.list);
    const dim3 blk(kTile, kTile);
    if (K <= 8)
        k_points_raster<8><<<n_tiles, blk, 0, st>>>(ws.proj, ws.tile_off, ws.list, S, n_t, r, r2_alpha, (int)K, feats, (int)C, image, idx, w,
                                                     zbuf, dist2);
    else
        k_points_raster<16><<<n_tiles, blk, 0, st>>>(ws.proj, ws.tile_off, ws.list, S, n_t, r, r2_alpha, (int)K, feats, (int)C, image, idx, w,
                                                      zbuf, dist2);
    MI3D_RETURN_LAUNCH();
}

int mi3d_points_render_backward(const float* points, uint32_t P, uint32_t C, const float* cam_k, const float* world2cam, float proj_w,
                                float proj_h, uint32_t H, uint32_t W, double radius, uint32_t K, const int* idx, const float* w,
                                const float* grad_image, float* grad_feats, mi3d_stream_t stream) {
    if (!valid_args(P, H, W, radius, K, C) || !points || !cam_k || !world2cam || !idx || !w || !grad_image || !grad_feats) return MI3D_ERR_ARG;
    k_points_feat_grad<<<mi3d_ceil_div(P, kPtThreads), kPtThreads, 0, (cudaStream_t)stream>>>(
        points, P, cam_k, world2cam, proj_w, proj_h, (int)H, (float)radius, (int)K, idx, w, grad_image, (int)C, grad_feats);
    MI3D_RETURN_LAUNCH();
}

int mi3d_points_zbuffer_visible(const double* points, uint32_t P, const double* cam_k, const double* world2cam, uint32_t H, uint32_t W,
                                unsigned long long* zbuf, uint8_t* mask, mi3d_stream_t stream) {
    if (P == 0) return MI3D_OK;
    if (!points || !cam_k || !world2cam || !zbuf || !mask || H == 0 || W == 0 || (uint64_t)H * W >= 0x80000000ull) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemsetAsync(zbuf, 0xff, (size_t)H * W * sizeof(unsigned long long), st));
    const unsigned blocks = mi3d_ceil_div(P, kPtThreads);
    k_zbuffer_min<<<blocks, kPtThreads, 0, st>>>(points, P, cam_k, world2cam, (int)H, (int)W, zbuf);
    k_zbuffer_mask<<<blocks, kPtThreads, 0, st>>>(points, P, cam_k, world2cam, (int)H, (int)W, zbuf, mask);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
