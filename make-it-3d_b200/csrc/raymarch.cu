// raymarch.cu -- occupancy-grid ray marching + alpha compositing for sm_90a (C ABI: include/mi3d.h)
//
// Replaces raymarching/src/raymarching.cu of the reference (file:line cited per entry point in
// include/mi3d.h).  Compiled with -fmad=false so that every fp32 op is a single IEEE rounding and the
// marched sample positions are bit-identical to the CPU oracle (oracle/raymarch_oracle.c).
//
// Notes: these kernels are launch-latency sized (N = 16k..65k rays); the design goal is *zero host
// synchronisation and zero fill traffic*:
//   * march_train is ONE kernel: count pass -> block scan -> decoupled look-back across CTAs (ticketed
//     block ids, so a CTA only ever waits on CTAs that already started) -> emit pass.  Compaction order is
//     the ray id, i.e. deterministic, unlike the reference's atomicAdd arrival order.
//   * near/far (slab test) is fused into the march kernel when no precomputed nears/fars are passed.
//   * the total sample count stays on the device (counter[0]); downstream kernels read it there.
#include "mi3d_internal.cuh"

namespace {

constexpr int kRayThreads = 128;

struct RayCtx {
    float ox, oy, oz, dx, dy, dz, rdx, rdy, rdz;
    float bound, dt_gamma, dt_min, dt_max, rH, H3f;
    uint32_t C, H;
    const uint8_t* grid;
};

__device__ __forceinline__ int level_from_pos(float x, float y, float z, int C) {
    const float mx = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
    int e; frexpf(mx, &e);
    return (int)fminf((float)(C - 1), fmaxf(0.0f, (float)e));
}
__device__ __forceinline__ int level_from_dt(float dt, float Hf, int C) {
    const float mx = dt * Hf * 0.5f;
    int e; frexpf(mx, &e);
    return (int)fminf((float)(C - 1), fmaxf(0.0f, (float)e));
}

__device__ __forceinline__ void slab_near_far(float ox, float oy, float oz, float rdx, float rdy, float rdz,
                                              const float* __restrict__ aabb, float min_near, float& tn, float& tf) {
    tn = (aabb[0] - ox) * rdx; tf = (aabb[3] - ox) * rdx;
    if (tn > tf) { float s = tn; tn = tf; tf = s; }
    float yn = (aabb[1] - oy) * rdy, yf = (aabb[4] - oy) * rdy;
    if (yn > yf) { float s = yn; yn = yf; yf = s; }
    if (tn > yf || yn > tf) { tn = tf = FLT_MAX; return; }
    if (yn > tn) tn = yn;
    if (yf < tf) tf = yf;
    float zn = (aabb[2] - oz) * rdz, zf = (aabb[5] - oz) * rdz;
    if (zn > zf) { float s = zn; zn = zf; zf = s; }
    if (tn > zf || zn > tf) { tn = tf = FLT_MAX; return; }
    if (zn > tn) tn = zn;
    if (zf < tf) tf = zf;
    if (tn < min_near) tn = min_near;
}

// Pixel-centre pinhole ray of batch ray i (nerf/utils.py:51-116 with N = -1: every pixel, row-major): view = i / rays_per_view,
// pixel = (i % rays_per_view) * pixel_stride + pixel_phase.  Same operation order as the reference's torch expression, one IEEE
// rounding per op (this file is compiled with -fmad=false):  xs = (x + 0.5 - cx) / fx, ys = (y + 0.5 - cy) / fy, zs = 1;
// depth_scale = 1 / sqrt(xs^2 + ys^2 + 1); dir = safe_normalize((xs, ys, 1)); rays_d = dir @ R^T; rays_o = t.
__device__ __forceinline__ void gen_ray(const mi3d_raygen& rg, uint32_t i, float o[3], float d[3], float& depth_scale,
                                        uint32_t& view, uint32_t& pixel) {
    view = i / rg.rays_per_view;
    pixel = (i - view * rg.rays_per_view) * rg.pixel_stride + rg.pixel_phase;
    const uint32_t px = pixel % rg.W, py = pixel / rg.W;
    const float* __restrict__ c = rg.cams + 16 * (size_t)view;
    const float fx = __ldg(c + 12), fy = __ldg(c + 13), cx = __ldg(c + 14), cy = __ldg(c + 15);
    const float xs = ((float)px + 0.5f - cx) / fx, ys = ((float)py + 0.5f - cy) / fy;
    const float ss = (xs * xs + ys * ys) + 1.0f;
    depth_scale = 1.0f / sqrtf(ss);
    const float q = sqrtf(fminf(fmaxf(ss, 1e-20f), 1e32f));          // safe_normalize, nerf/utils.py:47-48
    const float dx = xs / q, dy = ys / q, dz = 1.0f / q;
    #pragma unroll
    for (int k = 0; k < 3; k++) {
        d[k] = (dx * __ldg(c + 4 * k) + dy * __ldg(c + 4 * k + 1)) + dz * __ldg(c + 4 * k + 2);
        o[k] = __ldg(c + 4 * k + 3);
    }
}

__device__ __forceinline__ void ray_setup(RayCtx& r, const float* o, const float* d, float bound, float dt_gamma,
                                          uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t* grid) {
    r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
    r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    r.rdx = 1 / r.dx; r.rdy = 1 / r.dy; r.rdz = 1 / r.dz;
    r.bound = bound; r.dt_gamma = dt_gamma;
    r.dt_min = 2 * 1.7320508075688772f / (float)max_steps;
    r.dt_max = 2 * 1.7320508075688772f * (float)(1u << (C - 1)) / (float)H;
    r.rH = 1 / (float)H; r.H3f = (float)H * (float)H * (float)H;
    r.C = C; r.H = H; r.grid = grid;
}

// One ray, from t until far or until max_emit occupied samples.  EMIT=false only counts.
template <bool EMIT>
__device__ __forceinline__ uint32_t walk(const RayCtx& r, float& t, float far, uint32_t max_emit,
                                         float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas) {
    float last_t = t;
    uint32_t k = 0;
    const float Hf = (float)r.H, Hm1 = (float)(r.H - 1);
    const float sx = copysignf(1.0f, r.dx), sy = copysignf(1.0f, r.dy), sz = copysignf(1.0f, r.dz);
    while (t < far && k < max_emit) {
        const float x = mi3d_clampf(r.ox + t * r.dx, -r.bound, r.bound);
        const float y = mi3d_clampf(r.oy + t * r.dy, -r.bound, r.bound);
        const float z = mi3d_clampf(r.oz + t * r.dz, -r.bound, r.bound);
        const float dt = mi3d_clampf(t * r.dt_gamma, r.dt_min, r.dt_max);
        const int la = level_from_pos(x, y, z, (int)r.C), lb = level_from_dt(dt, Hf, (int)r.C);
        const int level = la > lb ? la : lb;
        const float mip_bound = fminf(scalbnf(1.0f, level), r.bound);
        const float mip_rbound = 1 / mip_bound;
        const int nx = (int)mi3d_clampf(0.5f * (x * mip_rbound + 1) * Hf, 0.0f, Hm1);
        const int ny = (int)mi3d_clampf(0.5f * (y * mip_rbound + 1) * Hf, 0.0f, Hm1);
        const int nz = (int)mi3d_clampf(0.5f * (z * mip_rbound + 1) * Hf, 0.0f, Hm1);
        const uint32_t index = (uint32_t)((float)level * r.H3f + (float)mi3d_morton((uint32_t)nx, (uint32_t)ny, (uint32_t)nz));
        const bool occ = __ldg(r.grid + (index >> 3)) & (1u << (index & 7u));
        if (occ) {
            if (EMIT) {
                xyzs[3 * k] = x; xyzs[3 * k + 1] = y; xyzs[3 * k + 2] = z;
                dirs[3 * k] = r.dx; dirs[3 * k + 1] = r.dy; dirs[3 * k + 2] = r.dz;
            }
            t += dt;
            if (EMIT) { deltas[2 * k] = dt; deltas[2 * k + 1] = t - last_t; }
            last_t = t;
            k++;
        } else {
            const float tx = (((nx + 0.5f + 0.5f * sx) * r.rH * 2 - 1) * mip_bound - x) * r.rdx;
            const float ty = (((ny + 0.5f + 0.5f * sy) * r.rH * 2 - 1) * mip_bound - y) * r.rdy;
            const float tz = (((nz + 0.5f + 0.5f * sz) * r.rH * 2 - 1) * mip_bound - z) * r.rdz;
            const float tt = t + fmaxf(0.0f, fminf(tx, fminf(ty, tz)));
            do { t += mi3d_clampf(t * r.dt_gamma, r.dt_min, r.dt_max); } while (t < tt);
        }
    }
    return k;
}

__global__ void __launch_bounds__(kRayThreads)
k_near_far(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ aabb,
           uint32_t N, float min_near, float* __restrict__ nears, float* __restrict__ fars) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    const float* o = rays_o + 3 * (size_t)n; const float* d = rays_d + 3 * (size_t)n;
    float tn, tf;
    slab_near_far(o[0], o[1], o[2], 1 / d[0], 1 / d[1], 1 / d[2], aabb, min_near, tn, tf);
    nears[n] = tn; fars[n] = tf;
}

__global__ void __launch_bounds__(kRayThreads)
k_get_rays(const mi3d_raygen rg, uint32_t N, float* __restrict__ rays_o, float* __restrict__ rays_d, float* __restrict__ depth_scale) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    float o[3], d[3], sc; uint32_t view, pixel;
    gen_ray(rg, n, o, d, sc, view, pixel);
    #pragma unroll
    for (int k = 0; k < 3; k++) { if (rays_o) rays_o[3 * (size_t)n + k] = o[k]; if (rays_d) rays_d[3 * (size_t)n + k] = d[k]; }
    if (depth_scale) depth_scale[n] = sc;
}

__global__ void k_morton3D(const int* __restrict__ coords, uint32_t N, int* __restrict__ indices) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    indices[n] = (int)mi3d_morton((uint32_t)coords[3 * (size_t)n], (uint32_t)coords[3 * (size_t)n + 1], (uint32_t)coords[3 * (size_t)n + 2]);
}
__global__ void k_morton3D_invert(const int* __restrict__ indices, uint32_t N, int* __restrict__ coords) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    const uint32_t v = (uint32_t)indices[n];
    coords[3 * (size_t)n] = (int)mi3d_compact3(v);
    coords[3 * (size_t)n + 1] = (int)mi3d_compact3(v >> 1);
    coords[3 * (size_t)n + 2] = (int)mi3d_compact3(v >> 2);
}

// One thread packs 8 cells = two float4 loads (coalesced 32 B per thread) -> one byte.
// thresh_dev (optional) lets the threshold stay on the device: thresh = min(*thresh_dev, thresh).
__global__ void k_packbits(const float* __restrict__ grid, uint32_t Nbytes, float thresh, const float* __restrict__ thresh_dev,
                           uint8_t* __restrict__ bits) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= Nbytes) return;
    if (thresh_dev) thresh = fminf(thresh, *thresh_dev);
    const float4 a = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n);
    const float4 b = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n + 1);
    uint32_t v = 0;
    v |= (a.x > thresh) ? 1u : 0u;   v |= (a.y > thresh) ? 2u : 0u;
    v |= (a.z > thresh) ? 4u : 0u;   v |= (a.w > thresh) ? 8u : 0u;
    v |= (b.x > thresh) ? 16u : 0u;  v |= (b.y > thresh) ? 32u : 0u;
    v |= (b.z > thresh) ? 64u : 0u;  v |= (b.w > thresh) ? 128u : 0u;
    bits[n] = (uint8_t)v;
}

// ---------------------------------------------------------------------------------------------
// Training march: count -> scan (block + decoupled look-back) -> emit, single launch.
// scan_ws layout (int32, zeroed by the host wrapper on the same stream):
//   [0] ticket, [1 .. 1+nblk) block aggregates, [1+nblk .. 1+2nblk) ready flags
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRayThreads)
k_march_train(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const uint8_t* __restrict__ grid,
              float bound, float dt_gamma, uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
              const float* __restrict__ nears_in, const float* __restrict__ fars_in,
              const float* __restrict__ aabb, float min_near, float* __restrict__ nears_out, float* __restrict__ fars_out,
              const float* __restrict__ noises, uint64_t seed,
              float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas,
              int* __restrict__ rays, int* __restrict__ counter, int* __restrict__ scan_ws,
              const mi3d_raygen rg, float* __restrict__ depth_scale_out) {
    __shared__ uint32_t s_bid, s_warp_tot[kRayThreads / 32], s_prefix;
    const uint32_t nblk = gridDim.x;
    if (threadIdx.x == 0) s_bid = (uint32_t)atomicAdd(scan_ws, 1);
    __syncthreads();
    const uint32_t bid = s_bid;
    const uint32_t n = bid * kRayThreads + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;

    RayCtx r;
    float t0 = 0.f, far = 0.f;
    uint32_t cnt = 0;
    if (n < N) {
        uint32_t view = 0, nkey = n;          // Philox key of the march jitter: (pixel, camera) when rays are generated here, so the
        if (rays_o) ray_setup(r, rays_o + 3 * (size_t)n, rays_d + 3 * (size_t)n, bound, dt_gamma, max_steps, C, H, grid);
        else {                                // draw does not depend on how a view's pixels are dealt to ranks (ray-parallel render)
            float o[3], d[3], sc;
            gen_ray(rg, n, o, d, sc, view, nkey);
            // identify the view by its camera position, not by its slot in this batch: the same view marched alone, in a multi-view
            // batch or dealt over ranks draws the same jitter
            view = (__float_as_uint(o[0]) * 0x9E3779B1u) ^ (__float_as_uint(o[1]) * 0x85EBCA77u) ^ (__float_as_uint(o[2]) * 0xC2B2AE3Du);
            ray_setup(r, o, d, bound, dt_gamma, max_steps, C, H, grid);
            if (depth_scale_out) depth_scale_out[n] = sc;
        }
        float near;
        if (nears_in) { near = nears_in[n]; far = fars_in[n]; }
        else {
            slab_near_far(r.ox, r.oy, r.oz, r.rdx, r.rdy, r.rdz, aabb, min_near, near, far);
            if (nears_out) { nears_out[n] = near; fars_out[n] = far; }
        }
        float noise;
        if (noises) noise = noises[n];
        else noise = mi3d_u01(mi3d_philox(make_uint4(nkey, view, 0u, 0x6d617263u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32))).x);
        t0 = near + mi3d_clampf(near * dt_gamma, r.dt_min, r.dt_max) * noise;
        float t = t0;
        cnt = walk<false>(r, t, far, max_steps, nullptr, nullptr, nullptr);
    }
    // block exclusive scan of cnt
    uint32_t incl = cnt;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) s_warp_tot[wid] = incl;
    __syncthreads();
    uint32_t warp_base = 0, block_tot = 0;
    #pragma unroll
    for (int w = 0; w < kRayThreads / 32; w++) { if (w < (int)wid) warp_base += s_warp_tot[w]; block_tot += s_warp_tot[w]; }
    const uint32_t local_off = warp_base + incl - cnt;

    volatile int* agg = scan_ws + 1;
    volatile int* flag = scan_ws + 1 + nblk;
    if (threadIdx.x == 0) { agg[bid] = (int)block_tot; __threadfence(); flag[bid] = 1; }
    if (wid == 0) {
        uint32_t sum = 0;
        for (uint32_t j = lane; j < bid; j += 32) {
            while (flag[j] == 0) { __nanosleep(20); }
            __threadfence();
            sum += (uint32_t)agg[j];
        }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) s_prefix = sum;
    }
    __syncthreads();
    const uint32_t prefix = s_prefix;
    // counter[0] += number of EMITTED samples.  Offsets are monotone in the ray id, so when the capacity M is exceeded the emitted
    // samples are the contiguous prefix [0, off) of the unique ray with off <= M < off + cnt (it and every later ray write nothing,
    // raymarching.cu:416).  The reference adds the uncapped total (raymarching.cu:405) and relies on its 268 MB zero-fill to make
    // the hole rows harmless; here nothing is zero-filled, so downstream kernels must see only rows that were written.
    const bool last = bid == nblk - 1 && threadIdx.x == 0;
    if (last) { if (prefix + block_tot <= M) counter[0] += (int)(prefix + block_tot); counter[1] += (int)N; scan_ws[0] = 0; }
    if (n >= N) return;
    const uint32_t off = prefix + local_off;
    rays[3 * (size_t)n] = (int)n; rays[3 * (size_t)n + 1] = (int)off; rays[3 * (size_t)n + 2] = (int)cnt;
    if (cnt != 0 && off <= M && off + cnt > M) counter[0] += (int)off;        // the one boundary ray of an overflowing march
    if (cnt == 0 || off + cnt > M) return;
    float t = t0;
    walk<true>(r, t, far, cnt, xyzs + 3 * (size_t)off, dirs + 3 * (size_t)off, deltas + 2 * (size_t)off);
}

// ---------------------------------------------------------------------------------------------
// Training composite (+ optional fused epilogue of NeRFRenderer.run_cuda: background mix, far-depth fill,
// depth_scale).  image_raw/ws are what the backward needs; image/depth are what the caller sees.
// ---------------------------------------------------------------------------------------------
// One WARP per ray: lanes take consecutive samples of the ray (coalesced 4 / 8 / 12-byte-stride loads instead of one thread striding
// through its ray), transmittance and the depth parameter come from warp scans, the early-out (raymarching.cu:565: stop after the
// sample that drives T below T_thresh) becomes a per-sample mask T_before >= T_thresh (T is monotone) plus a warp-uniform break.
// Same arithmetic per sample as the reference; only the association order of the running product / sums differs (~1e-7).
__global__ void __launch_bounds__(kRayThreads)
k_composite_train_fwd(const float* __restrict__ sigmas, const float* __restrict__ rgbs, const float* __restrict__ deltas,
                      const int* __restrict__ rays, uint32_t M, uint32_t N, float T_thresh,
                      float* __restrict__ weights_sum, float* __restrict__ depth, float* __restrict__ image,
                      const float* __restrict__ bg_color, float bg_scalar, int fuse_epilogue, float max_depth,
                      const float* __restrict__ depth_scale, float* __restrict__ image_out, float* __restrict__ depth_out, uint32_t rays_per_view) {
    const uint32_t n = (threadIdx.x + blockIdx.x * blockDim.x) >> 5, lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint32_t index = (uint32_t)rays[3 * (size_t)n], off = (uint32_t)rays[3 * (size_t)n + 1], cnt = (uint32_t)rays[3 * (size_t)n + 2];
    if (bg_color && rays_per_view) bg_color += 3 * (size_t)(index / rays_per_view);    // one background colour per view of the batch
    float T = 1.0f, t = 0.f, r = 0, g = 0, b = 0, ws = 0, d = 0;                      // T, t: carried across 32-sample chunks (warp-uniform)
    if (cnt != 0 && off + cnt <= M) {
        const float* sg = sigmas + off; const float* cl = rgbs + 3 * (size_t)off; const float* dl = deltas + 2 * (size_t)off;
        for (uint32_t base = 0; base < cnt; base += 32) {
            const uint32_t s = base + lane;
            const bool valid = s < cnt;
            float alpha = 0.f, dy = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
            if (valid) {
                const float2 de = *reinterpret_cast<const float2*>(dl + 2 * s);
                alpha = 1.0f - __expf(-sg[s] * de.x); dy = de.y;
                c0 = cl[3 * s]; c1 = cl[3 * s + 1]; c2 = cl[3 * s + 2];
            }
            float om = 1.0f - alpha, tt = dy;                          // inclusive scans: product of (1 - alpha), sum of deltas[:,1]
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float pm = __shfl_up_sync(0xffffffffu, om, o), pt = __shfl_up_sync(0xffffffffu, tt, o);
                if ((int)lane >= o) { om *= pm; tt += pt; }
            }
            float T_before = __shfl_up_sync(0xffffffffu, om, 1);
            T_before = T * (lane == 0 ? 1.0f : T_before);
            const float w = (valid && T_before >= T_thresh) ? alpha * T_before : 0.f;
            r += w * c0; g += w * c1; b += w * c2; ws += w; d += w * (t + tt);
            T *= __shfl_sync(0xffffffffu, om, 31);
            t += __shfl_sync(0xffffffffu, tt, 31);
            if (T < T_thresh) break;
        }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            r += __shfl_xor_sync(0xffffffffu, r, o); g += __shfl_xor_sync(0xffffffffu, g, o); b += __shfl_xor_sync(0xffffffffu, b, o);
            ws += __shfl_xor_sync(0xffffffffu, ws, o); d += __shfl_xor_sync(0xffffffffu, d, o);
        }
    }
    if (lane != 0) return;
    weights_sum[index] = ws; depth[index] = d;
    image[3 * (size_t)index] = r; image[3 * (size_t)index + 1] = g; image[3 * (size_t)index + 2] = b;
    if (fuse_epilogue) {
        const float tr = 1 - ws;
        const float b0 = bg_color ? bg_color[0] : bg_scalar, b1 = bg_color ? bg_color[1] : bg_scalar, b2 = bg_color ? bg_color[2] : bg_scalar;
        image_out[3 * (size_t)index] = r + tr * b0; image_out[3 * (size_t)index + 1] = g + tr * b1; image_out[3 * (size_t)index + 2] = b + tr * b2;
        float dd = d + tr * max_depth;
        if (depth_scale) dd = dd * depth_scale[index];
        depth_out[index] = dd;
    }
}

__global__ void __launch_bounds__(kRayThreads)
k_composite_train_bwd(const float* __restrict__ grad_ws, const float* __restrict__ grad_image, const float* __restrict__ grad_depth,
                      const float* __restrict__ sigmas, const float* __restrict__ rgbs, const float* __restrict__ deltas,
                      const int* __restrict__ rays, const float* __restrict__ weights_sum, const float* __restrict__ image,
                      uint32_t M, uint32_t N, float T_thresh,
                      const float* __restrict__ bg_color, float bg_scalar, int fuse_epilogue, float max_depth,
                      const float* __restrict__ depth_scale,
                      float* __restrict__ grad_sigmas, float* __restrict__ grad_rgbs, int zero_tail, uint32_t rays_per_view) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    const uint32_t index = (uint32_t)rays[3 * (size_t)n], off = (uint32_t)rays[3 * (size_t)n + 1], cnt = (uint32_t)rays[3 * (size_t)n + 2];
    if (bg_color && rays_per_view) bg_color += 3 * (size_t)(index / rays_per_view);
    if (cnt == 0 || off + cnt > M) return;
    const float gi0 = grad_image[3 * (size_t)index], gi1 = grad_image[3 * (size_t)index + 1], gi2 = grad_image[3 * (size_t)index + 2];
    float gw = grad_ws ? grad_ws[index] : 0.0f;
    if (fuse_epilogue) {
        // image_out = image + (1-ws)*bg ; depth_out = (depth + (1-ws)*max_depth) * depth_scale  (renderer.py:557,566-568)
        const float b0 = bg_color ? bg_color[0] : bg_scalar, b1 = bg_color ? bg_color[1] : bg_scalar, b2 = bg_color ? bg_color[2] : bg_scalar;
        gw -= gi0 * b0 + gi1 * b1 + gi2 * b2;
        if (grad_depth) gw -= grad_depth[index] * (depth_scale ? depth_scale[index] : 1.0f) * max_depth;
    }
    const float rf = image[3 * (size_t)index], gf = image[3 * (size_t)index + 1], bf = image[3 * (size_t)index + 2], wsf = weights_sum[index];
    const float* sg = sigmas + off; const float* cl = rgbs + 3 * (size_t)off; const float* dl = deltas + 2 * (size_t)off;
    float* gs = grad_sigmas + off; float* gr = grad_rgbs + 3 * (size_t)off;
    float T = 1.0f, r = 0, g = 0, b = 0, ws = 0;
    uint32_t s = 0;
    for (; s < cnt; s++) {
        const float dt = dl[2 * s];
        const float c0 = cl[3 * s], c1 = cl[3 * s + 1], c2 = cl[3 * s + 2];
        const float alpha = 1.0f - __expf(-sg[s] * dt);
        const float w = alpha * T;
        r += w * c0; g += w * c1; b += w * c2;
        ws += w;
        T *= 1.0f - alpha;
        gr[3 * s] = gi0 * w; gr[3 * s + 1] = gi1 * w; gr[3 * s + 2] = gi2 * w;
        gs[s] = dt * (gi0 * (T * c0 - (rf - r)) + gi1 * (T * c1 - (gf - g)) + gi2 * (T * c2 - (bf - b)) + gw * (1 - wsf));
        if (T < T_thresh) { s++; break; }
    }
    if (zero_tail) for (; s < cnt; s++) { gs[s] = 0.f; gr[3 * s] = 0.f; gr[3 * s + 1] = 0.f; gr[3 * s + 2] = 0.f; }
}

// ---------------------------------------------------------------------------------------------
// Inference march / composite (eval renderer, SURVEY 8f "next" row 2; kept B1-compatible).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRayThreads)
k_march_rays(uint32_t n_alive, uint32_t n_step, const int* __restrict__ rays_alive, const float* __restrict__ rays_t,
             const float* __restrict__ rays_o, const float* __restrict__ rays_d, float bound, float dt_gamma, uint32_t max_steps,
             uint32_t C, uint32_t H, const uint8_t* __restrict__ grid, const float* __restrict__ fars,
             float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas, const float* __restrict__ noises) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= n_alive) return;
    const int id = rays_alive[n];
    RayCtx r;
    ray_setup(r, rays_o + 3 * (size_t)id, rays_d + 3 * (size_t)id, bound, dt_gamma, max_steps, C, H, grid);
    float t = rays_t[id];
    t += mi3d_clampf(t * dt_gamma, r.dt_min, r.dt_max) * (noises ? noises[n] : 0.0f);
    const size_t base = (size_t)n * n_step;
    walk<true>(r, t, fars[id], n_step, xyzs + 3 * base, dirs + 3 * base, deltas + 2 * base);
}

__global__ void __launch_bounds__(kRayThreads)
k_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int* __restrict__ rays_alive, float* __restrict__ rays_t,
                 const float* __restrict__ sigmas, const float* __restrict__ rgbs, const float* __restrict__ normals,
                 const float* __restrict__ deltas, float* __restrict__ weights_sum, float* __restrict__ depth,
                 float* __restrict__ image, float* __restrict__ normal) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= n_alive) return;
    const int id = rays_alive[n];
    const size_t base = (size_t)n * n_step;
    float t = rays_t[id], d = depth[id], ws = weights_sum[id];
    float r = image[3 * (size_t)id], g = image[3 * (size_t)id + 1], b = image[3 * (size_t)id + 2];
    float nx = normal[3 * (size_t)id], ny = normal[3 * (size_t)id + 1], nz = normal[3 * (size_t)id + 2];
    uint32_t s = 0;
    while (s < n_step) {
        const size_t i = base + s;
        const float dt = deltas[2 * i];
        if (dt == 0) break;
        const float alpha = 1.0f - __expf(-sigmas[i] * dt);
        const float T = 1 - ws;
        const float w = alpha * T;
        ws += w;
        t += deltas[2 * i + 1];
        d += w * t;
        r += w * rgbs[3 * i]; g += w * rgbs[3 * i + 1]; b += w * rgbs[3 * i + 2];
        nx += w * normals[3 * i]; ny += w * normals[3 * i + 1]; nz += w * normals[3 * i + 2];
        if (T < T_thresh) break;
        s++;
    }
    if (s < n_step) rays_alive[n] = -1; else rays_t[id] = t;
    weights_sum[id] = ws; depth[id] = d;
    image[3 * (size_t)id] = r; image[3 * (size_t)id + 1] = g; image[3 * (size_t)id + 2] = b;
    normal[3 * (size_t)id] = nx; normal[3 * (size_t)id + 1] = ny; normal[3 * (size_t)id + 2] = nz;
}

// march_rays (raymarching.cu:907-1014) for the device-controlled evaluation loop (render.cu): n_step samples per alive ray, extents
// read from the control block; unused slots carry deltas = 0 (the reference zero-fills the buffers every iteration,
// raymarching.py:399-401; composite_rays stops at dt == 0).  The first-iteration jitter is Philox(seed, ray id).
__global__ void __launch_bounds__(kRayThreads)
k_eval_march(const Mi3dEvalCtl* __restrict__ ctl, const int* __restrict__ alive, const float* __restrict__ rays_t, const mi3d_render_eval_args a,
             const float* __restrict__ fars, float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas, int* __restrict__ counter) {
    const Mi3dEvalCtl c = *ctl;
    if (c.done) return;
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n == 0) counter[0] = c.rows;
    if (n >= (uint32_t)c.n_alive) return;
    const int id = alive[n];
    RayCtx r;
    ray_setup(r, a.rays_o + 3 * (size_t)id, a.rays_d + 3 * (size_t)id, a.bound, a.dt_gamma, a.max_steps, a.C, a.H, a.density_bitfield);
    float t = rays_t[id];
    if (c.step == 0 && a.perturb)
        t += mi3d_clampf(t * a.dt_gamma, r.dt_min, r.dt_max) * mi3d_u01(mi3d_philox(make_uint4((uint32_t)id, 0u, 0u, 0x6576616cu), make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32))).x);
    const size_t base = (size_t)n * c.n_step;
    const uint32_t k = walk<true>(r, t, fars[id], (uint32_t)c.n_step, xyzs + 3 * base, dirs + 3 * base, deltas + 2 * base);
    for (uint32_t s = k; s < (uint32_t)c.n_step; s++) {
        deltas[2 * (base + s)] = 0.f; deltas[2 * (base + s) + 1] = 0.f;
        #pragma unroll
        for (int q = 0; q < 3; q++) { xyzs[3 * (base + s) + q] = 0.f; dirs[3 * (base + s) + q] = 0.f; }
    }
}

}  // namespace

int mi3d_internal_eval_march(const Mi3dEvalCtl* ctl, const int* alive, const float* rays_t, const mi3d_render_eval_args* a, const float* fars,
                             float* xyzs, float* dirs, float* deltas, int* counter, cudaStream_t st) {
    k_eval_march<<<mi3d_ceil_div(a->N, kRayThreads), kRayThreads, 0, st>>>(ctl, alive, rays_t, *a, fars, xyzs, dirs, deltas, counter);
    MI3D_RETURN_LAUNCH();
}

extern "C" {

int mi3d_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N, float min_near,
                            float* nears, float* fars, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    k_near_far<<<mi3d_ceil_div(N, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(rays_o, rays_d, aabb, N, min_near, nears, fars);
    MI3D_RETURN_LAUNCH();
}

int mi3d_morton3D(const int* coords, uint32_t N, int* indices, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    k_morton3D<<<mi3d_ceil_div(N, 256), 256, 0, (cudaStream_t)stream>>>(coords, N, indices);
    MI3D_RETURN_LAUNCH();
}

int mi3d_morton3D_invert(const int* indices, uint32_t N, int* coords, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    k_morton3D_invert<<<mi3d_ceil_div(N, 256), 256, 0, (cudaStream_t)stream>>>(indices, N, coords);
    MI3D_RETURN_LAUNCH();
}

int mi3d_packbits(const float* grid, uint32_t n_bytes, float thresh, const float* thresh_dev, uint8_t* bitfield, mi3d_stream_t stream) {
    if (n_bytes == 0) return MI3D_OK;
    if (((uintptr_t)grid) & 15) return MI3D_ERR_ARG;
    k_packbits<<<mi3d_ceil_div(n_bytes, 256), 256, 0, (cudaStream_t)stream>>>(grid, n_bytes, thresh, thresh_dev, bitfield);
    MI3D_RETURN_LAUNCH();
}

size_t mi3d_march_rays_train_workspace_bytes(uint32_t N) {
    return (size_t)(1 + 2 * mi3d_ceil_div(N, kRayThreads)) * sizeof(int);
}

static int march_train_launch(const float* rays_o, const float* rays_d, const mi3d_raygen* rg, float* depth_scale_out,
                              const uint8_t* grid, float bound, float dt_gamma,
                              uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
                              const float* nears, const float* fars, const float* aabb, float min_near,
                              float* nears_out, float* fars_out, const float* noises, uint64_t seed,
                              float* xyzs, float* dirs, float* deltas, int* rays, int* counter,
                              void* workspace, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    if (!workspace || (!nears && !aabb) || C == 0 || C > 8) return MI3D_ERR_ARG;
    mi3d_raygen g{};
    if (!rays_o || !rays_d) {
        if (!rg || !rg->cams || rg->rays_per_view == 0 || rg->W == 0 || (uint64_t)rg->n_views * rg->rays_per_view != N) return MI3D_ERR_ARG;
        if ((uint64_t)(rg->rays_per_view - 1) * rg->pixel_stride + rg->pixel_phase >= (uint64_t)rg->H * rg->W) return MI3D_ERR_ARG;
        g = *rg; rays_o = rays_d = nullptr;
    }
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemsetAsync(workspace, 0, mi3d_march_rays_train_workspace_bytes(N), st));
    k_march_train<<<mi3d_ceil_div(N, kRayThreads), kRayThreads, 0, st>>>(rays_o, rays_d, grid, bound, dt_gamma, max_steps, N, C, H, M,
        nears, fars, aabb, min_near, nears_out, fars_out, noises, seed, xyzs, dirs, deltas, rays, counter, (int*)workspace, g, depth_scale_out);
    MI3D_RETURN_LAUNCH();
}

int mi3d_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid, float bound, float dt_gamma,
                          uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
                          const float* nears, const float* fars, const float* aabb, float min_near,
                          float* nears_out, float* fars_out, const float* noises, uint64_t seed,
                          float* xyzs, float* dirs, float* deltas, int* rays, int* counter,
                          void* workspace, mi3d_stream_t stream) {
    if (!rays_o || !rays_d) return MI3D_ERR_ARG;
    return march_train_launch(rays_o, rays_d, nullptr, nullptr, grid, bound, dt_gamma, max_steps, N, C, H, M, nears, fars, aabb, min_near,
                              nears_out, fars_out, noises, seed, xyzs, dirs, deltas, rays, counter, workspace, stream);
}

int mi3d_march_rays_train_cam(const mi3d_raygen* rg, float* depth_scale_out, const uint8_t* grid, float bound, float dt_gamma,
                              uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float* aabb, float min_near,
                              float* nears_out, float* fars_out, const float* noises, uint64_t seed,
                              float* xyzs, float* dirs, float* deltas, int* rays, int* counter, void* workspace, mi3d_stream_t stream) {
    return march_train_launch(nullptr, nullptr, rg, depth_scale_out, grid, bound, dt_gamma, max_steps, N, C, H, M, nullptr, nullptr, aabb, min_near,
                              nears_out, fars_out, noises, seed, xyzs, dirs, deltas, rays, counter, workspace, stream);
}

int mi3d_get_rays(const mi3d_raygen* rg, uint32_t N, float* rays_o, float* rays_d, float* depth_scale, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    if (!rg || !rg->cams || rg->rays_per_view == 0 || rg->W == 0 || (uint64_t)rg->n_views * rg->rays_per_view != N) return MI3D_ERR_ARG;
    if ((uint64_t)(rg->rays_per_view - 1) * rg->pixel_stride + rg->pixel_phase >= (uint64_t)rg->H * rg->W) return MI3D_ERR_ARG;
    k_get_rays<<<mi3d_ceil_div(N, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(*rg, N, rays_o, rays_d, depth_scale);
    MI3D_RETURN_LAUNCH();
}

int mi3d_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* deltas, const int* rays,
                                      uint32_t M, uint32_t N, float T_thresh, float* weights_sum, float* depth, float* image,
                                      const mi3d_epilogue* ep, float* image_out, float* depth_out, mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    const int fuse = ep != nullptr;
    if (fuse && (!image_out || !depth_out)) return MI3D_ERR_ARG;
    k_composite_train_fwd<<<mi3d_ceil_div(N, kRayThreads / 32), kRayThreads, 0, (cudaStream_t)stream>>>(
        sigmas, rgbs, deltas, rays, M, N, T_thresh, weights_sum, depth, image,
        fuse ? ep->bg_color : nullptr, fuse ? ep->bg_scalar : 0.f, fuse, fuse ? ep->max_depth : 0.f,
        fuse ? ep->depth_scale : nullptr, image_out, depth_out, fuse ? ep->rays_per_view : 0u);
    MI3D_RETURN_LAUNCH();
}

int mi3d_composite_rays_train_backward(const float* grad_weights_sum, const float* grad_image, const float* grad_depth,
                                       const float* sigmas, const float* rgbs, const float* deltas, const int* rays,
                                       const float* weights_sum, const float* image, uint32_t M, uint32_t N, float T_thresh,
                                       const mi3d_epilogue* ep, float* grad_sigmas, float* grad_rgbs, int zero_tail,
                                       mi3d_stream_t stream) {
    if (N == 0) return MI3D_OK;
    const int fuse = ep != nullptr;
    k_composite_train_bwd<<<mi3d_ceil_div(N, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(
        grad_weights_sum, grad_image, grad_depth, sigmas, rgbs, deltas, rays, weights_sum, image, M, N, T_thresh,
        fuse ? ep->bg_color : nullptr, fuse ? ep->bg_scalar : 0.f, fuse, fuse ? ep->max_depth : 0.f,
        fuse ? ep->depth_scale : nullptr, grad_sigmas, grad_rgbs, zero_tail, fuse ? ep->rays_per_view : 0u);
    MI3D_RETURN_LAUNCH();
}

int mi3d_march_rays(uint32_t n_alive, uint32_t n_step, const int* rays_alive, const float* rays_t, const float* rays_o,
                    const float* rays_d, float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H,
                    const uint8_t* grid, const float* nears, const float* fars, float* xyzs, float* dirs, float* deltas,
                    const float* noises, mi3d_stream_t stream) {
    (void)nears;
    if (n_alive == 0) return MI3D_OK;
    k_march_rays<<<mi3d_ceil_div(n_alive, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(
        n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, dt_gamma, max_steps, C, H, grid, fars, xyzs, dirs, deltas, noises);
    MI3D_RETURN_LAUNCH();
}

int mi3d_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int* rays_alive, float* rays_t, const float* sigmas,
                        const float* rgbs, const float* normals, const float* deltas, float* weights_sum, float* depth,
                        float* image, float* normal, mi3d_stream_t stream) {
    if (n_alive == 0) return MI3D_OK;
    k_composite_rays<<<mi3d_ceil_div(n_alive, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(
        n_alive, n_step, T_thresh, rays_alive, rays_t, sigmas, rgbs, normals, deltas, weights_sum, depth, image, normal);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
