// render.cu -- the training branch of NeRFRenderer.run_cuda (nerf/renderer.py:481-524,553-583) as ONE C-ABI call per direction.
//
//   mi3d_render_forward : [ray generation ->] near/far -> occupancy march -> fused field (hash grid + MLP + normals + shading +
//                         regulariser sums) -> composite + background / depth epilogue           (SURVEY.md 8b "mi3d_render_fwd")
//   mi3d_render_backward: composite backward -> fused field backward (gather | wgmma chain | RED scatter), accumulating into
//                         grad_table / grad_mlp                                                    (SURVEY.md 8b "mi3d_render_bwd")
// A non-Python host gets the whole fused path from these two entry points; nerf/field_ops.py uses them too.  Everything they
// launch is the same kernels the unfused B1 / B2 entry points expose (raymarch.cu, field.cu): this file only sequences them,
// derives the multi-view segment table on the device and carves the caller's workspace.  No allocation, no synchronisation.
//
// Multi-view batches / ray-parallel multi-GPU render (DESIGN.md section 5): a batch holds n_views * (N / n_views) rays; rank r of
// G ranks takes every G-th pixel of each of G views (mi3d_raygen stride / phase), so every rank marches ~1/G of every view's
// samples and the per-rank work is balanced whatever the poses are.  The reference's per-view means (loss_orient, loss_smooth:
// .mean() over the view's 128-padded sample rows) need the view's TOTAL sample count: forward phase MARCH leaves this rank's
// per-view counts in ws->view_counts, the host all-gathers them (G*G ints over NCCL, no host sync) and passes the table to
// phase SHADE, which builds the segment table (mi3d_view_segs) the field kernels read.
#include "mi3d_internal.cuh"

namespace {

// samples of view v in this rank's batch = rows between the first ray of view v and the first ray of view v + 1
__global__ void k_view_counts(const int* __restrict__ rays, const int* __restrict__ counter, uint32_t N, uint32_t n_views, uint32_t cap,
                              int* __restrict__ view_counts) {
    const uint32_t v = threadIdx.x;
    if (v >= n_views) return;
    const uint32_t rpv = N / n_views;
    const uint32_t total = min((uint32_t)counter[0], cap);
    const uint32_t b0 = min((uint32_t)rays[3 * (size_t)(v * rpv) + 1], total);
    const uint32_t b1 = v + 1 < n_views ? min((uint32_t)rays[3 * (size_t)((v + 1) * rpv) + 1], total) : total;
    view_counts[v] = (int)(b1 - b0);
}

// segment table: bounds of the real rows from this rank's own counts, mpad from the counts of all ranks, zero rows of the views in
// pad_view_mask appended after the real rows (clipped to the buffer capacity)
__global__ void k_view_segments(const int* __restrict__ my_counts, const int* __restrict__ all_counts, uint32_t n_ranks, uint32_t n_views,
                                uint32_t pad_view_mask, uint32_t align, uint32_t cap, mi3d_view_segs* __restrict__ segs) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    mi3d_view_segs s;
    s.n_views = n_views;
    uint32_t run = 0;
    for (uint32_t v = 0; v < MI3D_MAX_VIEWS; v++) s.mpad[v] = 1;
    for (uint32_t v = 0; v < n_views; v++) { s.bounds[v] = run; run += (uint32_t)my_counts[v]; }
    s.bounds[n_views] = run;
    for (uint32_t v = 0; v < n_views; v++) {
        uint32_t tot = 0;
        if (all_counts) { for (uint32_t r = 0; r < n_ranks; r++) tot += (uint32_t)all_counts[r * n_views + v]; }
        else tot = (uint32_t)my_counts[v];
        const uint32_t padded = align ? tot + align - tot % align : tot;       // raymarching.py:238-239 (always adds)
        s.mpad[v] = padded ? padded : 1;
        if ((pad_view_mask >> v) & 1u) run = min(run + (padded - tot), cap);
        s.bounds[n_views + v + 1] = run;
    }
    for (uint32_t j = 2 * n_views + 1; j < 2 * MI3D_MAX_VIEWS + 1; j++) s.bounds[j] = run;
    *segs = s;
}


// ---------------------------------------------------------------------------------------------------------
// Evaluation renderer (SURVEY 8f-2): the alive-ray loop of NeRFRenderer.run_cuda's non-training branch (nerf/renderer.py:526-551)
// with ALL control state on the device.  The reference iterates on the host: n_alive = rays_alive.shape[0] (a boolean-mask
// compaction, i.e. a device->host sync per iteration), n_step = clamp(N // n_alive, 1, 8), march -> field -> composite.
// Here a control block {n_alive, n_step, step, rows, next, done} lives in the workspace; every kernel reads its extent from it,
// the composite kernel appends surviving rays to the other half of a ping-pong alive list, and a one-thread kernel advances the
// block.  The host enqueues iterations without ever synchronising; it stops early when it sees the `done` word the advance kernel
// also writes to a caller-provided pinned / mapped host flag (a stale read only costs a few empty iterations).
// ---------------------------------------------------------------------------------------------------------
using EvalCtl = Mi3dEvalCtl;

__global__ void k_eval_init(uint32_t N, const float* __restrict__ nears, int* __restrict__ alive0, float* __restrict__ rays_t,
                            float* __restrict__ weights_sum, float* __restrict__ depth, float* __restrict__ image, float* __restrict__ normal,
                            EvalCtl* __restrict__ ctl, volatile int* done_host) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n == 0) {
        EvalCtl c; c.n_alive = (int)N; c.n_step = 1; c.step = 0; c.rows = (int)N; c.next = 0; c.done = N == 0; c.cur = 0; c.pad = 0;
        *ctl = c;
        if (done_host) *done_host = c.done;
    }
    if (n >= N) return;
    alive0[n] = (int)n; rays_t[n] = nears[n];
    weights_sum[n] = 0.f; depth[n] = 0.f;
    #pragma unroll
    for (int k = 0; k < 3; k++) { image[3 * (size_t)n + k] = 0.f; normal[3 * (size_t)n + k] = 0.f; }
}

// composite_rays (raymarching.cu:1024-1115) with normals mapped to (n + 1) / 2 like renderer.py:548; survivors go to the next list
__global__ void __launch_bounds__(128)
k_eval_composite(EvalCtl* __restrict__ ctl, const int* __restrict__ alive, int* __restrict__ alive_next, float* __restrict__ rays_t, float T_thresh,
                 const float* __restrict__ sigmas, const float* __restrict__ rgbs, const float* __restrict__ normals, const float* __restrict__ deltas,
                 float* __restrict__ weights_sum, float* __restrict__ depth, float* __restrict__ image, float* __restrict__ normal) {
    const EvalCtl c = *ctl;
    if (c.done) return;
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= (uint32_t)c.n_alive) return;
    const int id = alive[n];
    const size_t base = (size_t)n * c.n_step;
    float t = rays_t[id], d = depth[id], ws = weights_sum[id];
    float r = image[3 * (size_t)id], g = image[3 * (size_t)id + 1], b = image[3 * (size_t)id + 2];
    float nx = normal[3 * (size_t)id], ny = normal[3 * (size_t)id + 1], nz = normal[3 * (size_t)id + 2];
    int s = 0;
    while (s < c.n_step) {
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
        nx += w * ((normals[3 * i] + 1) / 2); ny += w * ((normals[3 * i + 1] + 1) / 2); nz += w * ((normals[3 * i + 2] + 1) / 2);
        if (T < T_thresh) break;
        s++;
    }
    if (s >= c.n_step) { rays_t[id] = t; alive_next[atomicAdd(&ctl->next, 1)] = id; }
    weights_sum[id] = ws; depth[id] = d;
    image[3 * (size_t)id] = r; image[3 * (size_t)id + 1] = g; image[3 * (size_t)id + 2] = b;
    normal[3 * (size_t)id] = nx; normal[3 * (size_t)id + 1] = ny; normal[3 * (size_t)id + 2] = nz;
}

__global__ void k_eval_advance(EvalCtl* __restrict__ ctl, uint32_t N, uint32_t max_steps, volatile int* done_host) {
    EvalCtl c = *ctl;
    if (c.done) return;
    c.step += c.n_step;                                   // renderer.py:551
    c.n_alive = c.next; c.next = 0; c.cur ^= 1;
    if (c.n_alive <= 0 || (uint32_t)c.step >= max_steps) { c.done = 1; c.n_alive = 0; c.rows = 0; }
    else { const int q = (int)N / c.n_alive; c.n_step = q < 1 ? 1 : (q > 8 ? 8 : q); c.rows = c.n_alive * c.n_step; }   // renderer.py:541
    *ctl = c;
    if (done_host && c.done) *done_host = 1;
}

// final background mix (renderer.py:553-570 for the eval branch): image / normal += (1 - ws) * bg ; depth fix-up
__global__ void k_eval_finish(uint32_t N, const float* __restrict__ bg_color, float bg_scalar, float max_depth, const float* __restrict__ depth_scale,
                              const float* __restrict__ weights_sum, float* __restrict__ depth, float* __restrict__ image, float* __restrict__ normal) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    const float tr = 1 - weights_sum[n];
    #pragma unroll
    for (int k = 0; k < 3; k++) {
        const float bgk = bg_color ? bg_color[k] : bg_scalar;
        image[3 * (size_t)n + k] += tr * bgk; normal[3 * (size_t)n + k] += tr * bgk;
    }
    float dd = depth[n] + tr * max_depth;
    if (depth_scale) dd *= depth_scale[n];
    depth[n] = dd;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

uint32_t sample_cap(uint32_t N, uint32_t max_steps, uint32_t max_samples, uint32_t n_views) {
    uint64_t c = (uint64_t)N * max_steps;
    if (max_samples && max_samples < c) c = max_samples;
    c += 128ull * n_views;                 // room for the aligned zero rows of every view (raymarching.py:237-241)
    return (uint32_t)(c > 0xFFFFFF00ull ? 0xFFFFFF00ull : c);
}

int fill_io(const mi3d_render_args* ra, const mi3d_render_ws* ws, bool use_segs, mi3d_field_io* io) {
    *io = mi3d_field_io{};
    io->xyzs = ws->xyzs; io->dirs = ws->dirs; io->counter = ws->counter; io->m_fixed = 0; io->align = 128; io->cap = ws->cap;
    io->smooth_noise = ra->smooth_noise; io->seed = ra->seed + 1;
    io->enc_cache = ws->enc_cache; io->enc_cache_tiles = ws->enc_cache_tiles; io->enc_cache_valid = 0;
    io->segs = use_segs ? ws->segs : nullptr; io->n_views = ra->n_views; io->noise_mode = ra->noise_mode;
    return MI3D_OK;
}

bool args_ok(const mi3d_render_args* ra, const mi3d_render_ws* ws) {
    if (!ra || !ws || ra->N == 0 || ra->n_views == 0 || ra->n_views > MI3D_MAX_VIEWS || ra->N % ra->n_views) return false;
    if (ra->N != ws->N || ra->n_views > ws->n_views) return false;
    if (!ra->rays_o && !ra->raygen) return false;
    if (ra->all_counts && (ra->n_ranks == 0)) return false;
    return true;
}

}  // namespace

extern "C" {

size_t mi3d_render_workspace_bytes(uint32_t N, uint32_t max_steps, uint32_t max_samples, uint32_t n_views, uint32_t enc_cache_tiles) {
    mi3d_render_ws ws;
    if (mi3d_render_workspace_carve(nullptr, N, max_steps, max_samples, n_views, enc_cache_tiles, &ws) != MI3D_OK) return 0;
    return ws.bytes;
}

// HOST: lay the per-sample / per-ray buffers out inside one caller-owned device blob (base may be NULL to size it only)
int mi3d_render_workspace_carve(void* base, uint32_t N, uint32_t max_steps, uint32_t max_samples, uint32_t n_views, uint32_t enc_cache_tiles,
                                mi3d_render_ws* out) {
    if (!out || N == 0 || n_views == 0 || n_views > MI3D_MAX_VIEWS) return MI3D_ERR_ARG;
    const uint32_t cap = sample_cap(N, max_steps, max_samples, n_views);
    size_t off = 0;
    auto take = [&](size_t bytes) { void* p = base ? (void*)((char*)base + off) : nullptr; off = align_up(off + bytes, 256); return p; };
    *out = mi3d_render_ws{};
    out->N = N; out->cap = cap; out->n_views = n_views;
    out->xyzs = (float*)take((size_t)cap * 12); out->dirs = (float*)take((size_t)cap * 12); out->deltas = (float*)take((size_t)cap * 8);
    out->sigmas = (float*)take((size_t)cap * 4); out->rgbs = (float*)take((size_t)cap * 12); out->tape = (float*)take((size_t)cap * 64);
    out->g_sigmas = (float*)take((size_t)cap * 4); out->g_rgbs = (float*)take((size_t)cap * 12);
    out->rays = (int*)take((size_t)N * 12); out->counter = (int*)take(16);
    out->nears = (float*)take((size_t)N * 4); out->fars = (float*)take((size_t)N * 4);
    out->ws_raw = (float*)take((size_t)N * 4); out->depth_raw = (float*)take((size_t)N * 4); out->image_raw = (float*)take((size_t)N * 12);
    out->depth_scale = (float*)take((size_t)N * 4);
    out->scan_ws = take(mi3d_march_rays_train_workspace_bytes(N));
    out->loss_partials = (float*)take((size_t)2 * n_views * mi3d_field_grid_ctas(0) * 4);
    out->view_counts = (int*)take(MI3D_MAX_VIEWS * 4);
    out->segs = (mi3d_view_segs*)take(sizeof(mi3d_view_segs));
    const uint32_t tiles = (cap + 127) / 128;
    out->enc_cache_tiles = enc_cache_tiles < tiles ? enc_cache_tiles : tiles;
    out->enc_cache = out->enc_cache_tiles ? (float*)take(mi3d_field_enc_cache_bytes(out->enc_cache_tiles)) : nullptr;
    if (!base) out->enc_cache = nullptr;
    out->bytes = off;
    return MI3D_OK;
}

int mi3d_render_forward(const mi3d_render_args* ra, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                        const mi3d_field_cfg* cfg, const mi3d_render_ws* ws, int phases, float* image, float* depth, float* weights_sum,
                        float* loss_orient, float* loss_smooth, mi3d_stream_t stream) {
    if (!args_ok(ra, ws) || !table || !hg || !mlp || !cfg) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const bool use_segs = ra->n_views > 1 || ra->all_counts != nullptr;
    if (phases & MI3D_RENDER_PHASE_MARCH) {
        MI3D_CHECK(cudaMemsetAsync(ws->counter, 0, 2 * sizeof(int), st));                           // renderer.py:504
        const uint32_t M = ws->cap - 128 * ws->n_views;
        int r;
        if (ra->rays_o)
            r = mi3d_march_rays_train(ra->rays_o, ra->rays_d, ra->density_bitfield, ra->bound, ra->dt_gamma, ra->max_steps, ra->N, ra->C, ra->H, M,
                                      nullptr, nullptr, ra->aabb, ra->min_near, ws->nears, ws->fars, ra->noises, ra->seed, ws->xyzs, ws->dirs,
                                      ws->deltas, ws->rays, ws->counter, ws->scan_ws, stream);
        else
            r = mi3d_march_rays_train_cam(ra->raygen, ws->depth_scale, ra->density_bitfield, ra->bound, ra->dt_gamma, ra->max_steps, ra->N, ra->C,
                                          ra->H, M, ra->aabb, ra->min_near, ws->nears, ws->fars, ra->noises, ra->seed, ws->xyzs, ws->dirs,
                                          ws->deltas, ws->rays, ws->counter, ws->scan_ws, stream);
        if (r) return r;
        if (use_segs) k_view_counts<<<1, 32, 0, st>>>(ws->rays, ws->counter, ra->N, ra->n_views, M, ws->view_counts);
    }
    if (phases & MI3D_RENDER_PHASE_SHADE) {
        if (!image || !depth || !weights_sum) return MI3D_ERR_ARG;
        if (use_segs)
            k_view_segments<<<1, 32, 0, st>>>(ws->view_counts, ra->all_counts, ra->n_ranks, ra->n_views, ra->pad_view_mask, 128u, ws->cap, ws->segs);
        mi3d_field_io io;
        fill_io(ra, ws, use_segs, &io);
        int r = mi3d_field_forward(&io, table, hg, mlp, cfg, ws->sigmas, ws->rgbs, nullptr, ws->tape, ws->loss_partials, loss_orient, loss_smooth, stream);
        if (r) return r;
        mi3d_epilogue ep{};
        ep.bg_color = ra->bg_color; ep.bg_scalar = ra->bg_scalar; ep.max_depth = ra->max_depth;
        ep.depth_scale = ra->rays_o ? ra->depth_scale : ws->depth_scale;
        ep.rays_per_view = ra->n_views > 1 ? ra->N / ra->n_views : 0u;
        // M = the MARCH capacity: a ray the march dropped (off + cnt > M) must composite to the background, not from unwritten rows
        r = mi3d_composite_rays_train_forward(ws->sigmas, ws->rgbs, ws->deltas, ws->rays, ws->cap - 128 * ws->n_views, ra->N, ra->T_thresh, ws->ws_raw, ws->depth_raw,
                                              ws->image_raw, &ep, image, depth, stream);
        if (r) return r;
        MI3D_CHECK(cudaMemcpyAsync(weights_sum, ws->ws_raw, (size_t)ra->N * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    MI3D_RETURN_LAUNCH();
}

int mi3d_render_backward(const mi3d_render_args* ra, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                         const mi3d_field_cfg* cfg, const mi3d_render_ws* ws, const float* grad_image, const float* grad_depth,
                         const float* grad_weights_sum, const float* grad_loss_orient, const float* grad_loss_smooth, float* grad_table,
                         const mi3d_mlp_grad* grad_mlp, void* bwd_workspace, int enc_cache_valid, mi3d_stream_t stream) {
    if (!args_ok(ra, ws) || !table || !hg || !mlp || !cfg || !grad_image || !grad_table || !grad_mlp) return MI3D_ERR_ARG;
    const bool use_segs = ra->n_views > 1 || ra->all_counts != nullptr;
    mi3d_epilogue ep{};
    ep.bg_color = ra->bg_color; ep.bg_scalar = ra->bg_scalar; ep.max_depth = ra->max_depth;
    ep.depth_scale = ra->rays_o ? ra->depth_scale : ws->depth_scale;
    ep.rays_per_view = ra->n_views > 1 ? ra->N / ra->n_views : 0u;
    int r = mi3d_composite_rays_train_backward(grad_weights_sum, grad_image, grad_depth, ws->sigmas, ws->rgbs, ws->deltas, ws->rays, ws->ws_raw,
                                               ws->image_raw, ws->cap - 128 * ws->n_views, ra->N, ra->T_thresh, &ep, ws->g_sigmas, ws->g_rgbs, 1, stream);
    if (r) return r;
    mi3d_field_io io;
    fill_io(ra, ws, use_segs, &io);
    io.enc_cache_valid = enc_cache_valid ? 1u : 0u;
    return mi3d_field_backward(&io, table, hg, mlp, cfg, ws->tape, ws->g_sigmas, ws->g_rgbs, nullptr, grad_loss_orient, grad_loss_smooth,
                               grad_table, grad_mlp, bwd_workspace, stream);
}


// ---- evaluation renderer: the whole alive-ray loop, no host synchronisation ----
size_t mi3d_render_eval_workspace_bytes(uint32_t N) {
    const size_t rows = (size_t)N + 128;                                // n_alive * n_step <= N (n_step = clamp(N / n_alive, 1, 8))
    size_t b = 256;                                                    // control block
    b += align_up((size_t)N * 4, 256) * 5;                             // alive x2, rays_t, nears, fars
    b += align_up(rows * 12, 256) * 4 + align_up(rows * 8, 256) + align_up(rows * 4, 256);   // xyzs, dirs, rgbs, normals | deltas | sigmas
    b += 256;                                                          // row counter
    return b;
}

int mi3d_render_eval(const mi3d_render_eval_args* a, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp, const mi3d_field_cfg* cfg,
                     void* workspace, int* done_flag_host, float* weights_sum, float* depth, float* image, float* normal, mi3d_stream_t stream) {
    if (!a || !table || !hg || !mlp || !cfg || !workspace || !weights_sum || !depth || !image || !normal || !a->rays_o || !a->rays_d || !a->aabb) return MI3D_ERR_ARG;
    const uint32_t N = a->N;
    if (N == 0) return MI3D_OK;
    cudaStream_t st = (cudaStream_t)stream;
    char* p = (char*)workspace;
    auto take = [&](size_t bytes) { void* q = p; p += align_up(bytes, 256); return q; };
    const size_t rows = (size_t)N + 128;
    EvalCtl* ctl = (EvalCtl*)take(256);
    int* alive[2] = {(int*)take((size_t)N * 4), (int*)take((size_t)N * 4)};
    float* rays_t = (float*)take((size_t)N * 4); float* nears = (float*)take((size_t)N * 4); float* fars = (float*)take((size_t)N * 4);
    float* xyzs = (float*)take(rows * 12); float* dirs = (float*)take(rows * 12); float* rgbs = (float*)take(rows * 12); float* normals = (float*)take(rows * 12);
    float* deltas = (float*)take(rows * 8); float* sigmas = (float*)take(rows * 4);
    int* counter = (int*)take(256);
    int r = mi3d_near_far_from_aabb(a->rays_o, a->rays_d, a->aabb, N, a->min_near, nears, fars, stream);
    if (r) return r;
    const unsigned blocks = (N + 127) / 128;
    k_eval_init<<<blocks, 128, 0, st>>>(N, nears, alive[0], rays_t, weights_sum, depth, image, normal, ctl, done_flag_host);
    mi3d_field_io io{};
    io.xyzs = xyzs; io.dirs = dirs; io.counter = counter; io.m_fixed = 0; io.align = 128; io.cap = (uint32_t)rows;
    mi3d_field_cfg fc = *cfg;
    fc.n_evals = 7;                                        // sigma, colour AND the finite-difference normal (renderer.py:547-548)
    for (uint32_t it = 0; it < a->max_steps; it++) {
        if (done_flag_host && *(volatile int*)done_flag_host) break;      // stale reads only cost empty iterations
        const int cur = (int)(it & 1);
        r = mi3d_internal_eval_march(ctl, alive[cur], rays_t, a, fars, xyzs, dirs, deltas, counter, st);
        if (r) return r;
        r = mi3d_field_forward(&io, table, hg, mlp, &fc, sigmas, rgbs, normals, nullptr, nullptr, nullptr, nullptr, stream);
        if (r) return r;
        k_eval_composite<<<blocks, 128, 0, st>>>(ctl, alive[cur], alive[cur ^ 1], rays_t, a->T_thresh, sigmas, rgbs, normals, deltas, weights_sum, depth, image, normal);
        k_eval_advance<<<1, 1, 0, st>>>(ctl, N, a->max_steps, done_flag_host);
    }
    k_eval_finish<<<blocks, 128, 0, st>>>(N, a->bg_color, a->bg_scalar, a->max_depth, a->depth_scale, weights_sum, depth, image, normal);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
