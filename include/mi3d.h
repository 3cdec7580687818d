/*
 * mi3d.h -- C ABI of the H100-native (sm_90a) Make-It-3D SDS-step hot path (libmi3d.so).
 *
 * Drop-in boundary (SURVEY.md 8b): these entry points are what the reference's pybind module `_raymarching`
 * (raymarching/src/bindings.cpp:5-23, raymarching/src/raymarching.h:7-22), its third-party tiny-cuda-nn
 * encoder (nerf/network_tcnn.py:54-65,107) and its diffusers U-Net / VAE calls (nerf/sd.py:117-174,212-220)
 * would bind instead.  Conventions for every function:
 *   - plain pointers are DEVICE pointers unless named *_host or documented otherwise; sizes are element counts
 *   - returns 0 on success, a cudaError_t value or MI3D_ERR_ARG (1000001) otherwise; never throws
 *   - never allocates device memory and never synchronises; work is enqueued on `stream`
 *     (pass torch.cuda.current_stream().cuda_stream); scratch comes from the caller, sized by *_workspace_bytes()
 *   - re-entrant; no global mutable state besides one-time kernel attribute setup
 *   - all floating-point tensors are fp32 contiguous, exactly as the reference wrappers pass them
 *     (custom_fwd(cast_inputs=torch.float32), raymarching/raymarching.py:33,175,252)
 */
#ifndef MI3D_H
#define MI3D_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mi3d_stream_t; /* cudaStream_t */

/* ------------------------------------------------------------------------------------------------------
 * B1: ray-march operators  (replace raymarching/src/raymarching.cu, called from raymarching/raymarching.py)
 * ------------------------------------------------------------------------------------------------------ */

/* replaces near_far_from_aabb, raymarching.cu:92-160 (wrapper raymarching.py:31-61) */
int mi3d_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N, float min_near,
                            float* nears, float* fars, mi3d_stream_t stream);

/* replaces morton3D / morton3D_invert, raymarching.cu:214-258 (raymarching.py:95-142) */
int mi3d_morton3D(const int* coords, uint32_t N, int* indices, mi3d_stream_t stream);
int mi3d_morton3D_invert(const int* indices, uint32_t N, int* coords, mi3d_stream_t stream);

/* replaces packbits, raymarching.cu:268-300 (raymarching.py:144-170).  n_bytes = C*H^3/8.
 * thresh_dev (nullable) is a device scalar: effective threshold = min(thresh, *thresh_dev) -- this is
 * renderer.py:630 `min(self.mean_density, self.density_thresh)` without the .item() host sync. */
int mi3d_packbits(const float* grid, uint32_t n_bytes, float thresh, const float* thresh_dev, uint8_t* bitfield,
                  mi3d_stream_t stream);

/* replaces march_rays_train, raymarching.cu:312-493 (raymarching.py:173-247).
 *  - nears/fars: precomputed [N] (B1 behaviour) or NULL, in which case the slab test against aabb[6] with
 *    min_near is fused into the kernel (optionally written to nears_out/fars_out, nullable).
 *  - noises: [N] U[0,1) (raymarching.py:226) or NULL -> in-kernel Philox keyed by (seed, ray id).
 *  - rays[n] = (n, offset, count): compaction is ordered by ray id (deterministic), not by atomic arrival.
 *  - counter[0] += EMITTED samples, counter[1] += N (caller zeroes it like renderer.py:504).
 *  - M = capacity of xyzs/dirs/deltas in rows; rays that do not fit write nothing (raymarching.cu:416).  Because
 *    offsets are ordered by ray id the emitted samples are always the contiguous prefix [0, counter[0]) -- on overflow
 *    counter[0] is the offset of the first dropped ray, not the uncapped total the reference adds (raymarching.cu:405):
 *    nothing is zero-filled here, so consumers must never see the unwritten rows.
 *  - workspace: mi3d_march_rays_train_workspace_bytes(N) bytes (zero-filled internally). */
size_t mi3d_march_rays_train_workspace_bytes(uint32_t N);
int mi3d_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* density_bitfield, float bound,
                          float dt_gamma, uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
                          const float* nears, const float* fars, const float* aabb, float min_near,
                          float* nears_out, float* fars_out, const float* noises, uint64_t seed,
                          float* xyzs, float* dirs, float* deltas, int* rays, int* counter,
                          void* workspace, mi3d_stream_t stream);

/* Ray generation (replaces get_rays, nerf/utils.py:51-116, for the N = -1 "every pixel" mode training uses, provider.py:297).
 * A batch holds n_views * rays_per_view rays: batch ray i belongs to view i / rays_per_view and to the row-major pixel
 * (i % rays_per_view) * pixel_stride + pixel_phase of that view.  stride 1 / phase 0 / rays_per_view = H*W is one full image;
 * stride G / phase r deals every G-th pixel of each of G views to rank r (ray-parallel render, DESIGN.md section 5).
 * cams: DEVICE [n_views][16] fp32 = rows 0..2 of the cam2world pose (3x4 row-major, R | t) followed by fx, fy, cx, cy. */
typedef struct {
    const float* cams;
    uint32_t n_views;
    uint32_t H, W;
    uint32_t rays_per_view;
    uint32_t pixel_stride, pixel_phase;
} mi3d_raygen;
/* rays_o / rays_d [N,3], depth_scale [N] (each nullable), N = n_views * rays_per_view */
int mi3d_get_rays(const mi3d_raygen* rg, uint32_t N, float* rays_o, float* rays_d, float* depth_scale, mi3d_stream_t stream);
/* mi3d_march_rays_train with the rays generated inside the kernel (no rays_o / rays_d tensors; near/far always fused):
 * depth_scale_out [N] nullable.  The Philox march jitter (noises == NULL) is keyed by (view, pixel), not by the batch index. */
int mi3d_march_rays_train_cam(const mi3d_raygen* rg, float* depth_scale_out, const uint8_t* density_bitfield, float bound,
                              float dt_gamma, uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
                              const float* aabb, float min_near, float* nears_out, float* fars_out, const float* noises,
                              uint64_t seed, float* xyzs, float* dirs, float* deltas, int* rays, int* counter,
                              void* workspace, mi3d_stream_t stream);

/* Optional fused epilogue of NeRFRenderer.run_cuda (nerf/renderer.py:553-570):
 *   image_out = image + (1 - ws) * bg ;  depth_out = (depth + (1 - ws) * max_depth) * depth_scale */
typedef struct {
    const float* bg_color;    /* device [3] or NULL -> bg_scalar (renderer.py:554-555 default 1) */
    float bg_scalar;
    float max_depth;          /* opt.max_depth, main.py:91 */
    const float* depth_scale; /* device [N] or NULL */
    uint32_t rays_per_view;   /* > 0: multi-view batch, bg_color is [n_views][3] and ray n uses row n / rays_per_view; 0: one colour */
} mi3d_epilogue;

/* replaces composite_rays_train_forward, raymarching.cu:501-590 (raymarching.py:250-281).
 * ep == NULL -> plain B1 behaviour (image_out/depth_out ignored). */
int mi3d_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* deltas, const int* rays,
                                      uint32_t M, uint32_t N, float T_thresh, float* weights_sum, float* depth,
                                      float* image, const mi3d_epilogue* ep, float* image_out, float* depth_out,
                                      mi3d_stream_t stream);

/* replaces composite_rays_train_backward, raymarching.cu:602-696 (raymarching.py:283-300).
 * grad_image is w.r.t. image (ep == NULL) or image_out (ep != NULL); grad_depth (nullable) is w.r.t. depth_out and
 * only reaches sigmas through (1 - ws) * max_depth, like autograd does in the reference (raymarching.py:287).
 * zero_tail != 0 writes zeros to samples after the early-out so the outputs need no pre-zeroing. */
int mi3d_composite_rays_train_backward(const float* grad_weights_sum, const float* grad_image, const float* grad_depth,
                                       const float* sigmas, const float* rgbs, const float* deltas, const int* rays,
                                       const float* weights_sum, const float* image, uint32_t M, uint32_t N,
                                       float T_thresh, const mi3d_epilogue* ep, float* grad_sigmas, float* grad_rgbs,
                                       int zero_tail, mi3d_stream_t stream);

/* replaces march_rays / composite_rays (inference), raymarching.cu:907-1022, :1024-1125 (raymarching.py:368-470) */
int mi3d_march_rays(uint32_t n_alive, uint32_t n_step, const int* rays_alive, const float* rays_t, const float* rays_o,
                    const float* rays_d, float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H,
                    const uint8_t* density_bitfield, const float* nears, const float* fars, float* xyzs, float* dirs,
                    float* deltas, const float* noises, mi3d_stream_t stream);
int mi3d_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int* rays_alive, float* rays_t,
                        const float* sigmas, const float* rgbs, const float* normals, const float* deltas,
                        float* weights_sum, float* depth, float* image, float* normal, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B2: field  (replaces tinycudann.Encoding + nerf/network_tcnn.py MLP / common_forward / normal / forward)
 * ------------------------------------------------------------------------------------------------------ */

/* Multiresolution hash grid geometry (tiny-cuda-nn HashGrid as configured at nerf/network_tcnn.py:54-65):
 * level l owns entries [offsets[l], offsets[l]+sizes[l]) of the flat fp32 table `encoder.params`
 * (2 features per entry, entry-major). */
typedef struct {
    uint32_t n_levels;
    uint32_t n_entries;
    uint32_t offsets[16];
    uint32_t sizes[16];
    uint32_t ress[16];
    float scales[16];
} mi3d_hashgrid;

/* HOST helper: fills *out (host struct, passed by pointer to the calls below). */
int mi3d_hashgrid_make(uint32_t n_levels, uint32_t base_resolution, double per_level_scale, uint32_t log2_hashmap_size,
                       mi3d_hashgrid* out);

/* stand-alone encoder: replaces tcnn.Encoding.forward / backward as called at nerf/network_tcnn.py:107.
 * x [E,3] in [0,1]; out / grad_out [E, 2*n_levels]; grad_table accumulates (+=). hg is a HOST pointer. */
int mi3d_hashgrid_forward(const float* x, uint32_t E, const float* table, const mi3d_hashgrid* hg, float* out, mi3d_stream_t stream);
int mi3d_hashgrid_backward(const float* x, uint32_t E, const float* grad_out, const mi3d_hashgrid* hg, float* grad_table, mi3d_stream_t stream);

/* sigma_net = MLP(32, 4, 64, 3) (nerf/network_tcnn.py:67, :13-32): PyTorch nn.Linear layout [out][in], biases on */
typedef struct { const float *w1, *b1, *w2, *b2, *w3, *b3; } mi3d_mlp;
typedef struct { float *w1, *b1, *w2, *b2, *w3, *b3; } mi3d_mlp_grad;

enum { MI3D_SHADING_ALBEDO = 0, MI3D_SHADING_LAMBERTIAN = 1, MI3D_SHADING_TEXTURELESS = 2, MI3D_SHADING_NORMAL = 3 };

typedef struct {
    float bound;          /* opt.bound */
    float blob_density;   /* opt.blob_density (main.py:56) */
    float blob_radius;    /* opt.blob_radius  (main.py:57) */
    int n_evals;          /* 1: sigma/albedo only; 7: + 6-tap finite-difference normal (network_tcnn.py:115-138);
                             13: + the perturbed normal of the smoothness loss (renderer.py:521-524) */
    int shading;          /* MI3D_SHADING_* (network_tcnn.py:146-170) */
    float ambient_ratio;
    const float* light_d; /* device [3] (multi-view batches: [n_views][3]), needed unless shading == albedo */
} mi3d_field_cfg;

/* Multi-view batches (several camera views' rays in one march: ray-parallel multi-GPU render, or several views per GPU).
 * Samples are emitted in ray order, hence grouped by view.  DEVICE table, written by mi3d_render_forward (phase SHADE):
 *   rows [bounds[s], bounds[s+1]),  s <  n_views : the samples of view s in this batch
 *                                   s >= n_views : zero rows of view s - n_views evaluated here (the reference pads every view's
 *                                                  sample list to the next multiple of 128 with xyz = dir = 0 rows that take part
 *                                                  in the loss means, raymarching.py:237-241; exactly one rank owns a view's)
 *   mpad[v] : padded sample count of the WHOLE view v, summed over all ranks -- the denominator of its loss means. */
#define MI3D_MAX_VIEWS 8
typedef struct {
    uint32_t n_views;
    uint32_t bounds[2 * MI3D_MAX_VIEWS + 1];
    uint32_t mpad[MI3D_MAX_VIEWS];
} mi3d_view_segs;

typedef struct {
    const float* xyzs;         /* [cap,3] sample positions (output of mi3d_march_rays_train) */
    const float* dirs;         /* [cap,3] or NULL */
    const int* counter;        /* device: counter[0] = number of valid rows M; NULL -> m_fixed */
    uint32_t m_fixed;
    uint32_t align;            /* 128 reproduces the zero-row padding of raymarching.py:237-241 in the loss means; 0 = none */
    uint32_t cap;              /* rows allocated in every per-sample buffer */
    const float* smooth_noise; /* [cap,3] N(0,1) (renderer.py:522) or NULL -> in-kernel Philox(seed,row) */
    uint64_t seed;
    /* optional encoding cache shared by one forward and the backward(s) that follow it: fp32 [enc_cache_tiles][13][128][32]
     * (mi3d_field_enc_cache_bytes).  mi3d_field_forward stores the hash-grid encodings of the first enc_cache_tiles 128-row tiles of
     * every evaluation point there; mi3d_field_backward, when enc_cache_valid != 0, reads them back instead of re-gathering the
     * table (same table, same samples: the caller vouches for it).  Rows beyond the cache are re-gathered.  NULL = off. */
    float* enc_cache;
    uint32_t enc_cache_tiles;
    uint32_t enc_cache_valid;
    /* multi-view batch: DEVICE table (NULL = one view: counter / m_fixed / align above describe the rows) and its view count.
     * With segs, loss_orient / loss_smooth / grad_loss_* are [n_views] arrays and loss_partials holds
     * 2 * n_views * mi3d_field_grid_ctas(0) floats. */
    const mi3d_view_segs* segs;
    uint32_t n_views;
    uint32_t noise_mode;       /* in-kernel smoothness perturbation keyed by 0: (seed, row)  1: (seed, sample position) */
} mi3d_field_io;
size_t mi3d_field_enc_cache_bytes(uint32_t tiles);

/* number of CTAs the persistent field kernels launch; loss_partials must hold 2 * mi3d_field_grid_ctas(0) floats */
int mi3d_field_grid_ctas(int backward);

/* Fused replacement of NeRFNetwork.forward (+ the regularisers of run_cuda):
 *   sigmas[row], rgbs[row,3], normals[row,3] (nullable), tape[row,16] (nullable; needed for backward),
 *   loss_orient / loss_smooth: device scalars (nullable), means over the padded row count like the reference. */
int mi3d_field_forward(const mi3d_field_io* io, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                       const mi3d_field_cfg* cfg, float* sigmas, float* rgbs, float* normals, float* tape,
                       float* loss_partials, float* loss_orient, float* loss_smooth, mi3d_stream_t stream);

/* Backward of the above: accumulates (+=) into grad_table [2*n_entries] and grad_mlp.  grad_* inputs are nullable
 * (treated as zero); grad_loss_* are device scalars.  No gradient w.r.t. positions (the reference requests none). */
int mi3d_field_backward(const mi3d_field_io* io, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                        const mi3d_field_cfg* cfg, const float* tape, const float* grad_sigmas, const float* grad_rgbs,
                        const float* grad_normals, const float* grad_loss_orient, const float* grad_loss_smooth,
                        float* grad_table, const mi3d_mlp_grad* grad_mlp, void* workspace, mi3d_stream_t stream);
/* workspace (nullable): mi3d_field_backward_workspace_bytes() bytes of scratch (one encoding staging buffer, 1.74 GB).  When given,
 * the backward runs per chunk of 1 048 576 samples: encodings come from io->enc_cache or from a full-occupancy gather kernel into the
 * scratch, then the tensor-core chain kernel runs and issues the table-gradient REDs itself.
 * When NULL the chain kernel also gathers in-kernel (slower: its eight gather warps are starved); the Python host always passes scratch. */
size_t mi3d_field_backward_workspace_bytes(void);

/* ------------------------------------------------------------------------------------------------------
 * Fused render step: the training branch of NeRFRenderer.run_cuda (nerf/renderer.py:481-524,553-583) as one call per
 * direction (SURVEY.md 8b "mi3d_render_fwd / mi3d_render_bwd").  Sequences the kernels behind the B1 / B2 entry points
 * above over one caller-owned workspace; see csrc/render.cu for the multi-view / ray-parallel protocol.
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    /* rays: explicit tensors, or generated in the march kernel from cameras when rays_o == NULL */
    const float* rays_o;          /* [N,3] */
    const float* rays_d;          /* [N,3] */
    const float* depth_scale;     /* [N] or NULL (explicit rays only; generated rays carry their own) */
    const mi3d_raygen* raygen;    /* HOST struct (its cams pointer is a device pointer) */
    uint32_t N;
    uint32_t n_views;             /* views in the batch, 1..MI3D_MAX_VIEWS; view of ray i = i / (N / n_views) */
    /* occupancy grid + march (renderer.py:481-508; min_near is the wrapper default 0.2, raymarching.py:34) */
    const uint8_t* density_bitfield;
    uint32_t C, H;
    float bound, dt_gamma;
    uint32_t max_steps;
    float min_near;
    const float* aabb;            /* device [6] */
    const float* noises;          /* [N] or NULL -> Philox(seed) */
    uint64_t seed;
    /* compositing + epilogue (renderer.py:553-570) */
    float T_thresh;
    const float* bg_color;        /* device [n_views][3] or NULL -> bg_scalar */
    float bg_scalar;
    float max_depth;
    /* regularisers (renderer.py:513-524) */
    const float* smooth_noise;    /* [cap,3] or NULL -> Philox(seed + 1) */
    uint32_t noise_mode;          /* mi3d_field_io.noise_mode */
    /* ray-parallel multi-rank render */
    const int* all_counts;        /* DEVICE [n_ranks][n_views]: every rank's ws->view_counts, all-gathered; NULL = this rank holds whole views */
    uint32_t n_ranks;
    uint32_t pad_view_mask;       /* bit v set: this rank evaluates the 128-alignment zero rows of view v (exactly one rank per view) */
} mi3d_render_args;

typedef struct {                  /* filled by mi3d_render_workspace_carve; all DEVICE pointers into the caller's blob */
    uint32_t N, cap, n_views;     /* cap = min(N * max_steps, max_samples) + 128 * n_views rows */
    float *xyzs, *dirs, *deltas, *sigmas, *rgbs, *tape, *g_sigmas, *g_rgbs;        /* per sample */
    int *rays, *counter;                                                            /* [N,3], [2]: counter[0] = emitted samples */
    float *nears, *fars, *ws_raw, *depth_raw, *image_raw, *depth_scale;             /* per ray */
    void* scan_ws;
    float* loss_partials;
    int* view_counts;             /* [MI3D_MAX_VIEWS] this rank's samples per view (written by phase MARCH of multi-view batches) */
    mi3d_view_segs* segs;
    float* enc_cache;
    uint32_t enc_cache_tiles;
    size_t bytes;
} mi3d_render_ws;

size_t mi3d_render_workspace_bytes(uint32_t N, uint32_t max_steps, uint32_t max_samples /* 0 = N * max_steps */, uint32_t n_views,
                                   uint32_t enc_cache_tiles);
int mi3d_render_workspace_carve(void* base, uint32_t N, uint32_t max_steps, uint32_t max_samples, uint32_t n_views,
                                uint32_t enc_cache_tiles, mi3d_render_ws* out);

enum { MI3D_RENDER_PHASE_MARCH = 1, MI3D_RENDER_PHASE_SHADE = 2, MI3D_RENDER_PHASE_ALL = 3 };
/* image [N,3], depth [N], weights_sum [N]; loss_orient / loss_smooth: device scalars (one view, single rank) or [n_views] arrays
 * of this rank's SHARE of every view's mean (multi-view: sum them over ranks).  phases: MARCH | SHADE; a multi-rank caller runs
 * MARCH, all-gathers ws->view_counts into args->all_counts, then runs SHADE. */
int mi3d_render_forward(const mi3d_render_args* args, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                        const mi3d_field_cfg* cfg, const mi3d_render_ws* ws, int phases, float* image, float* depth,
                        float* weights_sum, float* loss_orient, float* loss_smooth, mi3d_stream_t stream);
/* grad_image [N,3] required; grad_depth / grad_weights_sum [N] and grad_loss_* (scalars or [n_views]) nullable.  Accumulates (+=)
 * into grad_table / grad_mlp.  enc_cache_valid: the workspace still holds this forward's encodings. */
int mi3d_render_backward(const mi3d_render_args* args, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                         const mi3d_field_cfg* cfg, const mi3d_render_ws* ws, const float* grad_image, const float* grad_depth,
                         const float* grad_weights_sum, const float* grad_loss_orient, const float* grad_loss_smooth,
                         float* grad_table, const mi3d_mlp_grad* grad_mlp, void* bwd_workspace, int enc_cache_valid,
                         mi3d_stream_t stream);

/* Evaluation renderer (SURVEY.md 8f-2): the alive-ray loop of NeRFRenderer.run_cuda's non-training branch (nerf/renderer.py:526-551:
 * march_rays -> field -> composite_rays until every ray is terminated or max_steps is reached) in ONE call, all loop state on the
 * device (no per-iteration host synchronisation; the reference compacts the alive list with a boolean mask every iteration).
 * Outputs [N], [N], [N,3], [N,3] are (re)initialised inside and carry the background mix / depth fix-up of renderer.py:553-570.
 * done_flag_host (nullable): int in pinned, device-accessible HOST memory; lets the host stop enqueueing iterations early. */
typedef struct {
    const float* rays_o;          /* [N,3] */
    const float* rays_d;          /* [N,3] */
    const float* depth_scale;     /* [N] or NULL */
    uint32_t N;
    const uint8_t* density_bitfield;
    uint32_t C, H;
    float bound, dt_gamma;
    uint32_t max_steps;           /* 1024 in the reference's eval calls */
    float min_near;               /* 0.2 (wrapper default, raymarching.py:34) */
    const float* aabb;            /* device [6]: aabb_infer */
    float T_thresh;               /* 1e-4 (renderer.py:483 default passed to composite_rays) */
    int perturb;                  /* jitter the first march iteration */
    uint64_t seed;
    const float* bg_color;        /* device [3] or NULL -> bg_scalar */
    float bg_scalar;
    float max_depth;
} mi3d_render_eval_args;
size_t mi3d_render_eval_workspace_bytes(uint32_t N);
int mi3d_render_eval(const mi3d_render_eval_args* args, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                     const mi3d_field_cfg* cfg, void* workspace, int* done_flag_host, float* weights_sum, float* depth, float* image,
                     float* normal, mi3d_stream_t stream);

/* Replaces NeRFRenderer.update_extra_state (nerf/renderer.py:587-637): density_grid [C,H^3] EMA-max update from the
 * field at jittered cell centres, mean density (device scalar out), bitfield repack.  jitter: [C,H^3,3] U[0,1) or NULL
 * (Philox).  workspace: mi3d_density_grid_workspace_bytes(C,H). */
size_t mi3d_density_grid_workspace_bytes(uint32_t C, uint32_t H);
int mi3d_density_grid_update(float* density_grid, uint8_t* density_bitfield, uint32_t C, uint32_t H, float bound,
                             float decay, float density_thresh, const float* table, const mi3d_hashgrid* hg,
                             const mi3d_mlp* mlp, const mi3d_field_cfg* cfg, const float* jitter, uint64_t seed,
                             float* mean_density_out, void* workspace, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Parameter update that follows the hot path (SURVEY.md 8f-1): nn.utils.clip_grad_norm(max_norm) (nerf/utils.py:984) +
 * Adan.step() with its own global-norm clip (optimizer.py:102-198) + _single_tensor_adan (optimizer.py:201-256) in one
 * elementwise kernel over a flat (shard of a) parameter vector.  The global gradient norm stays on the device.
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    double lr;              /* group['lr'] (python floats of the reference are doubles; the host folds them in double) */
    double beta1, beta2, beta3, eps, weight_decay;     /* (0.98, 0.92, 0.99), 1e-8, 2e-5 (main.py:132) */
    float max_grad_norm;    /* Adan's global clip, 5.0; 0 = off */
    float clip_grad_norm;   /* Trainer's clip_grad_norm max_norm, 10; 0 = off */
    int no_prox;
    int step;               /* group['step'] AFTER the increment: 1 on the first call */
    int reset_prev;         /* != 0: treat neg_pre_grad as missing (optimizer.py:160) */
} mi3d_adan_cfg;
/* out (+)= sum(g[i]^2), deterministic (fixed-order partials, fp64 fold).  g 16-byte aligned.  workspace: mi3d_sumsq_workspace_bytes(). */
size_t mi3d_sumsq_workspace_bytes(void);
int mi3d_sumsq(const float* g, uint64_t n, float* out, int accumulate, void* workspace, mi3d_stream_t stream);
/* total_sumsq: DEVICE scalar = squared L2 norm of ALL gradients of the model before any clipping (every rank passes the global
 * value).  grad is rescaled in place like the reference does (p.grad ends up clipped); all state tensors are updated in place. */
int mi3d_adan_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* exp_avg_diff, float* neg_pre_grad, uint64_t n,
                   const float* total_sumsq, const mi3d_adan_cfg* cfg, mi3d_stream_t stream);

/* nn.utils.clip_grad_norm(max_norm) (nerf/utils.py:984) + torch.optim.Adam.step() (main.py:133-134: `--optim adam|adamw`) on one
 * parameter tensor, for a caller that launches once per tensor of the model. */
typedef struct {
    double lr;              /* group['lr'] */
    double beta1, beta2, eps;   /* (0.9, 0.99), 1e-15 (main.py:134) */
    int step;               /* the tensor's state['step'] AFTER the increment: 1 on the first call */
    float clip_grad_norm;   /* Trainer's clip_grad_norm max_norm, 10; 0 = off */
} mi3d_adam_cfg;
/* total_sumsq: DEVICE scalar = squared L2 norm of ALL gradients of the model before clipping (mi3d_sumsq over every tensor); may be
 * NULL when clip_grad_norm == 0.  With clip_grad_norm > 0, coef = clamp(clip_grad_norm / (sqrt(*total_sumsq) + 1e-6), max = 1) in
 * fp32 and grad is rescaled in place (p.grad ends up clipped, as torch's clip_grad_norm_ leaves it).  Then torch's _multi_tensor_adam
 * (capturable=False, amsgrad off, no weight decay) in its operation order: exp_avg.lerp_(g, 1 - beta1), exp_avg_sq.mul_(beta2)
 * .addcmul_(g, g, 1 - beta2), param.addcdiv_(exp_avg, sqrt(exp_avg_sq) / (1 - beta2^step)^0.5 + eps, -lr / (1 - beta1^step)), the
 * host scalars folded in double.  All n-element fp32 tensors are DEVICE and updated in place. */
int mi3d_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, uint64_t n, const float* total_sumsq,
                   const mi3d_adam_cfg* cfg, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Planned engines: SD (B3), the SD-2 text encoder (B3'), CLIP (B4), the contextual loss (B6), the refine U-Net (B7), DPT (B8) and
 * BLIP-2 (B9).  Each is made by its mi3d_<engine>_workspace_bytes / mi3d_<engine>_create (HOST: bytes of device workspace the engine
 * needs, 0 for a configuration it cannot run; create plans the launch lists inside the caller's workspace, NULL on failure), and all
 * share one handle type and the lifecycle below.  An engine's own entry points return MI3D_ERR_ARG for another engine's handle.
 * ------------------------------------------------------------------------------------------------------ */
typedef struct mi3d_engine* mi3d_engine_t;

void mi3d_engine_destroy(mi3d_engine_t h);
/* The parameter registry, in the engine's state_dict order (its section names the naming).  A '#...' suffix marks a derived copy,
 * written from the base tensor.  param_name: NULL, param_shape: -1 for an index out of range. */
int mi3d_engine_num_params(mi3d_engine_t h);
const char* mi3d_engine_param_name(mi3d_engine_t h, int i);
int mi3d_engine_param_shape(mi3d_engine_t h, int i, int* shape4); /* returns rank */
/* src = fp32 DEVICE tensor in torch's layout (for a '#' entry: the base tensor); it may be freed once the stream has passed the call.
 * partner_src (nullable): the second tensor of a pair written together, the ".bias" of an SD GEGLU proj weight.  The refine U-Net
 * reads its parameters on every call instead (MI3D_ERR_ARG). */
int mi3d_engine_load_param(mi3d_engine_t h, int i, const float* src, const float* partner_src, mi3d_stream_t stream);
/* CUDA-graph replay of the engine's static launch lists: from its third call on a list is one cudaGraphLaunch.  `stream` of the
 * run calls must then be capturable (not the legacy default stream).  Off by default.  graph_replays: lists currently instantiated. */
int mi3d_engine_set_graph_replay(mi3d_engine_t h, int enable);
int mi3d_engine_graph_replays(mi3d_engine_t h);
/* debug tap: device pointer + size of a named intermediate inside the workspace (the engine's section lists the names) */
int mi3d_engine_debug_tensor(mi3d_engine_t h, const char* name, void** ptr, size_t* bytes);

/* ------------------------------------------------------------------------------------------------------
 * B3: Stable-Diffusion guidance  (replaces the diffusers/cuDNN/cuBLAS calls behind nerf/sd.py:117-174, :212-220)
 * ------------------------------------------------------------------------------------------------------ */

/* The op layer every planned engine is built on, one op at a time: the test surface of the tensor-core tile kernel (wgmma with
 * register accumulators + TMA operand staging; the GEMMs and implicit 3x3 convs that stand in for cuBLAS / cuDNN under diffusers'
 * UNet2DConditionModel / AutoencoderKL, nerf/sd.py:146, :217), of the fused attention and of the row kernels.  Each call records one
 * op through the same plan::Builder / plan::TowerBuilder method the engines call (block-N choice, split-K planning, m_valid and
 * tensor-map encoding included) and runs it eagerly on `stream`.
 * mi3d_op_gemm: y = alpha * A . B^T + bias[N] + row_bias[m / rows_per_group] (+ residual), A [a_rows][K] and B [N][K] fp16 K-major,
 * out fp16 (out16) or fp32 (out32).  mode: 0 plain, 1 GEGLU (rows of B interleaved value / gate; out is [M, N/2]), 2 transposed
 * store (out is [N, M]), 3 / 4 quick-GELU and its input gradient (aux: the pre-activation), 7 GELU.
 * plan (nullable, int[2]): receives the tile kernel's block-N and split count the builder planned.
 * splitk_ws / splitk_bytes: the fp32 split-K scratch the builder may plan into (NULL / 0: no split-K). */
typedef struct {
    const void* a; long long lda, a_rows; int K; int a_z1; long long a_sz1; int a_z2; long long a_sz2;   /* Builder::Mat of A */
    const void* b; long long ldb, b_rows; int b_z1; long long b_sz1; int b_z2; long long b_sz2;          /* Builder::Mat of B */
    int N, batch, b_batched;
    void* out16; void* out32; long long ldc; int out_z1; long long out_s_lo, out_s_hi;                   /* Builder::Out */
    const float* bias; const float* row_bias; int rows_per_group; const void* residual; long long ld_res;   /* Builder::Epi */
    int mode; float alpha; void* aux;
} mi3d_op_gemm_args;
int mi3d_op_gemm(const mi3d_op_gemm_args* g, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream);
/* Builder::conv3: x [Nimg,H,W,Cin], w [Cout][3][3][Cin], y [Nimg,H,W,Cout]; row_bias [Nimg][Cout] (one row per image) */
int mi3d_op_conv3(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const float* bias, const float* row_bias,
                  const void* residual, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream);
/* Builder::conv3_s2 (3x3 stride 2 as im2col + GEMM): x [Nimg,H,W,C], w [Cout][3][3][C], y [Nimg,Ho,Wo,Cout]; pad_lo 1 (padding 1) or 0
 * (padding (0, 1, 0, 1)).  col: at least Nimg*Ho*Wo*9*C fp16 for the im2col matrix, which is left there. */
int mi3d_op_conv3_s2(const void* x, const void* w, void* y, int Nimg, int H, int W, int C, int Ho, int Wo, int Cout, const float* bias, int pad_lo,
                     void* col, size_t col_bytes, void* splitk_ws, size_t splitk_bytes, int* plan, mi3d_stream_t stream);
/* Builder::conv_small_cin: x fp16 [Nimg,H,W,Cin] (Cin 4 or 8), w fp32 [Cout][3][3][Cin], y fp16 [Nimg,H,W,Cout] (Cout % 8 == 0).
 * Builder::conv_small_cout: x fp16 [Nimg,H,W,Cin] (Cin % 8 == 0), w fp16 [Cout][3][3][Cin] (Cout 4 or 8), y fp32 [Nimg,H,W,Cout].
 * Both 3x3 stride 1 padding 1; bias nullable. */
int mi3d_op_conv_small_cin(const void* x, const float* w, const float* bias, void* y, int Nimg, int H, int W, int Cin, int Cout, mi3d_stream_t stream);
int mi3d_op_conv_small_cout(const void* x, const void* w, const float* bias, float* y, int Nimg, int H, int W, int Cin, int Cout,
                            mi3d_stream_t stream);
/* Builder::conv3_block (any H x W): mode 0 plain (+ residual), 5 ReLU, 6 ReLU input gradient masked by aux > 0 */
int mi3d_op_conv3_block(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const float* bias, int mode,
                        const void* aux, const void* residual, int* plan, mi3d_stream_t stream);
/* TowerBuilder attention on the packed qkv [B*Tpad][3C] of a block (C = 64 heads): mode 0 the fused attention as block_fwd calls it,
 * 1 attention_materialised, 2 attention_materialised causal.  Writes o [B*Tpad][C]; modes 1, 2 also need qkvT [B][3C][Tpad] and
 * S [B*heads][Tpad][Tpad] (left holding P). */
int mi3d_op_attention(const void* qkv, void* qkvT, void* S, void* o, int B, int T, int Tpad, int heads, int mode, mi3d_stream_t stream);
/* Builder::attention_core as the SD engine calls it: the fused attention for head_dim 40, 64, 80 or 160 (SD-2.x: 64 at every level;
 * SD-1.x: 40, 80, 160), o = softmax(q k^T / sqrt(head_dim)) v.  q [B*T, ldq], k / v [B*Tk, ldk / ldv], o [B*T, ldo], fp16, head h
 * at columns [h*head_dim, (h+1)*head_dim); only the first Tk_valid keys of every batch take part.  All ld % 8 == 0.  Any other
 * head_dim returns MI3D_ERR_ARG. */
int mi3d_op_attention_core(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                           int B, int T, int Tk, int Tk_valid, int heads, int head_dim, mi3d_stream_t stream);
/* row kernels with the engines' launch geometry: Builder::layernorm, clipk::k_layernorm_bwd (add nullable), Builder::softmax
 * (causal_tq > 0: clipk::k_softmax_causal over [rows / tq][tq][cols]), sdk::k_softmax_bwd, Builder::transpose ([Z][R][C] -> [Z][C][R]) */
int mi3d_op_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, int C, float eps, mi3d_stream_t stream);
int mi3d_op_layernorm_bwd(const void* x, const void* dy, const float* gamma, const void* add, void* dx, int rows, int C, float eps,
                          mi3d_stream_t stream);
int mi3d_op_softmax(void* s, size_t rows, int cols, int valid, int causal_tq, float scale, mi3d_stream_t stream);
int mi3d_op_softmax_bwd(const void* p, void* dp, size_t rows, int cols, float scale, mi3d_stream_t stream);
int mi3d_op_transpose(const void* in, void* out, int Z, int R, int C, mi3d_stream_t stream);
/* The SD engine's own kernels with the launch geometry it plans (sd_engine.cu).
 * mi3d_op_groupnorm: y = GroupNorm(+SiLU when silu) of x fp16 NHWC [N][HW][C] in G groups; stats: [N][G][2] doubles, zeroed by the caller,
 * left holding each group's (sum, sum of squares).  mi3d_op_groupnorm_bwd: dx = the input gradient of dy (+ add, nullable) given the
 * forward's stats; bstats: [N][G][2] zeroed doubles, left holding each group's sums of dg and dg * xhat (dg = dy * silu'(z) * gamma).
 * geom (nullable, int[3]): the planned CTAs per image, pixels per CTA and pixel lanes per CTA. */
int mi3d_op_groupnorm(const void* x, void* y, double* stats, const float* gamma, const float* beta, int N, int HW, int C, int G, float eps,
                      int silu, int* geom, mi3d_stream_t stream);
int mi3d_op_groupnorm_bwd(const void* x, const void* dy, const double* stats, double* bstats, const float* gamma, const float* beta,
                          const void* add, void* dx, int N, int HW, int C, int G, float eps, int silu, int* geom, mi3d_stream_t stream);
/* dx [N,H,W,C] of Builder::conv3_s2 from the gradient dcol [N*Ho*Wo][9*C] of its im2col matrix */
int mi3d_op_col2im_s2(const void* dcol, void* dx, int N, int H, int W, int C, int Ho, int Wo, int pad_lo, mi3d_stream_t stream);
/* The time-embedding linears: y_i[b][n] = bias_i[n] + sum_k act(x[b][k]) W_i[n][k] for b < B, x fp32 [B][K], W_i fp16 [N_i][K], y_i fp32
 * [B][N_i], bias_i nullable.  grouped 0: one layer (layers = 1) with optional SiLU on x and on y; grouped 1: the per-ResBlock projections,
 * `layers` of them in one launch, SiLU on x (silu_in = 1, silu_out = 0).  w, bias, y, N: host arrays of `layers` entries. */
int mi3d_op_linear_small(const float* x, const void* const* w, const float* const* bias, float* const* y, const int* N, int layers, int B, int K,
                         int silu_in, int silu_out, int grouped, mi3d_stream_t stream);
/* The per-view latent kernels of mi3d_sd_encode / _backward and mi3d_sd_unet_sds, for G views (view v: the v-th slice of every per-view
 * tensor): bilinear resize of rgb [G][3][H][W] to out fp16 [G][S][S][4] (2x - 1) and its input gradient from g fp32 [G][S*S][4];
 * the posterior sample latents [G][4][pix] from conv_out [G][pix][8] through quant_conv (qw [8][8], qb [8]) and eps [G][4][pix], and
 * its gradient g_conv_out [G][pix][8]; the noised U-Net input xin fp16 [2G][pix][4] (rows v and G + v of view v); CFG and the SDS
 * gradient from unet_out [2G][pix][4] into noise_pred / grad [G][4][pix] (each nullable).  t: device int64 timestep. */
int mi3d_op_interp_in(const float* rgb, int H, int W, void* out, int S, int G, mi3d_stream_t stream);
int mi3d_op_interp_bwd(const float* g, int S, float* grad_rgb, int H, int W, int G, mi3d_stream_t stream);
int mi3d_op_sample_latents(const float* conv_out, const float* qw, const float* qb, const float* eps, float* latents, int pix, int G,
                           mi3d_stream_t stream);
int mi3d_op_sample_latents_bwd(const float* conv_out, const float* qw, const float* qb, const float* eps, const float* g_lat, float* g_conv_out,
                               int pix, int G, mi3d_stream_t stream);
int mi3d_op_add_noise(const float* latents, const float* noise, const float* alphas_cumprod, const long long* t, void* xin, int pix, int G,
                      mi3d_stream_t stream);
int mi3d_op_cfg_sds(const float* unet_out, const float* noise, const float* alphas_cumprod, const long long* t, float guidance_scale,
                    float* noise_pred, float* grad, int pix, int G, mi3d_stream_t stream);

/* Stable-Diffusion engine: a statically planned launch list over the tile kernel above + memory-bound kernels.
 * Configuration mirrors diffusers' UNet2DConditionModel / AutoencoderKL config.json fields that nerf/sd.py:41,53 load. */
typedef struct {
    int in_ch, out_ch;        /* 4, 4 */
    int n_levels;             /* len(block_out_channels): 4 for SD-2.0-base; 0 = no U-Net in this engine */
    int block_out[4];         /* 320, 640, 1280, 1280 */
    int layers_per_block;     /* 2 */
    int heads[4];             /* SD-2.x: 5, 10, 20, 20 (head_dim 64); SD-1.x: 8, 8, 8, 8 (head_dim 40, 80, 160); head_dim 40 / 64 / 80 / 160 */
    int cross_dim;            /* 1024 (SD-1.x: 768) */
    int ctx_len;              /* 77 text tokens */
    int groups;               /* 32 */
    int latent_hw;            /* 64 (nerf/sd.py:124 always feeds 512x512 -> 64x64 latents) */
    int batch;                /* 2G: [uncond_0..uncond_{G-1}, text_0..text_{G-1}] for G views at one timestep (nerf/sd.py:143 is G = 1); the
                                 sampler (mi3d_sd_sample) is planned at batch 2 only */
    int proj_conv;            /* transformer proj_in / proj_out: 0 = Linear [C, C] (SD-2.x, use_linear_projection), 1 = 1x1 Conv2d
                                 [C, C, 1, 1] (SD-1.x); the same GEMM either way, only the registered parameter shape differs */
} mi3d_unet_cfg;

typedef struct {
    int in_ch, latent_ch;     /* 3, 4 */
    int n_levels;             /* 4; 0 = no VAE in this engine */
    int block_out[4];         /* 128, 256, 512, 512 */
    int layers_per_block;     /* 2 */
    int groups;               /* 32 */
    int image_hw;             /* 512 */
    int decoder;              /* != 0: also plan the decoder (mi3d_sd_decode; the denoise side branch of nerf/sd.py:153-159) */
    int batch;                /* images per encode / encode backward (G); 0 or 1 = one image.  The decoder always takes one image. */
} mi3d_vae_cfg;

/* weights + activations + tapes; nothing else is ever allocated */
size_t mi3d_sd_workspace_bytes(const mi3d_unet_cfg* unet, const mi3d_vae_cfg* vae);
mi3d_engine_t mi3d_sd_create(const mi3d_unet_cfg* unet, const mi3d_vae_cfg* vae, void* workspace, size_t workspace_bytes);
/* Parameters are enumerated by their diffusers state_dict names ("down_blocks.0.resnets.0.conv1.weight", VAE names are
 * prefixed as in AutoencoderKL: "encoder....", "quant_conv....").  Graph replay covers the static launch lists (U-Net,
 * VAE encode, VAE input-gradient, VAE decode, sampling step).  Debug taps: "unet.mid", "vae.grad_in", ... */

/* replaces nerf/sd.py:124 (F.interpolate to 512) + :133,212-220 (encode_imgs: vae.encode(2x-1).latent_dist.sample()*0.18215), for the
 * G = mi3d_vae_cfg.batch images the engine is planned for, each on its own (convs, GroupNorm and the mid-block attention are per image).
 * pred_rgb [G,3,H,W] fp32 in [0,1]; eps_posterior, latents [G,4,h,w] fp32 (h = image_hw/8). */
int mi3d_sd_encode(mi3d_engine_t h, const float* pred_rgb, int H, int W, const float* eps_posterior, float* latents, mi3d_stream_t stream);
/* the autograd half of latents.backward(gradient=grad) (nerf/sd.py:171): d latents -> d pred_rgb, weights frozen; [G,...] buffers as above */
int mi3d_sd_encode_backward(mi3d_engine_t h, const float* grad_latents, const float* eps_posterior, int H, int W, float* grad_pred_rgb,
                            mi3d_stream_t stream);
/* replaces nerf/sd.py:138-170: scheduler.add_noise, unet([x,x], t, text_embeddings).sample, CFG (text + gs*(text-uncond)),
 * w = 1 - alphas[t], grad = nan_to_num(w*(noise_pred - noise)), for G = mi3d_unet_cfg.batch / 2 views at ONE shared timestep.
 * t: DEVICE int64 scalar; alphas_cumprod: DEVICE fp32 [1000]; latents / noise fp32 [G,4,h,w]; text_embeddings fp32 [2G,77,cross_dim]
 * laid out [uncond_0..uncond_{G-1}, cond_0..cond_{G-1}] (view v's CFG pairs U-Net rows v and G+v); noise_pred / grad (nullable)
 * fp32 [G,4,h,w]. */
int mi3d_sd_unet_sds(mi3d_engine_t h, const float* latents, const float* noise, const long long* t, const float* alphas_cumprod,
                     const float* text_embeddings, float guidance_scale, float* noise_pred, float* grad, mi3d_stream_t stream);
/* The "denoise" side branch of train_step (nerf/sd.py:153-159), taken on non-large views when t <= 0.4 T:
 * replaces scheduler.step (DDIM, eta 0, t -> t-1; fp32 [G,4,h,w], n = 4*h*w*G elements, element-wise) and decode_latents (nerf/sd.py:201-210:
 * vae.decode(latents / 0.18215) -> (x/2 + 0.5).clamp(0,1); imgs fp32 [1,3,image_hw,image_hw]).  Forward only, like the reference. */
int mi3d_sd_ddim_step(const float* noise_pred, const float* latents_noisy, const long long* t, const float* alphas_cumprod,
                      float* prev_sample, int n, mi3d_stream_t stream);
int mi3d_sd_decode(mi3d_engine_t h, const float* latents, float* imgs, mi3d_stream_t stream);
/* Text-to-latents sampling (produce_latents, nerf/sd.py:176-199): DDIM with eta 0 and classifier-free guidance, n steps without the
 * host.  One entry of the schedule per step, built by the caller from the scheduler config: t (the U-Net timestep), alpha_t =
 * alphas_cumprod[t] and alpha_prev = alphas_cumprod[t - T/n], or final_alpha_cumprod when t - T/n < 0. */
typedef struct {
    long long t;
    float alpha_t, alpha_prev;
} mi3d_sd_schedule;
/* latents: DEVICE fp32 [1,4,h,w], x_T in, x_0 out.  sched: DEVICE table of n entries (1 <= n <= 1000).  prediction_type: 0 epsilon,
 * 1 v_prediction.  text_embeddings fp32 [2,77,cross_dim] (uncond first).  Per step: [x, x] -> U-Net at t_i -> CFG
 * (text + gs*(text - uncond), as the reference writes it) -> DDIMScheduler.step (clip_sample off) written back in place; the step body
 * is one static launch list that replays as a CUDA graph when graph replay is on.  Nothing is read back to the host. */
int mi3d_sd_sample(mi3d_engine_t h, float* latents, const mi3d_sd_schedule* sched, int n, int prediction_type, const float* text_embeddings,
                   float guidance_scale, mi3d_stream_t stream);
/* live timing of the tensor-core tile kernel: enable=1 starts recording CUDA events around every launch; enable=0 stops and
 * returns the summed kernel time (ms) and launch count (HOST pointers; synchronises on the recorded events). */
int mi3d_sd_profile(mi3d_engine_t h, int enable, float* gemm_ms_host, int* launches_host);
/* same, and (enable=0) also writes one text line per timed launch to dump_path_host: "M N K block_n splits conv batch epi ms" */
int mi3d_sd_profile_dump(mi3d_engine_t h, int enable, float* gemm_ms_host, int* launches_host, const char* dump_path_host);

/* ------------------------------------------------------------------------------------------------------
 * B3': Stable Diffusion text encoder  (replaces transformers' CLIPTextModel behind get_text_embeds, nerf/sd.py:68-85: OpenCLIP
 * ViT-H/14's text tower truncated to 23 layers, as every SD-2.x checkpoint ships it, or OpenAI CLIP ViT-L/14's, as SD-1.x ships it)
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    int width, layers, heads;  /* 1024, 23, 16 (SD-1.x: 768, 12, 12); head_dim 64; MLP width 4 x width */
    int context_len, vocab;    /* 77, 49408 */
    int max_batch;             /* prompts per call (1..8); 2 encodes [negative, positive] in one pass */
} mi3d_sd_text_cfg;

/* The MLP activation is exact-erf GELU (SD-2.x, OpenCLIP ViT-H/14) */
size_t mi3d_sd_text_workspace_bytes(const mi3d_sd_text_cfg* cfg);
mi3d_engine_t mi3d_sd_text_create(const mi3d_sd_text_cfg* cfg, void* workspace, size_t workspace_bytes);
/* The same engine with the MLP activation chosen by act: 0 = exact-erf GELU (SD-2.x; the two calls above), 1 = quick-GELU
 * x * sigmoid(1.702 x) (SD-1.x, OpenAI CLIP ViT-L/14's text tower); any other value is invalid (0 bytes / NULL). */
size_t mi3d_sd_text_act_workspace_bytes(const mi3d_sd_text_cfg* cfg, int act);
mi3d_engine_t mi3d_sd_text_act_create(const mi3d_sd_text_cfg* cfg, int act, void* workspace, size_t workspace_bytes);
/* Parameters are enumerated by transformers' CLIPTextModel state_dict names, in its order ("text_model.embeddings.token_embedding.weight"
 * .. "text_model.final_layer_norm.bias"; no position_ids).  The separate q / k / v projections are stored as row slices of one packed
 * weight. */
/* ids int64 [B,context_len] (DEVICE) -> out fp32 [B,context_len,width] (DEVICE): last_hidden_state, final_layer_norm applied to every
 * position.  Causal attention, no padding mask.  Ids outside [0, vocab) are clamped into it.  B <= max_batch. */
int mi3d_sd_text_encode(mi3d_engine_t h, const long long* ids, int B, float* out, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B4: CLIP losses  (replaces openai CLIP's encode_image / encode_text behind the per-step CLIP losses, nerf/utils.py:436-453, 561-563,
 * and the denoise branch's, nerf/sd.py:97-114, 157-158)
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    int image_res, patch;      /* 224, 16 */
    int width, layers, heads;  /* image tower: 768, 12, 12 (head_dim 64); layers = 0: no image tower in this engine */
    int embed_dim;             /* 512: output features of both towers */
    int context_len, vocab;    /* 77, 49408 */
    int text_width, text_layers, text_heads;   /* 512, 12, 8; text_layers = 0: no text tower in this engine */
    int max_batch;             /* images / prompts per call (1..8); 2 encodes [rendered, reference] in one pass */
} mi3d_clip_cfg;

size_t mi3d_clip_workspace_bytes(const mi3d_clip_cfg* cfg);
mi3d_engine_t mi3d_clip_create(const mi3d_clip_cfg* cfg, void* workspace, size_t workspace_bytes);
/* Parameters are enumerated by openai CLIP's state_dict names ("visual.conv1.weight", "transformer.resblocks.0.attn.in_proj_weight",
 * "visual.proj", ...), in openai's layout. */
/* img fp32 [B,3,H,W] -> feats fp32 [B,embed_dim] (encode_image).  aug != 0: the reference's aug first (Resize((res,res)): bilinear,
 * align_corners=False, no antialiasing; then Normalize with CLIP's mean / std); aug = 0: img is already augmented and res x res.
 * need_grad != 0 keeps a tape for mi3d_clip_encode_image_backward; any image forward replaces the previous tape.  B <= max_batch. */
int mi3d_clip_encode_image(mi3d_engine_t h, const float* img, int B, int H, int W, int aug, int need_grad, float* feats, mi3d_stream_t stream);
/* input gradient of the first n_grad images of the last (taped) image forward: dfeats fp32 [n_grad,embed_dim] -> dimg fp32
 * [n_grad,3,H,W] (overwritten).  Weights frozen.  MI3D_ERR_ARG without a tape or with n_grad outside 1..B of that forward. */
int mi3d_clip_encode_image_backward(mi3d_engine_t h, const float* dfeats, int n_grad, float* dimg, mi3d_stream_t stream);
/* tokens int64 [B,context_len] (clip.tokenize ids; the features are taken at each row's argmax, the EOT token) -> feats fp32
 * [B,embed_dim] (encode_text, causal attention).  Ids outside [0, vocab) are clamped into it. */
int mi3d_clip_encode_text(mi3d_engine_t h, const long long* tokens, int B, float* feats, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B5: refine-stage point renderer  (replaces pytorch3d's rasterize_points + alpha_composite as render_point drives them,
 * nerf/refine_utils.py:306-333, and the Python loop of z_buffer, refine_utils.py:167-208)
 * ------------------------------------------------------------------------------------------------------ */
/* HOST: workspace bytes of mi3d_points_render_forward for P points rasterised at H x W with NDC radius `radius` (0: invalid
 * arguments).  The bin lists are sized from a bound on the screen tiles one point can touch, so they cannot overflow. */
size_t mi3d_points_workspace_bytes(uint32_t P, uint32_t H, uint32_t W, double radius);
/* points [P,3], feats [P,C] (C in 1..32) fp32; cam_k [9] (row-major K) and world2cam [12] (rows 0..2 of the pose, R | t) are DEVICE
 * fp32 buffers.  Projection: c = R p + t, q = K c, u = q.x / q.z, x_ndc = -(u / proj_w * 2 - 1) (same for y with proj_h), z = q.z.
 * Naive pytorch3d rasterisation of an H x W image (H == W, else MI3D_ERR_ARG): pixel (y, x) has the NDC centre
 * (-1 + (2(W-1-x)+1)/W, -1 + (2(H-1-y)+1)/H); a point with z >= 0 covers it when dist2 < r*r (fp32 r = radius); each pixel keeps the
 * K (1..16) covering points with the smallest (z, index), ascending, empty slots -1.  alpha = 1 - sqrt(clamp(0.1 dist2 / fp32(radius^2),
 * 1e-3, 1)); image [1,C,H,W] = front-to-back alpha composite over the slots, background 0.
 * Outputs [H,W,K]: idx (required), w = T * alpha (the backward's weights; required with image), zbuf / dist2 (nullable, -1 when empty).
 * image == NULL rasterises only (feats unused).  workspace: mi3d_points_workspace_bytes() bytes. */
int mi3d_points_render_forward(const float* points, const float* feats, uint32_t P, uint32_t C, const float* cam_k, const float* world2cam,
                               float proj_w, float proj_h, uint32_t H, uint32_t W, double radius, uint32_t K, float* image, int* idx,
                               float* w, float* zbuf, float* dist2, void* workspace, size_t workspace_bytes, mi3d_stream_t stream);
/* grad_feats [P,C] (overwritten) = sum over the (pixel, slot) pairs holding each point of grad_image[c, pixel] * w; idx / w from the
 * forward with the same points and camera.  No gradient for points, radius or background (the reference requests none). */
int mi3d_points_render_backward(const float* points, uint32_t P, uint32_t C, const float* cam_k, const float* world2cam, float proj_w,
                                float proj_h, uint32_t H, uint32_t W, double radius, uint32_t K, const int* idx, const float* w,
                                const float* grad_image, float* grad_feats, mi3d_stream_t stream);
/* z_buffer visibility in fp64: project points [P,3] with DEVICE cam_k [9] / world2cam [12], (x, y) = rint(u, v) (half to even);
 * mask[i] (uint8) = in image && !(z_i - min z of the in-image points in that pixel > 1/H).  zbuf: DEVICE scratch of H*W uint64. */
int mi3d_points_zbuffer_visible(const double* points, uint32_t P, const double* cam_k, const double* world2cam, uint32_t H, uint32_t W,
                                unsigned long long* zbuf, uint8_t* mask, mi3d_stream_t stream);

/* B5, point-cloud construction (load_views, nerf/refine_utils.py:61-152, :335-410; csrc/views.cu, oracle/views_ref.py).  Square
 * H x W views only (H == W, else MI3D_ERR_ARG).  Images are row-major uint8 / uint16 [H,W]; depth is depth_u16 / 1000.0.
 * HOST: workspace bytes shared by the calls below (0: invalid size). */
size_t mi3d_views_workspace_bytes(uint32_t H, uint32_t W);
/* out[p] (0/1) = mask eroded with erode_k x erode_k == 255 (cv2.erode, window clipped to the image), and, when canny_thresh >= 0, not
 * within the dilate_k x dilate_k dilation of Canny(uint8(depth * eroded * 255) wrapped modulo 256, canny_thresh, canny_thresh).
 * Nullable outputs: masked_depth fp32 [H,W] = float32(depth * out); eroded (raw min), edges (0/255), dilated (0/255).  Odd k <= 31. */
int mi3d_views_mask(const uint16_t* depth, const uint8_t* mask, uint32_t H, uint32_t W, uint32_t erode_k, int canny_thresh, uint32_t dilate_k,
                    uint8_t* out, float* masked_depth, uint8_t* eroded, uint8_t* edges, uint8_t* dilated, void* workspace,
                    size_t workspace_bytes, mi3d_stream_t stream);
/* out[p] (0/1) = alphamask[p] == 1 and not covered, where covered = the erode_k x erode_k erosion of (uint8(render * 255) / 255 > 0.9);
 * render fp32 [H,W] (one channel of the canonical cloud rendered with unit colours).  quant (nullable) = uint8(render * 255). */
int mi3d_views_cover_mask(const float* render, const uint8_t* alphamask, uint32_t H, uint32_t W, uint32_t erode_k, uint8_t* out, uint8_t* quant,
                          void* workspace, size_t workspace_bytes, mi3d_stream_t stream);
/* points fp64 [H*W,3]: the world points (inv(K) [x, y, 1] D, then c2w) of the pixels with mask != 0, in row-major pixel order, and
 * count (DEVICE int32) of them; rows [count, H*W) are NaN.  kinv [9], c2w [12] (rows 0..2 of the pose) are DEVICE fp64.  With
 * cano_depth (fp32 [H,W], DEVICE), cam_k [9] and cano_w2c [12]: points whose canonical projection, rounded half to even, samples
 * (bilinear, zero padding, align_corners=False) a depth d with -0.2 <= z - d <= 1/H are dropped. */
int mi3d_views_backproject(const uint16_t* depth, const uint8_t* mask, uint32_t H, uint32_t W, const double* kinv, const double* c2w,
                           const double* cam_k, const double* cano_w2c, const float* cano_depth, double* points, int* count, void* workspace,
                           size_t workspace_bytes, mi3d_stream_t stream);
/* points_out fp64 [count,3] = points[keep != 0] in order (P <= H*W) and colours fp32 [count,3] sampled bilinearly at their projection
 * through cam_k / world2cam (DEVICE fp64) from exactly one of img_f32 [H,W,3] or img_u8 [H,W,3] (read as u8 / 255.0).  count: DEVICE. */
int mi3d_views_compact_colour(const double* points, uint32_t P, const uint8_t* keep, const double* cam_k, const double* world2cam,
                              const float* img_f32, const uint8_t* img_u8, uint32_t H, uint32_t W, double* points_out, float* colours,
                              int* count, void* workspace, size_t workspace_bytes, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B6: refine-stage contextual loss  (replaces the contextual_loss package's ContextualLoss(use_vgg=True, vgg_layer='relu5_4',
 * loss_type='cosine'), nerf/utils.py:36, 455-457, 810, 882)
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    int N, H, W;               /* images per call (1..16) and their size (16..4096 each): the plan is static for this shape */
} mi3d_cx_cfg;

size_t mi3d_cx_workspace_bytes(const mi3d_cx_cfg* cfg);
mi3d_engine_t mi3d_cx_create(const mi3d_cx_cfg* cfg, void* workspace, size_t workspace_bytes);
/* Parameters carry the package's state_dict names, "vgg_model.slice1.0.weight" .. "vgg_model.slice5.34.bias" (the '#dgrad' copy of
 * conv1_1 is written when its base tensor is loaded; loading the '#dgrad' entry itself does nothing).  Debug tap: "relu5_4", fp16
 * NHWC [2N,H/16,W/16,512], the x images first. */
/* x, y fp32 [N,3,H,W] -> loss: DEVICE fp32 scalar.  ImageNet normalisation, VGG19 features[0:36] of x and y in one batched pass
 * (fp16 storage, fp32 accumulation), then in fp32: centring by y's channel mean over batch and positions, L2 normalisation,
 * d = 1 - cos, d / (min_j d + 1e-5), w = exp((1 - .) / band_width), cx = w / sum_j w, loss = mean_n -log(mean_j max_i cx + 1e-5).
 * need_grad != 0 keeps the tape for mi3d_cx_backward; any forward replaces it. */
int mi3d_cx_forward(mi3d_engine_t h, const float* x, const float* y, float band_width, int need_grad, float* loss, mi3d_stream_t stream);
/* dx fp32 [N,3,H,W] (overwritten) = dloss * d loss / d x of the last forward; dloss: DEVICE fp32 scalar.  No gradient for y or the
 * weights.  MI3D_ERR_ARG without a tape. */
int mi3d_cx_backward(mi3d_engine_t h, const float* dloss, float* dx, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B7: refine-stage gated U-Net  (replaces the reference's nerf/unet.py UNet(num_input_channels=3+16) with its defaults:
 * feature_scale 4, bilinear upsampling, sigmoid output, gated blocks; nerf/utils.py:808, 863, 937)
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    int N, H, W;               /* images per call (1..16) and the finest level's size (4..4096 each, multiples of 4): the plan is static */
} mi3d_unet_shape;

size_t mi3d_unet_workspace_bytes(const mi3d_unet_shape* cfg);
mi3d_engine_t mi3d_unet_create(const mi3d_unet_shape* cfg, void* workspace, size_t workspace_bytes);
/* The registry lists the reference's 41 state_dict entries in its order ("start.block.conv_f.weight" .. "final.0.0.bias"), parameters
 * and BatchNorm buffers alike (shape rank 0: num_batches_tracked); they are passed to every call (state), not loaded.  Debug taps:
 * fp32 NCHW "cat1", "cat2", "d2", "up2", "up1", "out"; "in64" is a channel slice of "cat1". */
/* x0 [N,19,H,W], x1 [N,19,H/2,W/2], x2 [N,19,H/4,W/4] fp32 -> out [N,3,H,W] fp32.  state: one DEVICE pointer per registry entry, in
 * registry order, in torch's layouts: the fp32 parameters are read on every call (no reload after an optimizer step).  train != 0:
 * BatchNorm with batch statistics, and the fp32 running_mean / running_var and the int64 num_batches_tracked given are updated
 * once (momentum 0.1, unbiased variance); a NULL buffer pointer skips its update; MI3D_ERR_ARG when N x H/4 x W/4 < 2 (one value
 * per channel).  train == 0: the running statistics are read.
 * need_grad != 0 keeps the tape for mi3d_unet_backward; any forward replaces it. */
int mi3d_unet_forward(mi3d_engine_t h, const float* x0, const float* x1, const float* x2, void* const* state, int train, int need_grad,
                      float* out, mi3d_stream_t stream);
/* dout fp32 [N,3,H,W] -> dx0, dx1, dx2 (overwritten) and, for every parameter entry whose grads[i] is not NULL, its fp32 gradient
 * (overwritten; buffer entries are ignored), for the last forward.  May run any number of times per forward.  MI3D_ERR_ARG without
 * a tape. */
int mi3d_unet_backward(mi3d_engine_t h, const float* dout, float* dx0, float* dx1, float* dx2, float* const* grads, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B8: DPT-Hybrid depth model  (replaces the reference's DPT/dpt DPTDepthModel(backbone="vitb_rn50_384", non_negative=True) and timm
 * behind the reference image's depth prior, main.py:111-127, 196-214: ResNet-50v2 trunk, ViT-B/16 on 577 tokens, RefineNet decoder)
 * ------------------------------------------------------------------------------------------------------ */
/* one shape: a [1,3,384,384] image; the workspace must be zero-filled (padding rows and channels are never written) */
size_t mi3d_dpt_workspace_bytes(void);
mi3d_engine_t mi3d_dpt_create(void* workspace, size_t workspace_bytes);
/* Parameters are enumerated by the reference's DPTDepthModel.state_dict() names ("pretrained.model.cls_token" ..
 * "scratch.output_conv.4.bias"), every tensor the forward reads and nothing else (not pretrained.model.norm.*, pretrained.model.head.*
 * or scratch.refinenet4.resConfUnit1.*).  The trunk's convs are weight-standardised at load.  The forward always runs eagerly. */
/* img fp32 [1,3,384,384] (resized and normalised, DEVICE) -> out fp32 [1,384,384] inverse depth (DEVICE) */
int mi3d_dpt_forward(mi3d_engine_t h, const float* img, float* out, mi3d_stream_t stream);
/* the last forward's reassembled backbone features layer_1 .. layer_4 (i = 0..3) as fp32 NCHW: [1,256,96,96], [1,512,48,48],
 * [1,768,24,24], [1,768,12,12] */
int mi3d_dpt_tap(mi3d_engine_t h, int i, float* dst, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B9: BLIP-2 captioner  (replaces transformers' Blip2ForConditionalGeneration.generate(pixel_values) with Salesforce/blip2-opt-2.7b
 * behind the caption of the reference image when no --text is given, main.py:158-172: EVA ViT-g/14, Q-Former, greedy OPT-2.7B decode)
 * ------------------------------------------------------------------------------------------------------ */
typedef struct {
    int image_size, patch;                                   /* 224, 14 */
    int vision_width, vision_layers, vision_heads, vision_mlp;   /* 1408, 39, 16, 6144 (head_dim 88; exact GELU; LN eps 1e-6) */
    int qformer_width, qformer_layers, qformer_heads, qformer_ffn, cross_attention_frequency;   /* 768, 12, 12, 3072, 2 */
    int num_query_tokens;                                    /* 32 */
    int opt_width, opt_layers, opt_heads, opt_ffn, vocab;    /* 2560, 32, 32, 10240, 50272 (head_dim 80; ReLU FFN) */
    int max_positions;                                       /* 2048 (embed_positions has max_positions + 2 rows) */
    int image_token_index, bos_token_id, eos_token_id;       /* 50265, 2, 50118 */
} mi3d_blip2_cfg;

/* the workspace must be zero-filled */
size_t mi3d_blip2_workspace_bytes(const mi3d_blip2_cfg* cfg);
mi3d_engine_t mi3d_blip2_create(const mi3d_blip2_cfg* cfg, void* workspace, size_t workspace_bytes);
/* Parameters are enumerated by transformers' Blip2ForConditionalGeneration.state_dict() names, in its order ("query_tokens" ..
 * "language_model.model.decoder.layers.{L-1}.final_layer_norm.bias"), without the tied "language_model.lm_head.weight" (lm_head reads
 * embed_tokens).  OPT's q / k / v projections are stored as row slices of one packed weight. */
/* pixel_values fp32 [1,3,image_size,image_size] (DEVICE, processor-normalised) -> out fp32 [num_query_tokens, opt_width]
 * (language_model_inputs = language_projection(Q-Former(vision(pixel_values)))) */
int mi3d_blip2_encode(mi3d_engine_t h, const float* pixel_values, float* out, mi3d_stream_t stream);
/* Greedy caption: the prompt [image_token_index] x num_query_tokens + [bos_token_id], the query rows replaced by language_model_inputs,
 * then max_new_tokens greedy steps (1 .. 63 - num_query_tokens), each a causal pass over a fixed 64-row window, lm_head on the last
 * filled row only, argmax with the lowest index on ties.  After eos (< 0: none) no token is appended.  ids (DEVICE int64 [64]): the
 * prompt and the generated tokens; count (DEVICE int32 [1]): how many of them are valid (num_query_tokens + 1 + n).
 * forced_ids (DEVICE int64 [max_new_tokens], nullable): teacher forcing, step s appends forced_ids[s] instead of the argmax.
 * step_logits (DEVICE fp32 [max_new_tokens, vocab], nullable): the last-row logits of every step. */
int mi3d_blip2_generate(mi3d_engine_t h, const float* pixel_values, int max_new_tokens, long long eos_token_id, const long long* forced_ids,
                        long long* ids, int* count, float* step_logits, mi3d_stream_t stream);
/* the last call's intermediates as fp32 (DEVICE): "image_embeds" [T, vision_width] (T = (image_size / patch)^2 + 1, post_layernorm
 * applied), "query_output" [num_query_tokens, qformer_width], "language_model_inputs" [num_query_tokens, opt_width] */
int mi3d_blip2_tap(mi3d_engine_t h, const char* name, float* dst, mi3d_stream_t stream);
/* The weight-streaming GEMM on its own: y[M,N] = act(x[M,K] w[N,K]^T + bias (+ residual)), M <= 64, K % 32 == 0; x, w, residual, y
 * fp16, bias fp32 (nullable), relu != 0: ReLU.  workspace: mi3d_stream_gemm_workspace_bytes(M, N, K) bytes (fp32 partial sums). */
size_t mi3d_stream_gemm_workspace_bytes(int M, int N, int K);
int mi3d_stream_gemm_f16(const void* x, const void* w, const float* bias, const void* residual, int relu, void* y, int M, int N, int K,
                         void* workspace, size_t workspace_bytes, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B10: mesh export  (replaces PyMCubes' marching_cubes and the xatlas / nvdiffrast texel pass of NeRFRenderer.export_mesh,
 * nerf/renderer.py:157-330; csrc/mesh.cu, oracle/mesh_ref.py)
 * ------------------------------------------------------------------------------------------------------ */
/* Marching cubes (Bourke / Bloyd 256-case table) over volume fp32 [nx,ny,nz] (C order, (i,j,k) <-> (x,y,z)).  A corner is inside iff
 * sigma > iso_eff with iso_eff = iso, or min(iso, *iso_dev) when iso_dev (DEVICE scalar) is given.  One vertex per crossing grid edge,
 * owned by its lower end point p, at p + t e_a, t = (iso_eff - s_p) / (s_{p+e_a} - s_p) in fp32 without contraction; numbered by grid
 * point (C order), then axis x < y < z.  Faces: cells in C order, triangles in table order, right-hand normal pointing out of the
 * solid (toward sigma <= iso_eff).  Output order depends on the data only (no atomics decide it).
 * workspace: mi3d_mc_workspace_bytes(nx, ny, nz) bytes; 0 (and MI3D_ERR_ARG from the calls) when a dimension is below 2 or a vertex
 * or face count could overflow int32 (3 nx ny nz or 5 (nx-1)(ny-1)(nz-1) above INT32_MAX).
 * mi3d_mc_count writes counts = (V, F) (DEVICE int32 [2]) and fills the workspace; mi3d_mc_emit, on the same workspace, volume and
 * threshold, writes vertices fp32 [V,3] = position * scale + offset and faces int32 [F,3]. */
size_t mi3d_mc_workspace_bytes(uint32_t nx, uint32_t ny, uint32_t nz);
int mi3d_mc_count(const float* volume, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* iso_dev, void* workspace,
                  int* counts, mi3d_stream_t stream);
int mi3d_mc_emit(const float* volume, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* iso_dev, const void* workspace,
                 float scale, float offset, float* vertices, int* faces, mi3d_stream_t stream);
/* Texel pass of the per-face texture atlas (layout: T x T texels, cells of c x c texels, n cells per row, faces 2p / 2p+1 in cell p;
 * nerf/mesh.py::atlas_layout).  points fp32 [T*T,3]: each owned texel centre mapped through its face's affine UV -> xyz map and clamped
 * to [-bound, bound] (0 for unowned texels); owner int32 [T*T]: the face (-1: none); vt fp32 [3F,2]: UVs in [0,1] of the faces' corners
 * (u along texel columns, v along rows). */
int mi3d_mesh_atlas_texels(const float* vertices, const int* faces, uint32_t F, uint32_t T, uint32_t c, uint32_t n, float bound,
                           float* points, int* owner, float* vt, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B11: refine loop glue  (the per-iteration losses and the optimiser step of Trainer.refine, nerf/utils.py:865-894; csrc/refine.cu,
 * oracle/refine_ref.py)
 * ------------------------------------------------------------------------------------------------------ */
/* Image losses of one S x S iteration.  weights fp32 [S,S,ppp]: the scale-0 composite weights mi3d_points_render_forward writes;
 * coverage (nullable) fp32 [S,S] = sum over the ppp slots in slot order, bit-identical to the unit-colour render; dilated fp32 [S,S] =
 * its 5x5 max (MaxPool2d(5, 1, 2)); pred, gt fp32 [1,3,S,S], gt_mask fp32 [1,1,S,S] (gt and gt_mask may be NULL when front == 0).
 * losses fp32 [2] (DEVICE) = (1e-3 * sum(1 - pred (1 - dilated)), front ? 1000 * mean|pred m - gt m| : 0), each summed in fp64 in a
 * fixed order (run-to-run identical).  workspace: mi3d_refine_image_losses_workspace_bytes(S) bytes. */
size_t mi3d_refine_image_losses_workspace_bytes(uint32_t S);
int mi3d_refine_image_losses(const float* weights, uint32_t S, uint32_t ppp, const float* pred, const float* gt, const float* gt_mask,
                             int front, float* coverage, float* dilated, float* losses, void* workspace, size_t workspace_bytes,
                             mi3d_stream_t stream);
/* grad_pred fp32 [1,3,S,S] (overwritten) = d(g0 losses[0] + g1 losses[1]) / d pred with grad_losses = (g0, g1) (DEVICE fp32 [2]) and
 * the dilated mask of the forward, in the operation order of torch's autograd for the same expressions. */
int mi3d_refine_image_losses_backward(const float* pred, const float* gt, const float* gt_mask, const float* dilated, uint32_t S, int front,
                                      const float* grad_losses, float* grad_pred, mi3d_stream_t stream);
/* One parameter tensor of mi3d_refine_adam: n fp32 elements of param / grad / exp_avg / exp_avg_sq (DEVICE), at element `offset` of the
 * concatenation of all segments (offsets ascending, segment 0 at 0, no gaps). */
typedef struct {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    unsigned long long offset, n;
} mi3d_adam_segment;
/* One torch.optim.Adam step (amsgrad off, no weight decay; `step` counts from 1) over every segment of the DEVICE table segs [n_segs]
 * (1..256, total elements in all), in torch's operation order: exp_avg.lerp_(g, 1 - beta1), exp_avg_sq.mul_(beta2).addcmul_(g, g,
 * 1 - beta2), param.addcdiv_(exp_avg, sqrt(exp_avg_sq) / (1 - beta2^step)^0.5 + eps, -lr / (1 - beta1^step)).
 * origin (nullable) fp32 [p_cano + p_novel, 3]: segment 0 is then the refine cloud's [p_cano + p_novel, 19] buffer (cano rows first)
 * and its colour columns 0..2 take the gradient of w_cano MSE(colour_cano, origin_cano) + w_novel MSE(colour_novel, origin_novel)
 * on top of grad; reg (DEVICE fp32 [1]) gets that value for the parameters before the step (an empty region contributes 0).
 * workspace: mi3d_refine_adam_workspace_bytes(total) bytes, needed with origin only. */
size_t mi3d_refine_adam_workspace_bytes(unsigned long long total);
int mi3d_refine_adam(const mi3d_adam_segment* segs, int n_segs, unsigned long long total, double lr, double beta1, double beta2, double eps,
                     int step, const float* origin, uint32_t p_cano, uint32_t p_novel, double w_cano, double w_novel, float* reg,
                     void* workspace, size_t workspace_bytes, mi3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * B12: coarse loop glue  (the per-iteration losses of Trainer.train_step, nerf/utils.py:491-493, :519-533, :551-556;
 * csrc/coarse.cu, oracle/coarse_ref.py)
 * ------------------------------------------------------------------------------------------------------ */
/* Losses of one h x w training render (h, w >= 2).  image fp32 [h*w,3] (ray-major, as the renderer returns it), depth fp32 [h*w]
 * (may be NULL when front == 0), weights_sum fp32 [h*w]; ref_rgba fp32 [1,4,512,512]; bg_color fp32 [3] (DEVICE); depth_prior fp64
 * [512,512] and depth_mask uint8 [512,512] (nonzero = pixel used by the depth term; both may be NULL when front == 0).
 * up = bilinear upsample to 512 x 512 with align_corners=True and torch's fp32 source-index arithmetic.
 * Writes pred512 = up(image) and gt512 = ref[:3] alpha + bg (1 - alpha), fp32 [1,3,512,512], and terms fp32 [4] (DEVICE):
 *   terms[0] = mean(ws^2); terms[1] = mean(-a log2 a - (1-a) log2(1-a)), a = clamp(ws, 1e-5, 1-1e-5);
 *   terms[2] = front ? mean|pred512 - gt512| over 3 * 512^2 : 0;
 *   terms[3] = front ? clamp(cov(x, y) / sqrt(var x var y), -1, 1) : 0 over the masked pixels, x = nan_to_num(up(depth)), y = the
 *              prior (two-pass fp64; fewer than 2 masked pixels give NaN).
 * Every sum is fp64 with per-CTA partials folded in a fixed order (run-to-run identical).  workspace:
 * mi3d_coarse_losses_workspace_bytes(h, w) bytes (0: invalid size); it also carries what the backward reads, so it must stay
 * untouched between a forward and its backward. */
size_t mi3d_coarse_losses_workspace_bytes(uint32_t h, uint32_t w);
int mi3d_coarse_losses(const float* image, const float* depth, const float* weights_sum, uint32_t h, uint32_t w, const float* ref_rgba,
                       const float* bg_color, const double* depth_prior, const uint8_t* depth_mask, int front, float* pred512, float* gt512,
                       float* terms, void* workspace, size_t workspace_bytes, mi3d_stream_t stream);
/* Gradients of g . terms + <grad_pred512, pred512> with grad_terms = g (DEVICE fp32 [4]) and grad_pred512 fp32 [1,3,512,512]
 * (nullable), given the forward's pred512, gt512, prior, mask and workspace: grad_image [h*w,3], grad_depth [h*w] and
 * grad_weights_sum [h*w] (overwritten).  The upsample's adjoint is a gather in a fixed order (no atomics: bitwise repeatable);
 * nan_to_num passes no gradient where up(depth) was not finite, the clamps pass it at their bounds inclusive (and nowhere for a NaN
 * coefficient). */
int mi3d_coarse_losses_backward(const float* weights_sum, uint32_t h, uint32_t w, const float* pred512, const float* gt512,
                                const double* depth_prior, const uint8_t* depth_mask, int front, const float* grad_terms,
                                const float* grad_pred512, const void* workspace, size_t workspace_bytes, float* grad_image,
                                float* grad_depth, float* grad_weights_sum, mi3d_stream_t stream);

/* unit-test entry for the hand-written wgmma tf32 tiles of the field forward (3-term split, K-major operands):
 * mode 0 (the only one): d[128,N] = a[128,K] . b[N,K]^T, N in {16, 32, 64}, K in {32, 64, 96, 128}.  fp32 in/out. */
int mi3d_tf32_tile_test(const float* a, const float* b, float* d, int N, int K, int mode, mi3d_stream_t stream);

const char* mi3d_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MI3D_H */
