// field.cu -- fused NeRF field evaluation for sm_90a (C ABI: include/mi3d.h)
//
// One kernel evaluates, per marched sample, everything nerf/network_tcnn.py:102-170 + nerf/renderer.py:513-524
// do with 13 separate encoder/MLP passes in the reference:
//     multires hash-grid gather (tiny-cuda-nn HashGrid, fp32 table)  ->  32-64-64-4 MLP (fp32, bias, ReLU)
//     -> trunc_exp / sigmoid -> 6-tap finite-difference normal -> shading -> orientation / smoothness terms
// without materialising activations in HBM.  The finite-difference normals difference two densities 0.02 apart, so the
// MLP needs fp32-class products (plain fp16 / bf16 / tf32 inputs would put ~1e-2 relative error on the normals; see
// DESIGN.md): the layer GEMMs run on wgmma over split-precision operands.
//   k_field_fwd_tc    forward: 3-term tf32 split, one 128-sample tile per CTA at a time (owner / encoder / MMA warps)
//   k_field_bwd_tc    backward chain: recomputes the activations tile by tile, back-propagates through the MLP (6-term bf16
//                     split), keeps the weight gradients in registers across the whole persistent CTA and scatters the
//                     table gradient with vector reductions (RED.ADD.v2 / v4.f32) under the MMA chain
//   k_bwd_enc_scatter full-occupancy hash-grid gather that feeds the chain kernel its encodings through HBM
//   k_field_fwd       density only, fp32 FFMA tiles in shared memory: the density-grid refresh (mi3d_density_grid_update)
// plus the stand-alone hash-grid encoder (k_hashgrid_fwd / k_hashgrid_bwd) and the density-grid kernels (k_grid_*).
//
// Grid: persistent, gridDim = SM count (132 on H100 SXM) x resident CTAs; the number of valid rows is read from device memory
// (counter[0] written by mi3d_march_rays_train), so there is no host synchronisation between march and field.
#include "mi3d_common.cuh"
#include "tf32_tile.cuh"
#include "../../include/mi3d.h"
#include <stdlib.h>

namespace {

constexpr int T = 128;        // rows (samples) per tile
constexpr int TP = 132;       // padded row stride of the k-major activation tiles (floats)
constexpr int NT = 256;       // threads per CTA
constexpr int D_IN = 32, D_H = 64, D_OUT = 4;
constexpr float kFdEps = 1e-2f;      // network_tcnn.py:115
constexpr float kSmoothStd = 1e-2f;  // renderer.py:522

struct LevelSm { uint32_t offset, size, res, hashed; float scale; };

// ---------------------------------------------------------------------------------------------------------
// hash-grid helpers (tiny-cuda-nn grid.h semantics, see oracle/field_ref.py for the restatement + citations)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hg_index(uint32_t cx, uint32_t cy, uint32_t cz, const LevelSm& L) {
    uint32_t idx;
    if (L.hashed) {
        idx = cx ^ (cy * 2654435761u) ^ (cz * 805459861u);
        idx = (L.size & (L.size - 1)) == 0 ? (idx & (L.size - 1)) : (idx % L.size);
    } else {
        idx = cx + cy * L.res + cz * L.res * L.res;
        if (idx >= L.size) idx %= L.size;      // only when a coordinate sits exactly on the upper face
    }
    return idx;
}

struct CellW { uint32_t c[3]; float w[3]; };

__device__ __forceinline__ CellW hg_cell(float u0, float u1, float u2, float scale) {
    CellW r;
    #pragma unroll
    for (int d = 0; d < 3; d++) {
        const float p = fmaf(scale, d == 0 ? u0 : (d == 1 ? u1 : u2), 0.5f);
        const float f = floorf(p);
        r.c[d] = (uint32_t)(int32_t)f;
        r.w[d] = p - f;
    }
    return r;
}

// Encode levels [l0, l0+nl) of point u (in [0,1]^3) into enc[(2l+f) * stride + row].
__device__ __forceinline__ void encode_levels(const float* __restrict__ table, const LevelSm* __restrict__ lv, int l0, int nl,
                                              float u0, float u1, float u2, float* __restrict__ enc, int stride, int row) {
    #pragma unroll 2
    for (int i = 0; i < nl; i++) {
        const int l = l0 + i;
        const LevelSm L = lv[l];
        const CellW cw = hg_cell(u0, u1, u2, L.scale);
        const float2* __restrict__ base = reinterpret_cast<const float2*>(table) + L.offset;
        float2 v[8];
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            const uint32_t cx = cw.c[0] + (corner & 1), cy = cw.c[1] + ((corner >> 1) & 1), cz = cw.c[2] + ((corner >> 2) & 1);
            v[corner] = __ldg(base + hg_index(cx, cy, cz, L));
        }
        float f0 = 0.f, f1 = 0.f;
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            const float wx = (corner & 1) ? cw.w[0] : 1 - cw.w[0];
            const float wy = (corner & 2) ? cw.w[1] : 1 - cw.w[1];
            const float wz = (corner & 4) ? cw.w[2] : 1 - cw.w[2];
            const float wt = wx * wy * wz;
            f0 = fmaf(wt, v[corner].x, f0); f1 = fmaf(wt, v[corner].y, f1);
        }
        enc[(2 * l) * stride + row] = f0;
        enc[(2 * l + 1) * stride + row] = f1;
    }
}

// Scatter d(enc) of levels [l0,l0+nl) into the table gradient (one RED.v2.f32 per corner).
__device__ __forceinline__ void scatter_levels(float* __restrict__ gtable, const LevelSm* __restrict__ lv, int l0, int nl,
                                               float u0, float u1, float u2, const float* __restrict__ genc, int stride, int row) {
    #pragma unroll 1
    for (int i = 0; i < nl; i++) {
        const int l = l0 + i;
        const LevelSm L = lv[l];
        const float g0 = genc[(2 * l) * stride + row], g1 = genc[(2 * l + 1) * stride + row];
        if (g0 == 0.f && g1 == 0.f) continue;
        const CellW cw = hg_cell(u0, u1, u2, L.scale);
        float2* __restrict__ base = reinterpret_cast<float2*>(gtable) + L.offset;
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            const uint32_t cx = cw.c[0] + (corner & 1), cy = cw.c[1] + ((corner >> 1) & 1), cz = cw.c[2] + ((corner >> 2) & 1);
            const float wx = (corner & 1) ? cw.w[0] : 1 - cw.w[0];
            const float wy = (corner & 2) ? cw.w[1] : 1 - cw.w[1];
            const float wz = (corner & 4) ? cw.w[2] : 1 - cw.w[2];
            const float wt = wx * wy * wz;
            atomicAdd(base + hg_index(cx, cy, cz, L), make_float2(wt * g0, wt * g1));
        }
    }
}

// Warp-aggregated variant for the tensor-core backward: lanes are consecutive samples of (mostly) one ray, so at the coarse
// levels whole runs of lanes fall into the same cell.  A segmented inclusive scan keyed by the table index (5 shuffle steps)
// folds each run; only the last lane of a run issues the RED, so the L2 sees fewer same-address atomics.
// Must be called by all 32 lanes (inactive lanes pass active = false).
__device__ __forceinline__ void scatter_level_agg(float* __restrict__ gtable, const LevelSm& L, float u0, float u1, float u2,
                                                  float g0, float g1, bool active, bool aggregate, int lane) {
    const CellW cw = hg_cell(u0, u1, u2, L.scale);
    float2* __restrict__ base = reinterpret_cast<float2*>(gtable) + L.offset;
    // runs = maximal stretches of ADJACENT active lanes in the same cell: all eight corner keys of such lanes coincide, so the run
    // structure (segment ids + the five scan predicates) is computed once per level and shared by the 16 scanned values
    uint32_t heads = 0xffffffffu, takem = 0u;
    if (aggregate) {
        const uint32_t c0 = active ? cw.c[0] : 0xFFFFFF00u + (uint32_t)lane, c1 = cw.c[1], c2 = cw.c[2];
        const uint32_t p0 = __shfl_up_sync(0xffffffffu, c0, 1), p1 = __shfl_up_sync(0xffffffffu, c1, 1), p2 = __shfl_up_sync(0xffffffffu, c2, 1);
        heads = __ballot_sync(0xffffffffu, lane == 0 || p0 != c0 || p1 != c1 || p2 != c2);
        const int seg = __popc(heads & (0xffffffffu >> (31 - lane)));
        #pragma unroll
        for (int i = 0; i < 5; i++) {
            const int su = __shfl_up_sync(0xffffffffu, seg, 1 << i);
            if (lane >= (1 << i) && su == seg) takem |= 1u << i;
        }
    }
    const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
    const bool issue = active && (!aggregate || tail);
    // the two x-neighbours of a (cy, cz) corner pair are adjacent table entries whenever idx(x+1) == idx(x) ^ 1 (dense levels with an
    // even index; hashed power-of-two levels with an even cell x, where the +1 only flips bit 0 of the xor-hash): one 16-byte RED
    // then carries both.  Fewer, wider REDs cut the RED count, which is what bounds the scatter.
    #pragma unroll
    for (int yz = 0; yz < 4; yz++) {
        const uint32_t cy = cw.c[1] + (yz & 1), cz = cw.c[2] + (yz >> 1);
        const float wyz = ((yz & 1) ? cw.w[1] : 1 - cw.w[1]) * ((yz & 2) ? cw.w[2] : 1 - cw.w[2]);
        const float wt0 = (1 - cw.w[0]) * wyz, wt1 = cw.w[0] * wyz;
        float v00 = active ? wt0 * g0 : 0.f, v01 = active ? wt0 * g1 : 0.f, v10 = active ? wt1 * g0 : 0.f, v11 = active ? wt1 * g1 : 0.f;
        if (aggregate) {
            #pragma unroll
            for (int i = 0; i < 5; i++) {
                const float a00 = __shfl_up_sync(0xffffffffu, v00, 1 << i), a01 = __shfl_up_sync(0xffffffffu, v01, 1 << i);
                const float a10 = __shfl_up_sync(0xffffffffu, v10, 1 << i), a11 = __shfl_up_sync(0xffffffffu, v11, 1 << i);
                if ((takem >> i) & 1u) { v00 += a00; v01 += a01; v10 += a10; v11 += a11; }
            }
        }
        if (!issue) continue;
        const uint32_t i0 = hg_index(cw.c[0], cy, cz, L), i1 = hg_index(cw.c[0] + 1, cy, cz, L);
        const bool nz0 = v00 != 0.f || v01 != 0.f, nz1 = v10 != 0.f || v11 != 0.f;
        if (i1 == (i0 ^ 1u) && (nz0 || nz1)) {
            const bool lo = (i0 & 1u) == 0u;      // i0 is the even (first) entry of the pair
            atomicAdd(reinterpret_cast<float4*>(base + (i0 & ~1u)), lo ? make_float4(v00, v01, v10, v11) : make_float4(v10, v11, v00, v01));
        } else {
            if (nz0) atomicAdd(base + i0, make_float2(v00, v01));
            if (nz1) atomicAdd(base + i1, make_float2(v10, v11));
        }
    }
}

// The chain kernel's gather / scatter threads own (row, half) with the 16 levels dealt out in PAIRS: half h holds levels
// {4j + 2h, 4j + 2h + 1 : j = 0..3}, i.e. encoding columns [8j + 4h, 8j + 4h + 4).  (A contiguous split gave every warp-aggregated
// coarse level to half 0 and made those four warps the slowest link of the fused scatter.)
__device__ __forceinline__ int half_level(int i, int half) { return ((i >> 1) << 2) + 2 * half + (i & 1); }

// single-level-at-a-time variant (8 loads in flight): lower register pressure, used by the backward's prefetch
__device__ __forceinline__ void gather16s(const float* __restrict__ table, const LevelSm* __restrict__ lv, int half,
                                          float u0, float u1, float u2, float (&f)[16]) {
    #pragma unroll
    for (int i = 0; i < 8; i++) {
        const LevelSm L = lv[half_level(i, half)];
        const CellW cw = hg_cell(u0, u1, u2, L.scale);
        const float2* __restrict__ base = reinterpret_cast<const float2*>(table) + L.offset;
        float2 v[8];
        #pragma unroll
        for (int corner = 0; corner < 8; corner++)
            v[corner] = __ldg(base + hg_index(cw.c[0] + (corner & 1), cw.c[1] + ((corner >> 1) & 1), cw.c[2] + ((corner >> 2) & 1), L));
        float f0 = 0.f, f1 = 0.f;
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            const float wt = ((corner & 1) ? cw.w[0] : 1 - cw.w[0]) * ((corner & 2) ? cw.w[1] : 1 - cw.w[1]) * ((corner & 4) ? cw.w[2] : 1 - cw.w[2]);
            f0 = fmaf(wt, v[corner].x, f0); f1 = fmaf(wt, v[corner].y, f1);
        }
        f[2 * i] = f0; f[2 * i + 1] = f1;
    }
}

// gather + trilinear blend of levels [l0, l0 + lcount) (lcount <= 8) of point u into f[2i], f[2i+1].
// Levels are processed in PAIRS: 16 independent 8-byte loads are in flight per thread before any is consumed (the kernels
// wait on gather latency, so loads in flight are what counts).
__device__ __forceinline__ void gather16(const float* __restrict__ table, const LevelSm* __restrict__ lv, int l0, int lcount,
                                         float u0, float u1, float u2, float (&f)[16]) {
    #pragma unroll
    for (int i = 0; i < 8; i += 2) {
        if (i >= lcount) { f[2 * i] = 0.f; f[2 * i + 1] = 0.f; f[2 * i + 2] = 0.f; f[2 * i + 3] = 0.f; continue; }
        const bool two = i + 1 < lcount;
        const LevelSm La = lv[l0 + i], Lb = lv[l0 + (two ? i + 1 : i)];
        const CellW ca = hg_cell(u0, u1, u2, La.scale), cb = hg_cell(u0, u1, u2, Lb.scale);
        const float2* __restrict__ ba = reinterpret_cast<const float2*>(table) + La.offset;
        const float2* __restrict__ bb = reinterpret_cast<const float2*>(table) + Lb.offset;
        float2 va[8], vb[8];
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            va[corner] = __ldg(ba + hg_index(ca.c[0] + (corner & 1), ca.c[1] + ((corner >> 1) & 1), ca.c[2] + ((corner >> 2) & 1), La));
            vb[corner] = __ldg(bb + hg_index(cb.c[0] + (corner & 1), cb.c[1] + ((corner >> 1) & 1), cb.c[2] + ((corner >> 2) & 1), Lb));
        }
        float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
        #pragma unroll
        for (int corner = 0; corner < 8; corner++) {
            const float wa = ((corner & 1) ? ca.w[0] : 1 - ca.w[0]) * ((corner & 2) ? ca.w[1] : 1 - ca.w[1]) * ((corner & 4) ? ca.w[2] : 1 - ca.w[2]);
            const float wb = ((corner & 1) ? cb.w[0] : 1 - cb.w[0]) * ((corner & 2) ? cb.w[1] : 1 - cb.w[1]) * ((corner & 4) ? cb.w[2] : 1 - cb.w[2]);
            a0 = fmaf(wa, va[corner].x, a0); a1 = fmaf(wa, va[corner].y, a1);
            b0 = fmaf(wb, vb[corner].x, b0); b1 = fmaf(wb, vb[corner].y, b1);
        }
        f[2 * i] = a0; f[2 * i + 1] = a1;
        f[2 * i + 2] = two ? b0 : 0.f; f[2 * i + 3] = two ? b1 : 0.f;
    }
}

// ---------------------------------------------------------------------------------------------------------
// fp32 FFMA layer of k_field_fwd over shared memory: Out = relu(A W + bias).  A: [K][TP] (k-major), W: [K][N] row-major, Out: [N][TP].
// thread -> rows lane*4..+3, columns warp*NC..+NC-1 with NC = N/8.  Activations are k-major ([feature][row], row stride TP = 132
// floats = 4 mod 32) so that the 32 lanes of a warp read / write 128 consecutive rows (conflict-free LDS.128 / STS.128) and the
// weights are warp-broadcast LDS.128.
// ---------------------------------------------------------------------------------------------------------
template <int K, int N>
__device__ __forceinline__ void tile_gemm(const float* __restrict__ A, const float* __restrict__ W, const float* __restrict__ bias, float* Out) {
    constexpr int NC = N / 8;
    static_assert(NC == 4 || NC == 8, "column tile");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r0 = lane * 4, c0 = warp * NC;
    float acc[NC][4];
    #pragma unroll
    for (int c = 0; c < NC; c++) {
        const float b = bias[c0 + c];
        acc[c][0] = b; acc[c][1] = b; acc[c][2] = b; acc[c][3] = b;
    }
    #pragma unroll 8
    for (int k = 0; k < K; k++) {
        const float4 a = *reinterpret_cast<const float4*>(A + k * TP + r0);
        float w[NC];
        #pragma unroll
        for (int c4 = 0; c4 < NC / 4; c4++) {
            const float4 wv = *reinterpret_cast<const float4*>(W + k * N + c0 + 4 * c4);
            w[4 * c4] = wv.x; w[4 * c4 + 1] = wv.y; w[4 * c4 + 2] = wv.z; w[4 * c4 + 3] = wv.w;
        }
        #pragma unroll
        for (int c = 0; c < NC; c++) {
            acc[c][0] = fmaf(a.x, w[c], acc[c][0]); acc[c][1] = fmaf(a.y, w[c], acc[c][1]);
            acc[c][2] = fmaf(a.z, w[c], acc[c][2]); acc[c][3] = fmaf(a.w, w[c], acc[c][3]);
        }
    }
    #pragma unroll
    for (int c = 0; c < NC; c++) {
        const float4 o = make_float4(fmaxf(acc[c][0], 0.f), fmaxf(acc[c][1], 0.f), fmaxf(acc[c][2], 0.f), fmaxf(acc[c][3], 0.f));
        *reinterpret_cast<float4*>(Out + (c0 + c) * TP + r0) = o;
    }
}

// Output layer 64 -> 4: thread (row = tid & 127, pair = tid >> 7) computes outputs 2*pair, 2*pair+1.
__device__ __forceinline__ void out_layer(const float* __restrict__ H2, const float* __restrict__ W3t /*[64][4]*/, const float* __restrict__ b3,
                                          float* __restrict__ O) {
    const int row = threadIdx.x & (T - 1), pair = threadIdx.x >> 7;
    float o0 = b3[2 * pair], o1 = b3[2 * pair + 1];
    #pragma unroll 16
    for (int k = 0; k < D_H; k++) {
        const float h = H2[k * TP + row];
        const float2 w = *reinterpret_cast<const float2*>(W3t + 4 * k + 2 * pair);
        o0 = fmaf(h, w.x, o0); o1 = fmaf(h, w.y, o1);
    }
    O[(2 * pair) * TP + row] = o0; O[(2 * pair + 1) * TP + row] = o1;
}

// ---------------------------------------------------------------------------------------------------------
// shared memory of k_field_fwd
// ---------------------------------------------------------------------------------------------------------
struct Smem {
    float* wt1; float* b1; float* wt2; float* b2; float* w3t; float* b3;   // weights as [in][out]
    LevelSm* lv;
    float* enc; float* h1; float* h2; float* o;
};

__device__ __forceinline__ Smem carve(float* base) {
    Smem s;
    float* p = base;
    s.enc = p; p += D_IN * TP;
    s.h1 = p; p += D_H * TP;
    s.h2 = p; p += D_H * TP;
    s.o = p; p += D_OUT * TP;
    s.wt1 = p; p += D_IN * D_H; s.b1 = p; p += D_H;
    s.wt2 = p; p += D_H * D_H; s.b2 = p; p += D_H;
    s.w3t = p; p += D_H * D_OUT; s.b3 = p; p += D_OUT;
    s.lv = reinterpret_cast<LevelSm*>(p);
    return s;
}

constexpr size_t kFwdSmem = sizeof(float) * ((D_IN + 2 * D_H + D_OUT) * TP + D_IN * D_H + D_H + D_H * D_H + D_H + D_H * D_OUT + D_OUT)
                            + 16 * sizeof(LevelSm);

__device__ __forceinline__ void load_weights(const Smem& s, const mi3d_mlp& m, const mi3d_hashgrid& hg) {
    for (int i = threadIdx.x; i < D_H * D_IN; i += NT) s.wt1[(i % D_IN) * D_H + i / D_IN] = m.w1[i];      // W1 [64][32]
    for (int i = threadIdx.x; i < D_H * D_H; i += NT) s.wt2[(i % D_H) * D_H + i / D_H] = m.w2[i];         // W2 [64][64]
    for (int i = threadIdx.x; i < D_OUT * D_H; i += NT) s.w3t[(i % D_H) * D_OUT + i / D_H] = m.w3[i];     // W3 [4][64]
    for (int i = threadIdx.x; i < D_H; i += NT) { s.b1[i] = m.b1[i]; s.b2[i] = m.b2[i]; }
    if (threadIdx.x < D_OUT) s.b3[threadIdx.x] = m.b3[threadIdx.x];
    if (threadIdx.x < 16) {
        LevelSm L; const int l = threadIdx.x;
        if (l < (int)hg.n_levels) {
            L.offset = hg.offsets[l]; L.size = hg.sizes[l]; L.res = hg.ress[l]; L.scale = hg.scales[l];
            const uint64_t dense = (uint64_t)L.res * L.res * L.res;
            L.hashed = dense > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        s.lv[l] = L;
    }
}

__device__ __forceinline__ uint32_t padded_rows(uint32_t M, uint32_t align, uint32_t cap) {
    uint32_t m = M;
    if (align > 0) m += align - m % align;        // raymarching.py:238-239 (always adds, even when already aligned)
    return m < cap ? m : cap;
}

// position of evaluation e for a sample at x (perturbation pz = x + 0.01*noise for e >= 7)
__device__ __forceinline__ void eval_pos(int e, const float x[3], const float xp[3], float bound, float p[3]) {
    const float* base = e >= 7 ? xp : x;
    p[0] = base[0]; p[1] = base[1]; p[2] = base[2];
    if (e > 0) {
        const int t = (e - 1) % 6, axis = t >> 1;
        const float sgn = (t & 1) ? -kFdEps : kFdEps;
        // the reference clamps all three coordinates of the tap position (network_tcnn.py:117-122)
        #pragma unroll
        for (int d = 0; d < 3; d++) p[d] = mi3d_clampf(d == axis ? p[d] + sgn : p[d], -bound, bound);
    }
}

__device__ __forceinline__ float blob(const float p[3], float density, float two_r2) {
    const float d = (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2];
    return density * expf(-d / two_r2);
}

__device__ __forceinline__ float nan_to_num(float v) {
    if (isnan(v)) return 0.f;
    if (isinf(v)) return v > 0 ? FLT_MAX : -FLT_MAX;
    return v;
}

struct Normal { float g[3]; float q; float inv; float n[3]; bool finite[3]; bool in_clamp; };

__device__ __forceinline__ Normal make_normal(const float sp[3], const float sn[3]) {
    Normal r;
    #pragma unroll
    for (int a = 0; a < 3; a++) r.g[a] = -(0.5f * (sp[a] - sn[a]) / kFdEps);
    const float S = (r.g[0] * r.g[0] + r.g[1] * r.g[1]) + r.g[2] * r.g[2];
    r.in_clamp = (S >= 1e-20f) && (S <= 1e32f);
    r.q = fminf(fmaxf(S, 1e-20f), 1e32f);
    if (isnan(S)) r.q = S;
    const float rt = sqrtf(r.q);
    #pragma unroll
    for (int a = 0; a < 3; a++) {
        const float v = r.g[a] / rt;
        r.finite[a] = isfinite(v);
        r.n[a] = nan_to_num(v);
    }
    r.inv = 1.f / rt;
    return r;
}

// d(loss)/dg given d(loss)/dn, through nan_to_num and safe_normalize
__device__ __forceinline__ void normal_bwd(const Normal& nm, const float dn_in[3], float dg[3]) {
    float dn[3];
    #pragma unroll
    for (int a = 0; a < 3; a++) dn[a] = nm.finite[a] ? dn_in[a] : 0.f;
    // n = g * q^-1/2 ; dq = -0.5 q^-3/2 sum(dn*g)
    const float dot = (dn[0] * nm.g[0] + dn[1] * nm.g[1]) + dn[2] * nm.g[2];
    const float dq = -0.5f * dot * nm.inv * nm.inv * nm.inv;
    const float dS = nm.in_clamp ? dq : 0.f;
    #pragma unroll
    for (int a = 0; a < 3; a++) dg[a] = dn[a] * nm.inv + 2.f * dS * nm.g[a];
}

__device__ __forceinline__ void gauss_pair(uint64_t seed, uint32_t row, uint32_t salt, float out[3]) {
    const uint4 r = mi3d_philox(make_uint4(row, salt, 0u, 0x736d6f6fu), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float u1 = fmaxf(mi3d_u01(r.x), 5.9604645e-8f), u2 = mi3d_u01(r.y), u3 = fmaxf(mi3d_u01(r.z), 5.9604645e-8f), u4 = mi3d_u01(r.w);
    const float m1 = sqrtf(-2.f * logf(u1)), m2 = sqrtf(-2.f * logf(u3));
    out[0] = m1 * cospif(2.f * u2); out[1] = m1 * sinpif(2.f * u2); out[2] = m2 * cospif(2.f * u4);
}

// position-keyed variant: the draw is a pure function of (seed, sample position), i.e. independent of which rank / row evaluates
// the sample (ray-parallel render: a G-rank step must equal the single-process accumulation of the same views)
__device__ __forceinline__ void gauss_pos(uint64_t seed, const float x[3], float out[3]) {
    const uint4 r = mi3d_philox(make_uint4(__float_as_uint(x[0]), __float_as_uint(x[1]), __float_as_uint(x[2]), 0x706f7321u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float u1 = fmaxf(mi3d_u01(r.x), 5.9604645e-8f), u2 = mi3d_u01(r.y), u3 = fmaxf(mi3d_u01(r.z), 5.9604645e-8f), u4 = mi3d_u01(r.w);
    const float m1 = sqrtf(-2.f * logf(u1)), m2 = sqrtf(-2.f * logf(u3));
    out[0] = m1 * cospif(2.f * u2); out[1] = m1 * sinpif(2.f * u2); out[2] = m2 * cospif(2.f * u4);
}

// ---------------------------------------------------------------------------------------------------------
// Row bookkeeping.  Single view: rows [0, M) are samples, [M, m_pad) the reference's zero rows (raymarching.py:237-241).
// Multi-view batch (mi3d_view_segs): rows are ordered by ray id, hence by view; segment s < n_views holds the samples of view s,
// segment n_views + v the zero rows of view v that THIS rank evaluates; every per-sample mean is over the whole view's padded
// count mpad[v] (summed over ranks), so that sharding a view's rays over ranks changes nothing but the summation order.
// ---------------------------------------------------------------------------------------------------------
struct Rows { uint32_t M, m_pad; const mi3d_view_segs* segs; };
struct RowInfo { bool in_range, real; uint32_t view, mpad, pad_idx; };

__device__ __forceinline__ Rows rows_make(const int* counter, uint32_t m_fixed, uint32_t align, uint32_t cap, const mi3d_view_segs* segs) {
    Rows R; R.segs = segs;
    if (segs) { R.M = min(segs->bounds[segs->n_views], cap); R.m_pad = min(segs->bounds[2 * segs->n_views], cap); }
    else { R.M = counter ? min((uint32_t)counter[0], cap) : m_fixed; R.m_pad = padded_rows(R.M, align, cap); }
    return R;
}

__device__ __forceinline__ RowInfo row_info(const Rows& R, uint32_t row) {
    RowInfo ri;
    ri.in_range = row < R.m_pad; ri.real = row < R.M;
    if (!R.segs) { ri.view = 0; ri.mpad = R.m_pad; ri.pad_idx = row - R.M; return ri; }
    const uint32_t nv = R.segs->n_views;
    uint32_t sgm = 0;
    for (uint32_t j = 1; j < 2 * nv; j++) sgm += row >= R.segs->bounds[j] ? 1u : 0u;
    ri.view = sgm < nv ? sgm : sgm - nv;
    ri.mpad = R.segs->mpad[ri.view];
    ri.pad_idx = row - R.segs->bounds[sgm];
    return ri;
}

// smoothness-loss perturbation z ~ N(0,1)^3 of a row (renderer.py:522): injected array, Philox by row (single view), or Philox by
// position (multi-view / noise_mode 1; a view's zero rows are keyed by their index among them) -- either way the draw of a sample
// does not depend on which rank, batch or row evaluates it
__device__ __forceinline__ void smooth_z(const float* __restrict__ smooth_noise, uint64_t seed, uint32_t noise_mode, uint32_t row,
                                         const RowInfo& ri, const float x[3], float z[3]) {
    if (smooth_noise) { z[0] = smooth_noise[3 * (size_t)row]; z[1] = smooth_noise[3 * (size_t)row + 1]; z[2] = smooth_noise[3 * (size_t)row + 2]; }
    else if (noise_mode == 0) gauss_pair(seed, row, 1u, z);
    else if (ri.real) gauss_pos(seed, x, z);
    else gauss_pair(seed, ri.pad_idx, 2u, z);            // zero rows: keyed by their index among the view's zero rows
}

struct FwdArgs {
    const float* xyzs; const float* dirs; const int* counter; uint32_t m_fixed, align, cap;
    const float* table; mi3d_hashgrid hg; mi3d_mlp mlp;
    float bound, blob_density, two_r2;
    int n_evals, shading; float ratio; const float* light_d;
    const float* smooth_noise; uint64_t seed;
    float* sigmas; float* rgbs; float* normals; float* tape; float* loss_partials;
    float* enc_cache; uint32_t enc_cache_tiles;     // optional: encodings of the first enc_cache_tiles tiles, laid out like the backward's enc_buf
    const mi3d_view_segs* segs; uint32_t noise_mode; // multi-view batch (device table) / Philox keying of the smoothness perturbation
};

// ---------------------------------------------------------------------------------------------------------
// density only, plain fp32 FFMA: sigmas[row] = trunc_exp(h0(xyzs[row]) + blob) for rows [0, n).  The density-grid refresh evaluates
// every grid cell with it (mi3d_density_grid_update).
// CTA = 256 threads = one tile of T = 128 samples; each thread owns a 4-row x (N/8)-column register tile of a layer GEMM.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT, 2) k_field_fwd(const float* __restrict__ xyzs, uint32_t n, const float* __restrict__ table,
                                                     const mi3d_hashgrid hg, const mi3d_mlp mlp, float bound, float blob_density,
                                                     float two_r2, float* __restrict__ sigmas) {
    extern __shared__ __align__(16) float smem_raw[];
    const Smem s = carve(smem_raw);
    load_weights(s, mlp, hg);
    const int lrow = threadIdx.x & (T - 1), half = threadIdx.x >> 7;
    const int nl = (int)hg.n_levels, l0 = half * (nl / 2), lcount = half ? nl - nl / 2 : nl / 2;
    __syncthreads();

    for (uint32_t tile = blockIdx.x; (uint64_t)tile * T < n; tile += gridDim.x) {
        const uint32_t row = tile * T + lrow;
        const bool in_range = row < n;
        float p[3] = {0.f, 0.f, 0.f};
        if (in_range) { p[0] = xyzs[3 * (size_t)row]; p[1] = xyzs[3 * (size_t)row + 1]; p[2] = xyzs[3 * (size_t)row + 2]; }
        const float inv2b = 2.f * bound;
        encode_levels(table, s.lv, l0, lcount, (p[0] + bound) / inv2b, (p[1] + bound) / inv2b, (p[2] + bound) / inv2b, s.enc, TP, lrow);
        __syncthreads();
        tile_gemm<D_IN, D_H>(s.enc, s.wt1, s.b1, s.h1);
        __syncthreads();
        tile_gemm<D_H, D_H>(s.h1, s.wt2, s.b2, s.h2);
        __syncthreads();
        out_layer(s.h2, s.w3t, s.b3, s.o);
        __syncthreads();
        if (half == 0 && in_range) {
            // trunc_exp(h0 + blob(p)) with the fused multiply-adds spelled out: the compiler may contract blob()'s sum of squares either
            // way, and the grid (hence the bitfield that every rank of a multi-GPU step must agree on) should not depend on its choice
            const float d2 = fmaf(p[2], p[2], fmaf(p[0], p[0], p[1] * p[1]));
            sigmas[row] = expf(fmaf(blob_density, expf(-d2 / two_r2), s.o[lrow]));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// forward: the three layer GEMMs run on wgmma (tf32) with a 3-term split
//   x = hi + lo (hi = tf32-rounded x):  A.B ~= A_hi.B_hi + A_lo.B_hi + A_hi.B_lo     (error ~2^-21, fp32-class)
// so the finite-difference normals keep their accuracy while the MLP leaves the FFMA pipe.
// CTA = 512 threads, one 128-sample tile at a time (persistent):
//   warps 0-3   owners  : thread r owns sample r; epilogues (bias, ReLU, hi/lo split -> next A operand in shared memory,
//                         K-major 128B-swizzle layout) and all per-sample math / outputs
//   warps 4-11  encoders: hash-grid gathers for the NEXT evaluation while the MMA / epilogue chain of the current one runs
//   warps 12-15 MMA     : one warpgroup issues the wgmma chain; it writes each accumulator (registers, fragment layout) into a
//                         row-major staging tile in shared memory, from which owner r reads row r
// Hand-offs are mbarriers (count = arriving threads).
// ---------------------------------------------------------------------------------------------------------
// Accumulator hand-off between the MMA warpgroup and the row owners.  d[h] is an m64 accumulator (rows 64 h ..) in the wgmma fragment
// layout; stage_frag writes its columns [c0, c0 + nc) to dst[row * ld + col - c0] (rows 0..127), stg_row32 reads one row's 32 columns.
template <int R>
__device__ __forceinline__ void stage_frag(const float (&d)[2][R], float* dst, int ld, int c0, int nc, int wl, int lane) {
    #pragma unroll
    for (int h = 0; h < 2; h++)
        #pragma unroll
        for (int j = 0; j < R / 4; j++)
            #pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                const int row = 64 * h + 16 * wl + (lane >> 2) + 8 * hh, col = 8 * j + 2 * (lane & 3) - c0;
                if (col >= 0 && col < nc) {
                    if (col + 1 < nc) *reinterpret_cast<float2*>(dst + row * ld + col) = make_float2(d[h][4 * j + 2 * hh], d[h][4 * j + 2 * hh + 1]);
                    else dst[row * ld + col] = d[h][4 * j + 2 * hh];
                }
            }
}
__device__ __forceinline__ void stg_row32(const float* src, uint32_t (&v)[32]) {
    #pragma unroll
    for (int q = 0; q < 8; q++) {
        const float4 t = reinterpret_cast<const float4*>(src)[q];
        v[4 * q] = __float_as_uint(t.x); v[4 * q + 1] = __float_as_uint(t.y); v[4 * q + 2] = __float_as_uint(t.z); v[4 * q + 3] = __float_as_uint(t.w);
    }
}

namespace fwdtc {
using namespace ::ftc;
constexpr int kThreads = 512;
constexpr int kA1 = 128 * 32 * 4;             // one [128 x 32] fp32 tile = 16 KB
// smem carve (bytes): A1_hi, A1_lo, A2_hi[2], A2_lo[2], W1_hi, W1_lo, W2_hi[2], W2_lo[2], W3_hi[2], W3_lo[2], then misc
constexpr int oA1H = 0, oA1L = oA1H + kA1, oA2H = oA1L + kA1, oA2L = oA2H + 2 * kA1;
constexpr int oW1H = oA2L + 2 * kA1, oW1L = oW1H + 8192, oW2H = oW1L + 8192, oW2L = oW2H + 16384;
constexpr int oW3H = oW2L + 16384, oW3L = oW3H + 4096, oStg = oW3L + 4096;
constexpr int kStgLd = 68;                    // staging row stride (floats): float4 row reads by consecutive rows hit distinct banks
constexpr int oStg3 = oStg + 128 * kStgLd * 4;    // layer-3 outputs [128][4]: kept apart so that layer 1 of the next evaluation may stage
constexpr int oMisc = oStg3 + 128 * 4 * 4;
constexpr size_t kSmem = 1024 + oMisc + 2048;

// D (+)= A[128 x 32*KB] . B[N x 32*KB]^T over hi/lo split tiles as two m64 halves; a_hi/a_lo/b_hi/b_lo are smem addresses of the first
// K-block.  Issues, commits and waits.
template <int N>
__device__ __forceinline__ void mma_layer(float (&d)[2][N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, int kblocks,
                                          uint32_t a_kb_stride, uint32_t b_kb_stride) {
    wg::fence();
    #pragma unroll
    for (int h = 0; h < 2; h++) issue_3tf32<N>(d[h], a_hi + 8192u * h, a_lo + 8192u * h, a_kb_stride, b_hi, b_lo, b_kb_stride, 32 * kblocks, 0u);
    wg::commit();
    wg::wait<0>();
    wg::reg_fence(d[0]); wg::reg_fence(d[1]);
}
}  // namespace fwdtc

__global__ void __launch_bounds__(fwdtc::kThreads, 1) k_field_fwd_tc(const FwdArgs a) {
    using namespace fwdtc;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* sm = smem_dyn + ((1024u - (tc::smem_u32(smem_dyn) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    float* b1s = reinterpret_cast<float*>(sm + oMisc);          // 64
    float* b2s = b1s + 64;                                      // 64
    float* b3s = b2s + 64;                                      // 4 (+pad)
    LevelSm* lv = reinterpret_cast<LevelSm*>(b3s + 8);          // 16 * 20 B
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + oMisc + 896);   // a1_full, a1_empty, d1_full, a2_full, d2_full, a3_full, d3_full
    float* red = reinterpret_cast<float*>(bars + 8);            // [2][4] loss partials
    float* s_loss = red + 8;                                    // [MI3D_MAX_VIEWS][2] per-view loss sums (multi-view batches)
    __shared__ mi3d_view_segs segs_sm;
    uint64_t *a1_full = bars, *a1_empty = bars + 1, *d1_full = bars + 2, *a2_full = bars + 3, *d2_full = bars + 4, *a3_full = bars + 5, *d3_full = bars + 6;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // ---- one-time setup: weights split hi/lo into UMMA B-operand tiles ([out][in] is already [N][K] K-major) ----
    for (int i = tid; i < D_H * D_IN; i += kThreads) {           // W1 [64][32]
        const int n = i / D_IN, k = i % D_IN; const float v = a.mlp.w1[i], h = tf32_hi(v);
        *reinterpret_cast<float*>(sm + oW1H + sw_off(n, k)) = h; *reinterpret_cast<float*>(sm + oW1L + sw_off(n, k)) = v - h;
    }
    for (int i = tid; i < D_H * D_H; i += kThreads) {            // W2 [64][64] -> two K-blocks of [64 x 32]
        const int n = i / D_H, k = i % D_H; const float v = a.mlp.w2[i], h = tf32_hi(v);
        const uint32_t o = (k >> 5) * 8192 + sw_off(n, k & 31);
        *reinterpret_cast<float*>(sm + oW2H + o) = h; *reinterpret_cast<float*>(sm + oW2L + o) = v - h;
    }
    for (int i = tid; i < 16 * D_H; i += kThreads) {             // W3 [4][64] zero-padded to N = 16 -> two K-blocks of [16 x 32]
        const int n = i / D_H, k = i % D_H; const float v = n < D_OUT ? a.mlp.w3[n * D_H + k] : 0.f, h = tf32_hi(v);
        const uint32_t o = (k >> 5) * 2048 + sw_off(n, k & 31);
        *reinterpret_cast<float*>(sm + oW3H + o) = h; *reinterpret_cast<float*>(sm + oW3L + o) = v - h;
    }
    for (int i = tid; i < D_H; i += kThreads) { b1s[i] = a.mlp.b1[i]; b2s[i] = a.mlp.b2[i]; }
    if (tid < D_OUT) b3s[tid] = a.mlp.b3[tid];
    if (tid < 16) {
        LevelSm L; const int l = tid;
        if (l < (int)a.hg.n_levels) {
            L.offset = a.hg.offsets[l]; L.size = a.hg.sizes[l]; L.res = a.hg.ress[l]; L.scale = a.hg.scales[l];
            L.hashed = (uint64_t)L.res * L.res * L.res > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        lv[l] = L;
    }
    if (a.segs && tid < (int)(sizeof(mi3d_view_segs) / 4)) reinterpret_cast<uint32_t*>(&segs_sm)[tid] = reinterpret_cast<const uint32_t*>(a.segs)[tid];
    if (tid < 2 * MI3D_MAX_VIEWS) s_loss[tid] = 0.f;
    if (tid == 0) {
        tc::mbar_init(a1_full, 256); tc::mbar_init(a1_empty, 128); tc::mbar_init(d1_full, 128); tc::mbar_init(a2_full, 128);
        tc::mbar_init(d2_full, 128); tc::mbar_init(a3_full, 128); tc::mbar_init(d3_full, 128);
        tc::fence_barrier_init();
    }
    tc::fence_proxy_async();                 // weight tiles were written through the generic proxy, wgmma reads through the async proxy
    __syncthreads();
    const uint32_t sbase = tc::smem_u32(sm);
    const float* stg = reinterpret_cast<const float*>(sm + oStg);
    const float* stg3 = reinterpret_cast<const float*>(sm + oStg3);

    const Rows R = rows_make(a.counter, a.m_fixed, a.align, a.cap, a.segs ? &segs_sm : nullptr);
    const uint32_t m_pad = R.m_pad;
    const int n_evals = a.n_evals;
    const float inv2b = 2.f * a.bound;
    float acc_orient = 0.f, acc_smooth = 0.f;
    uint32_t it = 0;                         // global evaluation counter -> mbarrier phase parity

    if (warp < 4) {
        // ================================ owners ================================
        const int r = tid;
        for (uint32_t tile = blockIdx.x; (uint64_t)tile * T < m_pad; tile += gridDim.x) {
            const uint32_t row = tile * T + r;
            const RowInfo ri = row_info(R, row);
            const bool in_range = ri.in_range, real = ri.real;
            const bool lit = a.shading != MI3D_SHADING_ALBEDO && ri.mpad < 1000000u;      // network_tcnn.py:159 fallback, per view
            float light[3] = {0.f, 0.f, 0.f};                                             // multi-view: one light direction per view
            if (a.light_d) { const float* lp = a.light_d + (R.segs ? 3 * ri.view : 0u); light[0] = lp[0]; light[1] = lp[1]; light[2] = lp[2]; }
            float x[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f}, xp[3] = {0.f, 0.f, 0.f};
            if (real) {
                x[0] = a.xyzs[3 * (size_t)row]; x[1] = a.xyzs[3 * (size_t)row + 1]; x[2] = a.xyzs[3 * (size_t)row + 2];
                if (a.dirs) { d[0] = a.dirs[3 * (size_t)row]; d[1] = a.dirs[3 * (size_t)row + 1]; d[2] = a.dirs[3 * (size_t)row + 2]; }
            }
            if (n_evals > 7 && in_range) {
                float z[3];
                smooth_z(a.smooth_noise, a.seed, a.noise_mode, row, ri, x, z);
                #pragma unroll
                for (int c = 0; c < 3; c++) xp[c] = x[c] + z[c] * kSmoothStd;
            }
            float sigma0 = 0.f, alb[3] = {0.f, 0.f, 0.f}, tapv[12];
            #pragma unroll
            for (int i = 0; i < 12; i++) tapv[i] = 0.f;
            for (int e = 0; e < n_evals; e++, it++) {
                const uint32_t par = it & 1;
                // ---- epilogue 1: H1 = relu(D1 + b1) -> A2 (hi/lo) ----
                tc::mbar_wait(d1_full, par);
                #pragma unroll 1
                for (int c0 = 0; c0 < D_H; c0 += 32) {
                    uint32_t v[32];
                    stg_row32(stg + r * kStgLd + c0, v);
                    #pragma unroll
                    for (int q = 0; q < 8; q++) {
                        float h[4], l[4];
                        #pragma unroll
                        for (int j = 0; j < 4; j++) { const float t = fmaxf(__uint_as_float(v[4 * q + j]) + b1s[c0 + 4 * q + j], 0.f); h[j] = tf32_hi(t); l[j] = t - h[j]; }
                        const uint32_t o = (c0 >> 5) * kA1 + sw_off(r, 4 * q);
                        *reinterpret_cast<float4*>(sm + oA2H + o) = make_float4(h[0], h[1], h[2], h[3]);
                        *reinterpret_cast<float4*>(sm + oA2L + o) = make_float4(l[0], l[1], l[2], l[3]);
                    }
                }
                tc::fence_proxy_async();
                mbar_arrive(a2_full);
                // ---- epilogue 2: H2 = relu(D2 + b2) -> A3 (reuses the A2 tiles: layer-2 MMAs have retired) ----
                tc::mbar_wait(d2_full, par);
                #pragma unroll 1
                for (int c0 = 0; c0 < D_H; c0 += 32) {
                    uint32_t v[32];
                    stg_row32(stg + r * kStgLd + c0, v);
                    #pragma unroll
                    for (int q = 0; q < 8; q++) {
                        float h[4], l[4];
                        #pragma unroll
                        for (int j = 0; j < 4; j++) { const float t = fmaxf(__uint_as_float(v[4 * q + j]) + b2s[c0 + 4 * q + j], 0.f); h[j] = tf32_hi(t); l[j] = t - h[j]; }
                        const uint32_t o = (c0 >> 5) * kA1 + sw_off(r, 4 * q);
                        *reinterpret_cast<float4*>(sm + oA2H + o) = make_float4(h[0], h[1], h[2], h[3]);
                        *reinterpret_cast<float4*>(sm + oA2L + o) = make_float4(l[0], l[1], l[2], l[3]);
                    }
                }
                tc::fence_proxy_async();
                mbar_arrive(a3_full);
                // ---- epilogue 3: outputs ----
                tc::mbar_wait(d3_full, par);
                uint32_t o4[4];
                {
                    const float4 t4 = *reinterpret_cast<const float4*>(stg3 + 4 * r);
                    o4[0] = __float_as_uint(t4.x); o4[1] = __float_as_uint(t4.y); o4[2] = __float_as_uint(t4.z); o4[3] = __float_as_uint(t4.w);
                }
                float p[3];
                eval_pos(e, x, xp, a.bound, p);
                const float sg = expf(__uint_as_float(o4[0]) + b3s[0] + blob(p, a.blob_density, a.two_r2));
                if (e == 0) {
                    sigma0 = sg;
                    #pragma unroll
                    for (int c = 0; c < 3; c++) alb[c] = 1.f / (1.f + expf(-(__uint_as_float(o4[1 + c]) + b3s[1 + c])));
                } else {
                    #pragma unroll
                    for (int i = 0; i < 12; i++) if (i == e - 1) tapv[i] = sg;
                }
            }
            if (in_range) {
                float col[3] = {alb[0], alb[1], alb[2]};
                if (n_evals >= 7) {
                    const float sp[3] = {tapv[0], tapv[2], tapv[4]}, sn[3] = {tapv[1], tapv[3], tapv[5]};
                    const Normal nm = make_normal(sp, sn);
                    if (lit) {
                        const float ndl = (nm.n[0] * light[0] + nm.n[1] * light[1]) + nm.n[2] * light[2];
                        const float lam = a.ratio + (1 - a.ratio) * fmaxf(ndl, 0.1f);
                        if (a.shading == MI3D_SHADING_TEXTURELESS) { col[0] = col[1] = col[2] = lam; }
                        else if (a.shading == MI3D_SHADING_NORMAL) { col[0] = (nm.n[0] + 1) / 2; col[1] = (nm.n[1] + 1) / 2; col[2] = (nm.n[2] + 1) / 2; }
                        else { col[0] = alb[0] * lam; col[1] = alb[1] * lam; col[2] = alb[2] * lam; }
                    }
                    const float wgt = 1.f - expf(-sigma0);
                    const float ndd = fmaxf((nm.n[0] * d[0] + nm.n[1] * d[1]) + nm.n[2] * d[2], 0.f);
                    const float t_orient = wgt * (ndd * ndd);
                    float t_smooth = 0.f;
                    if (n_evals > 7) {
                        const float sp2[3] = {tapv[6], tapv[8], tapv[10]}, sn2[3] = {tapv[7], tapv[9], tapv[11]};
                        const Normal np = make_normal(sp2, sn2);
                        t_smooth = (fabsf(nm.n[0] - np.n[0]) + fabsf(nm.n[1] - np.n[1])) + fabsf(nm.n[2] - np.n[2]);
                    }
                    if (!R.segs) { acc_orient += t_orient; acc_smooth += t_smooth; }       // fixed-order sums, divided once at the end
                    else {                                                                  // per-view means over the whole view's rows
                        const float inv = 1.f / (float)ri.mpad;
                        atomicAdd(s_loss + 2 * ri.view, t_orient * inv); atomicAdd(s_loss + 2 * ri.view + 1, t_smooth * (inv / 3.f));
                    }
                    if (a.normals) { a.normals[3 * (size_t)row] = nm.n[0]; a.normals[3 * (size_t)row + 1] = nm.n[1]; a.normals[3 * (size_t)row + 2] = nm.n[2]; }
                }
                a.sigmas[row] = sigma0;
                if (a.rgbs) { a.rgbs[3 * (size_t)row] = col[0]; a.rgbs[3 * (size_t)row + 1] = col[1]; a.rgbs[3 * (size_t)row + 2] = col[2]; }
                if (a.tape) {
                    float4* tp = reinterpret_cast<float4*>(a.tape + 16 * (size_t)row);
                    tp[0] = make_float4(sigma0, alb[0], alb[1], alb[2]);
                    tp[1] = make_float4(tapv[0], tapv[1], tapv[2], tapv[3]);
                    tp[2] = make_float4(tapv[4], tapv[5], tapv[6], tapv[7]);
                    tp[3] = make_float4(tapv[8], tapv[9], tapv[10], tapv[11]);
                }
            }
        }
    } else if (warp < 12) {
        // ================================ encoders ================================
        const int et = tid - 128, r = et & (T - 1), half = et >> 7;
        const int nl = (int)a.hg.n_levels, l0 = half * (nl / 2), lcount = half ? nl - nl / 2 : nl / 2;
        for (uint32_t tile = blockIdx.x; (uint64_t)tile * T < m_pad; tile += gridDim.x) {
            const uint32_t row = tile * T + r;
            const RowInfo ri = row_info(R, row);
            const bool in_range = ri.in_range, real = ri.real;
            float x[3] = {0.f, 0.f, 0.f}, xp[3] = {0.f, 0.f, 0.f};
            if (real) { x[0] = a.xyzs[3 * (size_t)row]; x[1] = a.xyzs[3 * (size_t)row + 1]; x[2] = a.xyzs[3 * (size_t)row + 2]; }
            if (n_evals > 7 && in_range) {
                float z[3];
                smooth_z(a.smooth_noise, a.seed, a.noise_mode, row, ri, x, z);
                #pragma unroll
                for (int c = 0; c < 3; c++) xp[c] = x[c] + z[c] * kSmoothStd;
            }
            for (int e = 0; e < n_evals; e++, it++) {
                float p[3];
                eval_pos(e, x, xp, a.bound, p);
                const float u0 = (p[0] + a.bound) / inv2b, u1 = (p[1] + a.bound) / inv2b, u2 = (p[2] + a.bound) / inv2b;
                // gather first (registers), then wait for the A1 buffer to be released by the previous evaluation's layer-1 MMAs
                float f[16];
                gather16(a.table, lv, l0, lcount, u0, u1, u2, f);
                if (a.enc_cache && tile < a.enc_cache_tiles) {        // keep the encodings for the backward pass (it would re-gather them)
                    float4* dst = reinterpret_cast<float4*>(a.enc_cache + ((size_t)tile * 13 + e) * (T * 32) + (size_t)r * 32 + 16 * half);
                    #pragma unroll
                    for (int q = 0; q < 4; q++) dst[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
                }
                if (it > 0) tc::mbar_wait(a1_empty, (it - 1) & 1);
                #pragma unroll
                for (int i = 0; i < 8; i++) {
                    if (i >= lcount) continue;
                    const int k = 2 * (l0 + i);
                    const float h0 = tf32_hi(f[2 * i]), h1 = tf32_hi(f[2 * i + 1]);
                    const uint32_t o = sw_off(r, k);
                    *reinterpret_cast<float2*>(sm + oA1H + o) = make_float2(h0, h1);
                    *reinterpret_cast<float2*>(sm + oA1L + o) = make_float2(f[2 * i] - h0, f[2 * i + 1] - h1);
                }
                tc::fence_proxy_async();
                mbar_arrive(a1_full);
            }
        }
    } else {
        // ================================ MMA warpgroup ================================
        float* stg_w = reinterpret_cast<float*>(sm + oStg);
        float* stg3_w = reinterpret_cast<float*>(sm + oStg3);
        const int wl = warp & 3;
        for (uint32_t tile = blockIdx.x; (uint64_t)tile * T < m_pad; tile += gridDim.x) {
            for (int e = 0; e < n_evals; e++, it++) {
                const uint32_t par = it & 1;
                float d[2][32];
                tc::mbar_wait(a1_full, par);
                mma_layer<64>(d, sbase + oA1H, sbase + oA1L, sbase + oW1H, sbase + oW1L, 1, kA1, 8192);
                mbar_arrive(a1_empty);
                stage_frag<32>(d, stg_w, kStgLd, 0, 64, wl, lane);
                mbar_arrive(d1_full);
                tc::mbar_wait(a2_full, par);
                mma_layer<64>(d, sbase + oA2H, sbase + oA2L, sbase + oW2H, sbase + oW2L, 2, kA1, 8192);
                stage_frag<32>(d, stg_w, kStgLd, 0, 64, wl, lane);
                mbar_arrive(d2_full);
                tc::mbar_wait(a3_full, par);
                float d3[2][8];
                mma_layer<16>(d3, sbase + oA2H, sbase + oA2L, sbase + oW3H, sbase + oW3L, 2, kA1, 2048);
                stage_frag<8>(d3, stg3_w, 4, 0, 4, wl, lane);
                mbar_arrive(d3_full);
            }
        }
    }
    // ---- loss partials (owners only hold non-zero accumulators) + teardown ----
    {
        float v0 = acc_orient, v1 = acc_smooth;
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) { v0 += __shfl_xor_sync(0xffffffffu, v0, o); v1 += __shfl_xor_sync(0xffffffffu, v1, o); }
        if (warp < 4 && lane == 0) { red[warp] = v0; red[4 + warp] = v1; }
    }
    __syncthreads();
    if (tid == 0 && a.loss_partials && !a.segs) {
        a.loss_partials[2 * blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
        a.loss_partials[2 * blockIdx.x + 1] = (red[4] + red[5]) + (red[6] + red[7]);
    }
    if (a.loss_partials && a.segs && tid < 2 * (int)segs_sm.n_views) a.loss_partials[(size_t)blockIdx.x * 2 * segs_sm.n_views + tid] = s_loss[tid];
}

// loss_orient = sum / m_pad ; loss_smooth = sum / (3 m_pad)   (renderer.py:517-518, 523-524: .mean() over the padded rows).
// Multi-view (n_views > 0): partials are [cta][view][2] and already carry the 1 / mpad[view] factors; outputs are [n_views] arrays.
__global__ void k_loss_finalize(const float* __restrict__ partials, int n_part, const int* __restrict__ counter, uint32_t m_fixed,
                                uint32_t align, uint32_t cap, float* __restrict__ loss_orient, float* __restrict__ loss_smooth, int n_views) {
    if (blockIdx.x != 0) return;
    if (n_views > 0) {
        if ((int)threadIdx.x >= 2 * n_views) return;
        float t = 0.f;
        for (int i = 0; i < n_part; i++) t += partials[(size_t)i * 2 * n_views + threadIdx.x];
        float* dst = (threadIdx.x & 1) ? loss_smooth : loss_orient;
        if (dst) dst[threadIdx.x >> 1] = t;
        return;
    }
    if (threadIdx.x != 0) return;
    float t0 = 0.f, t1 = 0.f;
    for (int i = 0; i < n_part; i++) { t0 += partials[2 * i]; t1 += partials[2 * i + 1]; }
    const uint32_t M = counter ? min((uint32_t)counter[0], cap) : m_fixed;
    const float m_pad = (float)padded_rows(M, align, cap);
    if (loss_orient) *loss_orient = t0 / m_pad;
    if (loss_smooth) *loss_smooth = t1 / (3.f * m_pad);
}

// ---------------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------------
struct BwdArgs {
    const float* xyzs; const float* dirs; const int* counter; uint32_t m_fixed, align, cap;
    const float* table; mi3d_hashgrid hg; mi3d_mlp mlp;
    float bound, blob_density, two_r2;
    int n_evals, shading; float ratio; const float* light_d;
    const float* smooth_noise; uint64_t seed;
    const float* tape;
    const float* g_sigmas; const float* g_rgbs; const float* g_normals; const float* g_loss_orient; const float* g_loss_smooth;
    float* g_table; mi3d_mlp_grad g_mlp;
    // tiles [tile0, tile1) of this launch; enc_buf: their encodings [tile - tile0][13][128][32] (see k_bwd_enc_scatter), NULL = the
    // chain kernel gathers them itself
    float* enc_buf; uint32_t tile0, tile1;
    const mi3d_view_segs* segs; uint32_t noise_mode;   // multi-view: g_loss_orient / g_loss_smooth are [n_views] arrays
};

// d(loss)/d(h) of the 13 evaluations of one sample from the upstream gradients and the forward tape (sigma0, albedo, tap sigmas):
// shading / orientation / smoothness -> normals -> finite differences -> tap densities -> trunc_exp / sigmoid pre-activations.
__device__ __forceinline__ void sample_out_grads(const BwdArgs& a, uint32_t row, bool real, const float (&d)[3], bool lit, const float (&light)[3],
                                                 float Go, float Gs, bool need_ptaps, float (&dh)[4], float (&dtap)[12]) {
            const float4* tp = reinterpret_cast<const float4*>(a.tape + 16 * (size_t)row);
            const float4 t0 = tp[0], t1 = tp[1], t2 = tp[2], t3 = tp[3];
            const float sigma0 = t0.x, alb[3] = {t0.y, t0.z, t0.w};
            const float tapv[12] = {t1.x, t1.y, t1.z, t1.w, t2.x, t2.y, t2.z, t2.w, t3.x, t3.y, t3.z, t3.w};
            float gs = 0.f, gc[3] = {0.f, 0.f, 0.f};
            if (real) {
                if (a.g_sigmas) gs = a.g_sigmas[row];
                if (a.g_rgbs) { gc[0] = a.g_rgbs[3 * (size_t)row]; gc[1] = a.g_rgbs[3 * (size_t)row + 1]; gc[2] = a.g_rgbs[3 * (size_t)row + 2]; }
            }
            float dalb[3] = {gc[0], gc[1], gc[2]};
            float dn[3] = {0.f, 0.f, 0.f}, dnp[3] = {0.f, 0.f, 0.f};
            if (a.n_evals >= 7) {
                const float sp[3] = {tapv[0], tapv[2], tapv[4]}, sn[3] = {tapv[1], tapv[3], tapv[5]};
                const Normal nm = make_normal(sp, sn);
                if (a.g_normals && real) { dn[0] += a.g_normals[3 * (size_t)row]; dn[1] += a.g_normals[3 * (size_t)row + 1]; dn[2] += a.g_normals[3 * (size_t)row + 2]; }
                if (lit) {
                    const float ndl = (nm.n[0] * light[0] + nm.n[1] * light[1]) + nm.n[2] * light[2];
                    const float lam = a.ratio + (1 - a.ratio) * fmaxf(ndl, 0.1f);
                    float dlam = 0.f;
                    if (a.shading == MI3D_SHADING_TEXTURELESS) { dlam = (gc[0] + gc[1]) + gc[2]; dalb[0] = dalb[1] = dalb[2] = 0.f; }
                    else if (a.shading == MI3D_SHADING_NORMAL) { dn[0] += 0.5f * gc[0]; dn[1] += 0.5f * gc[1]; dn[2] += 0.5f * gc[2]; dalb[0] = dalb[1] = dalb[2] = 0.f; }
                    else { dlam = (gc[0] * alb[0] + gc[1] * alb[1]) + gc[2] * alb[2]; dalb[0] = gc[0] * lam; dalb[1] = gc[1] * lam; dalb[2] = gc[2] * lam; }
                    if (ndl >= 0.1f) {
                        const float k = dlam * (1 - a.ratio);
                        dn[0] += k * light[0]; dn[1] += k * light[1]; dn[2] += k * light[2];
                    }
                }
                if (Go != 0.f) {
                    const float wgt = 1.f - expf(-sigma0);
                    const float ndd = (nm.n[0] * d[0] + nm.n[1] * d[1]) + nm.n[2] * d[2];
                    if (ndd > 0.f) { const float k = Go * wgt * 2.f * ndd; dn[0] += k * d[0]; dn[1] += k * d[1]; dn[2] += k * d[2]; }
                }
                Normal np;
                if (need_ptaps) {
                    const float sp2[3] = {tapv[6], tapv[8], tapv[10]}, sn2[3] = {tapv[7], tapv[9], tapv[11]};
                    np = make_normal(sp2, sn2);
                    #pragma unroll
                    for (int c = 0; c < 3; c++) {
                        const float df = nm.n[c] - np.n[c];
                        const float sg = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f);
                        dn[c] += Gs * sg; dnp[c] -= Gs * sg;
                    }
                }
                float dg[3];
                normal_bwd(nm, dn, dg);
                #pragma unroll
                for (int ax = 0; ax < 3; ax++) {
                    // g = -(0.5 (s+ - s-) / eps)  ->  ds+ = -0.5/eps dg ; ds- = +0.5/eps dg ; dh0 = ds * exp(min(h,15)) = ds * min(s, e^15)
                    const float k = 0.5f / kFdEps * dg[ax];
                    dtap[2 * ax] = -k * fminf(tapv[2 * ax], 3269017.372472110639f);
                    dtap[2 * ax + 1] = k * fminf(tapv[2 * ax + 1], 3269017.372472110639f);
                }
                if (need_ptaps) {
                    normal_bwd(np, dnp, dg);
                    #pragma unroll
                    for (int ax = 0; ax < 3; ax++) {
                        const float k = 0.5f / kFdEps * dg[ax];
                        dtap[6 + 2 * ax] = -k * fminf(tapv[6 + 2 * ax], 3269017.372472110639f);
                        dtap[6 + 2 * ax + 1] = k * fminf(tapv[6 + 2 * ax + 1], 3269017.372472110639f);
                    }
                }
            }
            dh[0] = gs * fminf(sigma0, 3269017.372472110639f);       // activation.py:12-16
            #pragma unroll
            for (int c = 0; c < 3; c++) dh[1 + c] = dalb[c] * alb[c] * (1.f - alb[c]);
}

// the 16 encoding columns of one (row, half): four 16-byte chunks, 8 floats apart (see half_level)
__device__ __forceinline__ void load16(const float* __restrict__ src, float (&f)[16]) {
    #pragma unroll
    for (int q = 0; q < 4; q++) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src) + 2 * q);
        f[4 * q] = v.x; f[4 * q + 1] = v.y; f[4 * q + 2] = v.z; f[4 * q + 3] = v.w;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Gather kernel of the backward.  The chain kernel (k_field_bwd_tc) can afford only 8 gather / scatter warps next to ~200 KB of
// operand tiles, and the scatter keeps them busy.  The hash-grid gather is embarrassingly parallel over (sample, level), so it runs
// as a full-occupancy kernel ahead of the chain kernel and hands it the encodings through a per-chunk HBM buffer (128 B per
// evaluation):
//   k_bwd_enc_scatter: work item = (tile, evaluation), thread = (row, group of 4 levels)  -> enc_buf[tile - tile0][e][row][32]
//   k_field_bwd_tc   : loads them, runs the MMA chain and scatters d(enc) itself
// ---------------------------------------------------------------------------------------------------------
// which evaluations can receive a non-zero gradient (uniform over the launch; identical in the gather and chain kernels)
struct BwdPlan { int e_end; bool need_ptaps; };
__device__ __forceinline__ BwdPlan bwd_plan(const BwdArgs& a, const Rows& R) {
    const int nv = R.segs ? (int)R.segs->n_views : 1;
    bool lit = false, go = false, gs = false;
    for (int v = 0; v < nv; v++) {
        const uint32_t mpad = R.segs ? R.segs->mpad[v] : R.m_pad;
        lit |= a.shading != MI3D_SHADING_ALBEDO && mpad < 1000000u;
        go |= a.g_loss_orient && a.n_evals >= 7 && a.g_loss_orient[v] != 0.f;
        gs |= a.g_loss_smooth && a.n_evals > 7 && a.g_loss_smooth[v] != 0.f;
    }
    BwdPlan p;
    p.need_ptaps = gs;
    const bool need_taps = a.n_evals >= 7 && (gs || go || lit || a.g_normals != nullptr);
    p.e_end = !need_taps ? 1 : (gs ? 13 : 7);
    return p;
}

__global__ void __launch_bounds__(512, 2) k_bwd_enc_scatter(const BwdArgs a) {
    __shared__ LevelSm lv[16];
    __shared__ mi3d_view_segs segs_sm;
    if (a.segs && threadIdx.x >= 32 && threadIdx.x < 32 + sizeof(mi3d_view_segs) / 4)
        reinterpret_cast<uint32_t*>(&segs_sm)[threadIdx.x - 32] = reinterpret_cast<const uint32_t*>(a.segs)[threadIdx.x - 32];
    if (threadIdx.x < 16) {
        LevelSm L; const int l = threadIdx.x;
        if (l < (int)a.hg.n_levels) {
            L.offset = a.hg.offsets[l]; L.size = a.hg.sizes[l]; L.res = a.hg.ress[l]; L.scale = a.hg.scales[l];
            L.hashed = (uint64_t)L.res * L.res * L.res > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        lv[l] = L;
    }
    __syncthreads();
    const Rows R = rows_make(a.counter, a.m_fixed, a.align, a.cap, a.segs ? &segs_sm : nullptr);
    const uint32_t m_pad = R.m_pad;
    const int e_end = bwd_plan(a, R).e_end;
    const int r = threadIdx.x & (T - 1), lg = threadIdx.x >> 7;   // levels 4 lg .. 4 lg + 3
    const float inv2b = 2.f * a.bound;
    // persistent grid-stride loop over (tile, evaluation) work items of this chunk
    for (uint32_t w = blockIdx.x;; w += gridDim.x) {
        const uint32_t tile = a.tile0 + w / (uint32_t)e_end;
        const int e = (int)(w % (uint32_t)e_end);
        if (tile >= a.tile1 || (uint64_t)tile * T >= m_pad) break;
        const uint32_t row = tile * T + r;
        const RowInfo ri = row_info(R, row);
        const bool in_range = ri.in_range, real = ri.real;
        float x[3] = {0.f, 0.f, 0.f}, xp[3] = {0.f, 0.f, 0.f};
        if (real) { x[0] = a.xyzs[3 * (size_t)row]; x[1] = a.xyzs[3 * (size_t)row + 1]; x[2] = a.xyzs[3 * (size_t)row + 2]; }
        if (e >= 7 && in_range) {
            float z[3];
            smooth_z(a.smooth_noise, a.seed, a.noise_mode, row, ri, x, z);
            #pragma unroll
            for (int c = 0; c < 3; c++) xp[c] = x[c] + z[c] * kSmoothStd;
        }
        float p[3];
        eval_pos(e, x, xp, a.bound, p);
        const float u0 = (p[0] + a.bound) / inv2b, u1 = (p[1] + a.bound) / inv2b, u2 = (p[2] + a.bound) / inv2b;
        const size_t base = ((size_t)(tile - a.tile0) * 13 + e) * (T * 32) + (size_t)r * 32 + 8 * lg;
        float f[16];
        gather16(a.table, lv, 4 * lg, 4, u0, u1, u2, f);
        float4* dst = reinterpret_cast<float4*>(a.enc_buf + base);
        dst[0] = make_float4(f[0], f[1], f[2], f[3]); dst[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
}

// ---------------------------------------------------------------------------------------------------------
// backward chain kernel.  Same roles as k_field_fwd_tc; per evaluation the MMA warpgroup runs
//   F1: D1 = Enc W1^T          F2: D2 = H1 W2^T                               (recompute, K-major operands)
//   G2: dH1 = dZ2 W2           WG2: dW2 += dZ2^T H1   (A3/A2/W2 tiles re-read MN-major: no transposed copies)
//   G1: dEnc = dZ1 W1          WG1: dW1 += dZ1^T Enc
// all as bf16 3-way splits x = h + m + l with six product terms (wgmma bf16, fp32-class; 16-bit operands can be consumed
// MN-major, tf32 ones cannot).  dW2 / dW1 accumulate in the MMA warpgroup's registers across the whole persistent CTA and are
// flushed once at the end.  D1 / D2 / dH1 reach the owners through a [128 x 32] staging tile, half an accumulator at a time
// (stg_full / stg_empty); dEnc is written as fp32 [128][32] over the dZ tiles once G1 / WG1 have retired, the encoder warps read it
// there (d4_full -> denc_free) and scatter it (RED.v2.f32).  dZ3 -> dH2 (K = 4) and dW3 / db3 stay on the owner threads; db2 / db1
// are column sums the owners take from registers.
// ---------------------------------------------------------------------------------------------------------
namespace bwdtc {
using namespace ::fbf;
constexpr int kThreads = 512;
constexpr int kTile = 128 * 128;               // one [128 x 64 bf16] tile = 16 KB
// every operand = three part tiles (h, m, l) back to back; tiles are [rows x 64 bf16]
constexpr int oE = 0;                                              // Enc  3 x [128 x 64] (cols 32..63 stay zero)
constexpr int oH = oE + 3 * kTile;                                 // H1   3 x [128 x 64]
constexpr int oZ = oH + 3 * kTile;                                 // dZ2 then dZ1, 3 x [128 x 64]
constexpr int oW1 = oZ + 3 * kTile;                                // W1   3 x [64 x 64] (cols 32..63 zero)
constexpr int oW2 = oW1 + 3 * 8192;                                // W2   3 x [64 x 64]
constexpr int oStg = oW2 + 3 * 8192;                               // staging [128][kStgLd] fp32: 32 accumulator columns at a time
constexpr int kStgLd = 36;
constexpr int oMisc = oStg + 128 * kStgLd * 4;
constexpr size_t kSmem = 1024 + oMisc + 3072;
// Which levels' table-gradient REDs are warp-aggregated (scatter_level_agg): those with scale below this, i.e. where a cell spans
// several march steps (2 / scale  >  ~1.5 dt_min): levels 0..7 of the reference grid.  The scans cost issue slots next to the owner
// warps; the REDs they remove are the ones that serialise in L2 (the benchmark scene concentrates every sample in a sphere of radius
// 0.2: ~2 k occupied cells at level 5).
constexpr float kAggScaleMax = 100.f;

// one halving step of warp_colsum32: columns i and i + N of lanes L and L ^ N fold into column i
template <int N>
__device__ __forceinline__ void colsum_step(float (&v)[32], int lane) {
    const bool up = (lane & N) != 0;
    #pragma unroll
    for (int i = 0; i < N; i++) {
        const float keep = up ? v[i + N] : v[i], send = up ? v[i] : v[i + N];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, N);
    }
}

// column-wise sum over the 32 lanes of a warp of v[0..31]; lane j returns the total of column j (recursive halving, 31 shuffles).
// The steps are spelled out: a `for (n = 16; n >= 1; n >>= 1)` loop is not unrolled, and its variable inner trip count puts v
// in local memory.
__device__ __forceinline__ float warp_colsum32(float (&v)[32], int lane) {
    colsum_step<16>(v, lane); colsum_step<8>(v, lane); colsum_step<4>(v, lane); colsum_step<2>(v, lane); colsum_step<1>(v, lane);
    return v[0];
}

// The owners' column loops below run twice (`#pragma unroll 1`, c0 = 0, 32).  State kept per 32-column half is a register pair that
// each pass updates at [0] and then rotates, so after both passes [0] / [1] hold the halves c0 = 0 / 32: indexing it by c0 instead
// would place it in local memory.
template <typename V>
__device__ __forceinline__ void rot2(V (&v)[2]) { const V t = v[0]; v[0] = v[1]; v[1] = t; }
}  // namespace bwdtc

// Per-role cycle breakdown of k_field_bwd_tc (tools/prof_field_bwd.py builds a separate library with -DMI3D_FIELD_BWD_CLOCKS).
// Each thread sums clock64() intervals in registers; lane 0 of every warp adds its totals to g_field_bwd_clocks[slot] at the end:
//   0 owners: total   1 owners: waiting on stg_full
//   2 MMA: total      3 MMA: waiting on a1..a4_full
//   4 encoders: total 5 encoders: waiting on d4_full   6 encoders: scattering
//   7 evaluations run (one add per CTA)
// Without the switch the macros expand to nothing.
#ifdef MI3D_FIELD_BWD_CLOCKS
__device__ unsigned long long g_field_bwd_clocks[8];
#define BWD_CLK_VAR(v) long long v = 0
#define BWD_CLK_T(t) const long long t = clock64()
#define BWD_CLK_ACC(v, t) v += clock64() - t
#define BWD_CLK_FLUSH(slot, v) do { if (lane == 0) atomicAdd(&g_field_bwd_clocks[slot], (unsigned long long)(v)); } while (0)
#else
#define BWD_CLK_VAR(v)
#define BWD_CLK_T(t)
#define BWD_CLK_ACC(v, t)
#define BWD_CLK_FLUSH(slot, v)
#endif

__global__ void __launch_bounds__(bwdtc::kThreads, 1) k_field_bwd_tc(const BwdArgs a) {
    using namespace bwdtc;
    {   // chunk entirely past the (device-side) sample count: nothing to do
        const Rows R0 = rows_make(a.counter, a.m_fixed, a.align, a.cap, a.segs);
        if ((uint64_t)a.tile0 * T >= R0.m_pad) return;
    }
    __shared__ mi3d_view_segs segs_sm;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* sm = smem_dyn + ((1024u - (tc::smem_u32(smem_dyn) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    float* b1s = reinterpret_cast<float*>(sm + oMisc);          // 64
    float* b2s = b1s + 64;                                      // 64
    float* w3s = b2s + 64;                                      // [4][64]
    LevelSm* lv = reinterpret_cast<LevelSm*>(w3s + 256);        // 16 * 20 B = 320 B  (ends at 1856)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + oMisc + 2048);
    uint64_t *a1_full = bars, *d1_full = bars + 1, *a2_full = bars + 2, *a3_full = bars + 3, *a4_full = bars + 4, *d4_full = bars + 5,
             *stg_full = bars + 6, *stg_empty = bars + 7, *denc_free = bars + 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < (oMisc - oE) / 16; i += kThreads) reinterpret_cast<uint4*>(sm + oE)[i] = make_uint4(0, 0, 0, 0);   // zero pads, finite tiles
    __syncthreads();
    for (int i = tid; i < D_H * D_IN; i += kThreads) {           // W1 [64][32] -> rows j, cols i (K-major for F1, MN-major for G1)
        const int n = i / D_IN, k = i % D_IN; __nv_bfloat16 h, m, l; split3(a.mlp.w1[i], h, m, l);
        const uint32_t o = oW1 + sw_off16(n, k);
        *reinterpret_cast<__nv_bfloat16*>(sm + o) = h; *reinterpret_cast<__nv_bfloat16*>(sm + o + 8192) = m; *reinterpret_cast<__nv_bfloat16*>(sm + o + 16384) = l;
    }
    for (int i = tid; i < D_H * D_H; i += kThreads) {            // W2 [64][64]
        const int n = i / D_H, k = i % D_H; __nv_bfloat16 h, m, l; split3(a.mlp.w2[i], h, m, l);
        const uint32_t o = oW2 + sw_off16(n, k);
        *reinterpret_cast<__nv_bfloat16*>(sm + o) = h; *reinterpret_cast<__nv_bfloat16*>(sm + o + 8192) = m; *reinterpret_cast<__nv_bfloat16*>(sm + o + 16384) = l;
    }
    for (int i = tid; i < D_OUT * D_H; i += kThreads) w3s[i] = a.mlp.w3[i];
    for (int i = tid; i < D_H; i += kThreads) { b1s[i] = a.mlp.b1[i]; b2s[i] = a.mlp.b2[i]; }
    if (tid < 16) {
        LevelSm L; const int l = tid;
        if (l < (int)a.hg.n_levels) {
            L.offset = a.hg.offsets[l]; L.size = a.hg.sizes[l]; L.res = a.hg.ress[l]; L.scale = a.hg.scales[l];
            L.hashed = (uint64_t)L.res * L.res * L.res > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        lv[l] = L;
    }
    if (a.segs && tid < (int)(sizeof(mi3d_view_segs) / 4)) reinterpret_cast<uint32_t*>(&segs_sm)[tid] = reinterpret_cast<const uint32_t*>(a.segs)[tid];
    if (tid == 0) {
        tc::mbar_init(a1_full, 256); tc::mbar_init(d1_full, 128); tc::mbar_init(a2_full, 128); tc::mbar_init(a3_full, 128);
        tc::mbar_init(a4_full, 128); tc::mbar_init(d4_full, 128); tc::mbar_init(stg_full, 128); tc::mbar_init(stg_empty, 128);
        tc::mbar_init(denc_free, 256);
        tc::fence_barrier_init();
    }
    tc::fence_proxy_async();
    __syncthreads();
    const uint32_t sbase = tc::smem_u32(sm);

    const Rows R = rows_make(a.counter, a.m_fixed, a.align, a.cap, a.segs ? &segs_sm : nullptr);
    const uint32_t m_pad = R.m_pad;
    const BwdPlan plan = bwd_plan(a, R);
    const bool need_ptaps = plan.need_ptaps;
    const int e_end = plan.e_end;
    const float inv2b = 2.f * a.bound;
    uint32_t it = 0;

    if (warp < 4) {
        // ================================ owners ================================
        const int r = tid;
        const float* stg = reinterpret_cast<const float*>(sm + oStg);
        uint32_t su = 0;                     // staging hand-offs taken so far (mbarrier phase)
        BWD_CLK_T(clk_role); BWD_CLK_VAR(clk_wait);
        auto stg_take = [&](uint32_t (&v)[32]) {
            BWD_CLK_T(t0);
            tc::mbar_wait(stg_full, su & 1u);
            BWD_CLK_ACC(clk_wait, t0);
            stg_row32(stg + r * kStgLd, v);
            mbar_arrive(stg_empty);
            su++;
        };
        // persistent partial sums over this warp's rows: lane j owns columns j and j+32 of dW3[o][.] ; db3 on lane o
        float aw3[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}}, ab3 = 0.f;
        // db2 / db1 = column sums of dZ2 / dZ1 over this warp's rows, same lane <-> column mapping.  (Round 1 had the encoder warps
        // re-read the dZ tiles from shared memory behind two extra "readers done" barriers; that tied the encoders to the middle of
        // every evaluation and kept the fused RED scatter from running under the MMA chain.  The owners hold the values in registers.)
        float ab2[2] = {0.f, 0.f}, ab1[2] = {0.f, 0.f};
        for (uint32_t tile = a.tile0 + blockIdx.x; tile < a.tile1 && (uint64_t)tile * T < m_pad; tile += gridDim.x) {
            const uint32_t row = tile * T + r;
            const RowInfo ri = row_info(R, row);
            const bool in_range = ri.in_range, real = ri.real;
            float d[3] = {0.f, 0.f, 0.f};
            if (real && a.dirs) { d[0] = a.dirs[3 * (size_t)row]; d[1] = a.dirs[3 * (size_t)row + 1]; d[2] = a.dirs[3 * (size_t)row + 2]; }
            float dh[4] = {0.f, 0.f, 0.f, 0.f}, dtap[12];
            #pragma unroll
            for (int i = 0; i < 12; i++) dtap[i] = 0.f;
            if (in_range) {
                float light[3] = {0.f, 0.f, 0.f};
                if (a.light_d) { const float* lp = a.light_d + (R.segs ? 3 * ri.view : 0u); light[0] = lp[0]; light[1] = lp[1]; light[2] = lp[2]; }
                // upstream gradients of this row's view: d(mean over the view's mpad rows) (renderer.py:517-518, 523-524)
                const bool lit = a.shading != MI3D_SHADING_ALBEDO && ri.mpad < 1000000u;
                const float Go = (a.g_loss_orient && a.n_evals >= 7) ? a.g_loss_orient[ri.view] / (float)ri.mpad : 0.f;
                const float Gs = (a.g_loss_smooth && a.n_evals > 7) ? a.g_loss_smooth[ri.view] / (3.f * (float)ri.mpad) : 0.f;
                sample_out_grads(a, row, real, d, lit, light, Go, Gs, need_ptaps, dh, dtap);
            }
            for (int e = 0; e < e_end; e++, it++) {
                float dO[4] = {0.f, 0.f, 0.f, 0.f};
                if (e == 0) { dO[0] = dh[0]; dO[1] = dh[1]; dO[2] = dh[2]; dO[3] = dh[3]; }
                else {
                    // dtap[e - 1], taken from the front: a select on e would be compiled to an indexed load from local memory
                    dO[0] = dtap[0];
                    #pragma unroll
                    for (int i = 0; i < 11; i++) dtap[i] = dtap[i + 1];
                }
                uint32_t m1[2] = {0u, 0u};
                // ---- epilogue 1: H1 = relu(D1 + b1) -> A2 ; remember the ReLU mask ----
                #pragma unroll 1
                for (int c0 = 0; c0 < D_H; c0 += 32) {
                    uint32_t v[32];
                    stg_take(v);
                    uint32_t mk = 0u;
                    float tv[32];
                    #pragma unroll
                    for (int j = 0; j < 32; j++) { const float t = fmaxf(__uint_as_float(v[j]) + b1s[c0 + j], 0.f); if (t > 0.f) mk |= 1u << j; tv[j] = t; }
                    #pragma unroll
                    for (int q = 0; q < 4; q++) {
                        uint4 ph, pm, pl;
                        split8(reinterpret_cast<const float(&)[8]>(tv[8 * q]), ph, pm, pl);
                        const uint32_t o = oH + sw_off16(r, c0 + 8 * q);
                        *reinterpret_cast<uint4*>(sm + o) = ph; *reinterpret_cast<uint4*>(sm + o + kTile) = pm; *reinterpret_cast<uint4*>(sm + o + 2 * kTile) = pl;
                    }
                    m1[0] = mk; rot2(m1);
                }
                tc::fence_proxy_async();
                mbar_arrive(a2_full);
                // ---- epilogue 2: H2 = relu(D2 + b2) ; dZ2 = relu'(H2) * (dO W3) -> A3 ; dW3 / db3 partial sums ----
                // A3 (the dZ tiles) free: the previous evaluation's G1 / WG1 have retired and its dEnc (written over them) was read
                if (it > 0) tc::mbar_wait(denc_free, (it - 1) & 1);
                #pragma unroll 1
                for (int c0 = 0; c0 < D_H; c0 += 32) {
                    uint32_t v[32];
                    stg_take(v);
                    float h2[32];
                    #pragma unroll
                    for (int j = 0; j < 32; j++) h2[j] = fmaxf(__uint_as_float(v[j]) + b2s[c0 + j], 0.f);
                    float tv[32];
                    #pragma unroll
                    for (int j = 0; j < 32; j++) {
                        const int c = c0 + j;
                        float g = dO[0] * w3s[c];
                        if (e == 0) g = fmaf(dO[3], w3s[192 + c], fmaf(dO[2], w3s[128 + c], fmaf(dO[1], w3s[64 + c], g)));
                        tv[j] = h2[j] > 0.f ? g : 0.f;
                    }
                    #pragma unroll
                    for (int q = 0; q < 4; q++) {
                        uint4 ph, pm, pl;
                        split8(reinterpret_cast<const float(&)[8]>(tv[8 * q]), ph, pm, pl);
                        const uint32_t o = oZ + sw_off16(r, c0 + 8 * q);
                        *reinterpret_cast<uint4*>(sm + o) = ph; *reinterpret_cast<uint4*>(sm + o + kTile) = pm; *reinterpret_cast<uint4*>(sm + o + 2 * kTile) = pl;
                    }
                    ab2[0] += warp_colsum32(tv, lane); rot2(ab2);      // db2 (tv is dead after the stores above)
                    // dW3[o][c0 + lane] += sum over this warp's rows of dO[o] * H2[.][c0 + lane]
                    {
                        float t[32];
                        #pragma unroll
                        for (int j = 0; j < 32; j++) t[j] = dO[0] * h2[j];
                        aw3[0][0] += warp_colsum32(t, lane);
                        if (e == 0) {
                            #pragma unroll
                            for (int o = 1; o < 4; o++) {
                                #pragma unroll
                                for (int j = 0; j < 32; j++) t[j] = dO[o] * h2[j];
                                aw3[o][0] += warp_colsum32(t, lane);
                            }
                        }
                        #pragma unroll
                        for (int o = 0; o < 4; o++) rot2(aw3[o]);
                    }
                }
                tc::fence_proxy_async();
                mbar_arrive(a3_full);
                {   // db3[o] = sum of dO[o] over rows: lane o keeps the total
                    float s0 = dO[0], s1 = dO[1], s2 = dO[2], s3 = dO[3];
                    #pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                        s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o);
                    }
                    ab3 += lane == 0 ? s0 : (lane == 1 ? s1 : (lane == 2 ? s2 : (lane == 3 ? s3 : 0.f)));
                }
                // ---- epilogue 3: dZ1 = relu'(H1) * dH1 -> A3 (after G2 / WG2 retired and the db2 readers are done) ----
                #pragma unroll 1
                for (int c0 = 0; c0 < D_H; c0 += 32) {
                    uint32_t v[32];
                    stg_take(v);
                    const uint32_t mk = m1[0]; rot2(m1);
                    float tv[32];
                    #pragma unroll
                    for (int j = 0; j < 32; j++) tv[j] = (mk >> j) & 1u ? __uint_as_float(v[j]) : 0.f;
                    #pragma unroll
                    for (int q = 0; q < 4; q++) {
                        uint4 ph, pm, pl;
                        split8(reinterpret_cast<const float(&)[8]>(tv[8 * q]), ph, pm, pl);
                        const uint32_t o = oZ + sw_off16(r, c0 + 8 * q);
                        *reinterpret_cast<uint4*>(sm + o) = ph; *reinterpret_cast<uint4*>(sm + o + kTile) = pm; *reinterpret_cast<uint4*>(sm + o + 2 * kTile) = pl;
                    }
                    ab1[0] += warp_colsum32(tv, lane); rot2(ab1);      // db1
                }
                tc::fence_proxy_async();
                mbar_arrive(a4_full);
            }
        }
        // flush dW3 / db3 partials (one RED per lane per warp)
        #pragma unroll
        for (int o = 0; o < 4; o++) { atomicAdd(a.g_mlp.w3 + o * D_H + lane, aw3[o][0]); atomicAdd(a.g_mlp.w3 + o * D_H + 32 + lane, aw3[o][1]); }
        if (lane < 4) atomicAdd(a.g_mlp.b3 + lane, ab3);
        atomicAdd(a.g_mlp.b2 + lane, ab2[0]); atomicAdd(a.g_mlp.b2 + 32 + lane, ab2[1]);
        atomicAdd(a.g_mlp.b1 + lane, ab1[0]); atomicAdd(a.g_mlp.b1 + 32 + lane, ab1[1]);
        BWD_CLK_FLUSH(0, clock64() - clk_role); BWD_CLK_FLUSH(1, clk_wait);
    } else if (warp < 12) {
        // ================================ encoders / scatterers ================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 96;");
        const int et = tid - 128, r = et & (T - 1), half = et >> 7;
        const float* denc = reinterpret_cast<const float*>(sm + oZ);
        const bool ext = a.enc_buf != nullptr;
        // One stream of evaluations over this CTA's tiles, (tile, e) in order, counted by `it` like the owners and the MMA warpgroup.
        // Software pipeline with ping-pong E: the encoding uses 32 of the tile's 64 columns, so evaluation `it` lives in columns
        // 32 (it & 1) .. + 31 (operand start address + 64 B).  E(it+2) is written at the END of iteration `it` (its half was last read
        // by chain(it), retired at d4(it)), after the scatter of dEnc(it) under which its gather loads were in flight; chain(it+1) then
        // starts the moment chain(it) retires -- the MMA warp has already seen a1(it+1).  The fetch cursor runs two evaluations ahead
        // of the scatter across tile boundaries, so a tile's first chains run under the previous tile's last scatters (with e_end = 1,
        // every evaluation is a tile of its own).
        uint32_t ftile = a.tile0 + blockIdx.x;   // fetch cursor: (ftile, fe), with the row state of ftile
        int fe = 0;
        float x[3], xp[3];
        bool f_in_range = false;
        // scatter positions and row masks of evaluations it, it+1, it+2 (slot 2 is filled by the fetch of iteration it)
        float u[3][3];
        bool inr[3];
        auto write_E = [&](const float (&ff)[16], const uint32_t itw) {
            const int ecol = 32 * (int)(itw & 1u);
            #pragma unroll
            for (int i = 0; i < 8; i++) {
                const int k = 2 * half_level(i, half) + ecol;
                uint32_t h2, m2, l2;
                split3x2(ff[2 * i], ff[2 * i + 1], h2, m2, l2);
                const uint32_t o = oE + sw_off16(r, k);
                *reinterpret_cast<uint32_t*>(sm + o) = h2;
                *reinterpret_cast<uint32_t*>(sm + o + kTile) = m2;
                *reinterpret_cast<uint32_t*>(sm + o + 2 * kTile) = l2;
            }
            tc::fence_proxy_async();
            mbar_arrive(a1_full);
        };
        // encodings of the next evaluation of the stream into ff, its scatter position into uu and row mask into ir; false past the end
        auto fetch = [&](float (&ff)[16], float (&uu)[3], bool& ir) -> bool {
            if (ftile >= a.tile1 || (uint64_t)ftile * T >= m_pad) return false;
            if (fe == 0) {
                const uint32_t row = ftile * T + r;
                const RowInfo ri = row_info(R, row);
                f_in_range = ri.in_range;
                #pragma unroll
                for (int c = 0; c < 3; c++) { x[c] = 0.f; xp[c] = 0.f; }
                if (ri.real) { x[0] = a.xyzs[3 * (size_t)row]; x[1] = a.xyzs[3 * (size_t)row + 1]; x[2] = a.xyzs[3 * (size_t)row + 2]; }
                if (a.n_evals > 7 && ri.in_range) {
                    float z[3];
                    smooth_z(a.smooth_noise, a.seed, a.noise_mode, row, ri, x, z);
                    #pragma unroll
                    for (int c = 0; c < 3; c++) xp[c] = x[c] + z[c] * kSmoothStd;
                }
            }
            float p[3];
            eval_pos(fe, x, xp, a.bound, p);
            uu[0] = (p[0] + a.bound) / inv2b; uu[1] = (p[1] + a.bound) / inv2b; uu[2] = (p[2] + a.bound) / inv2b;
            ir = f_in_range;
            if (ext) load16(a.enc_buf + ((size_t)(ftile - a.tile0) * 13 + fe) * (T * 32) + (size_t)r * 32 + 4 * half, ff);
            else gather16s(a.table, lv, half, uu[0], uu[1], uu[2], ff);
            if (++fe == e_end) { fe = 0; ftile += gridDim.x; }
            return true;
        };
        float f[16];
        uint32_t n_fetched = 0;
        BWD_CLK_T(clk_role); BWD_CLK_VAR(clk_wait); BWD_CLK_VAR(clk_scatter);
        if (fetch(f, u[0], inr[0])) {
            n_fetched++;
            write_E(f, 0);
            if (fetch(f, u[1], inr[1])) {
                n_fetched++;
                // a1 may run at most one phase ahead of its waiter: F1(0) issued (d1) => the MMA warp has consumed a1 phase 0
                tc::mbar_wait(d1_full, 0);
                write_E(f, 1);
            }
        }
        for (; it < n_fetched; it++) {
            // dEnc (this thread's 16 columns of its row: 8j + 4 half .. + 3, j = 0..3) into registers
            BWD_CLK_T(t0);
            tc::mbar_wait(d4_full, it & 1);
            BWD_CLK_ACC(clk_wait, t0);
            uint32_t g[16];
            #pragma unroll
            for (int j = 0; j < 4; j++) {
                const float4 t = *reinterpret_cast<const float4*>(denc + r * 32 + 8 * j + 4 * half);
                g[4 * j] = __float_as_uint(t.x); g[4 * j + 1] = __float_as_uint(t.y); g[4 * j + 2] = __float_as_uint(t.z); g[4 * j + 3] = __float_as_uint(t.w);
            }
            mbar_arrive(denc_free);
            const bool next = fetch(f, u[2], inr[2]);      // evaluation it+2: loads in flight under the scatter
            n_fetched += next;
            BWD_CLK_T(t1);
            #pragma unroll 1
            for (int i = 0; i < 8; i++) {
                float g0 = 0.f, g1 = 0.f;
                #pragma unroll
                for (int q = 0; q < 8; q++) if (q == i) { g0 = __uint_as_float(g[2 * q]); g1 = __uint_as_float(g[2 * q + 1]); }
                const LevelSm L = lv[half_level(i, half)];
                scatter_level_agg(a.g_table, L, u[0][0], u[0][1], u[0][2], g0, g1, inr[0], L.scale < kAggScaleMax, lane);
            }
            BWD_CLK_ACC(clk_scatter, t1);
            if (next) write_E(f, it + 2);
            #pragma unroll
            for (int c = 0; c < 3; c++) { u[0][c] = u[1][c]; u[1][c] = u[2][c]; }
            inr[0] = inr[1]; inr[1] = inr[2];
        }
        BWD_CLK_FLUSH(4, clock64() - clk_role); BWD_CLK_FLUSH(5, clk_wait); BWD_CLK_FLUSH(6, clk_scatter);
    } else {
        // ================================ MMA warpgroup ================================
        // two accumulators plus the resident dW2 / dW1 do not fit the 128-register share of a 512-thread CTA: take the encoders' spare ones
        asm volatile("setmaxnreg.inc.sync.aligned.u32 192;");
        float* stg_w = reinterpret_cast<float*>(sm + oStg);
        float* denc_w = reinterpret_cast<float*>(sm + oZ);
        const int wl = warp & 3;
        // dW2 [64 x 64], dW1 [64 x 32] over every sample of this CTA: each evaluation's product starts a fresh accumulator and is added
        // here in fp32 (round to nearest) -- a chain of thousands of accumulating MMAs drifts further from the fp32 sum
        float dw2[32], dw1[16];
        #pragma unroll
        for (int i = 0; i < 32; i++) dw2[i] = 0.f;
        #pragma unroll
        for (int i = 0; i < 16; i++) dw1[i] = 0.f;
        uint32_t su = 0;
        auto stage = [&](const float (&d)[2][32]) {         // 64 accumulator columns, 32 at a time, to the owners
            #pragma unroll
            for (int c0 = 0; c0 < 64; c0 += 32) {
                if (su > 0) tc::mbar_wait(stg_empty, (su - 1) & 1u);
                stage_frag<32>(d, stg_w, kStgLd, c0, 32, wl, lane);
                mbar_arrive(stg_full);
                su++;
            }
        };
        auto rows64 = [](const Operand& o, int h) { return Operand{o.base + 8192u * (uint32_t)h, o.part_stride, o.lbo}; };   // K-major A: rows 64 h ..
        BWD_CLK_T(clk_role); BWD_CLK_VAR(clk_wait);
        auto wait_full = [&](uint64_t* bar, uint32_t parity) {
            BWD_CLK_T(t0);
            tc::mbar_wait(bar, parity);
            BWD_CLK_ACC(clk_wait, t0);
        };
        for (uint32_t tile = a.tile0 + blockIdx.x; tile < a.tile1 && (uint64_t)tile * T < m_pad; tile += gridDim.x) {
            for (int e = 0; e < e_end; e++, it++) {
                const uint32_t par = it & 1;
                const uint32_t eoff = 64u * (it & 1u);                      // ping-pong E: columns 32 (it & 1) .. + 31 of the tile
                const Operand E{sbase + oE + eoff, (uint32_t)kTile, (uint32_t)kTile}, H{sbase + oH, (uint32_t)kTile, (uint32_t)kTile};
                const Operand Z{sbase + oZ, (uint32_t)kTile, (uint32_t)kTile};
                const Operand W1{sbase + oW1, 8192u, 8192u}, W2{sbase + oW2, 8192u, 8192u};
                float d[2][32];
                if (it == 0) {                                      // it > 0: consumed before d4 of the previous evaluation
                    wait_full(a1_full, 0);
                    mbar_arrive(d1_full);                           // the encoders' one wait on d1 (before they write E(1))
                }
                wg::fence();
                #pragma unroll
                for (int h = 0; h < 2; h++) issue_bf16x3<64, 0, 0>(d[h], rows64(E, h), W1, 32, 0u);   // F1 (K = 32: the zero columns 32..63 are skipped)
                wg::commit(); wg::wait<0>(); wg::reg_fence(d[0]); wg::reg_fence(d[1]);
                stage(d);
                wait_full(a2_full, par);
                wg::fence();
                #pragma unroll
                for (int h = 0; h < 2; h++) issue_bf16x3<64, 0, 0>(d[h], rows64(H, h), W2, 64, 0u);   // F2
                wg::commit(); wg::wait<0>(); wg::reg_fence(d[0]); wg::reg_fence(d[1]);
                stage(d);
                wait_full(a3_full, par);
                wg::fence();
                #pragma unroll
                for (int h = 0; h < 2; h++) issue_bf16x3<64, 0, 1>(d[h], rows64(Z, h), W2, 64, 0u);   // G2 : dH1 = dZ2 W2
                float t2[32];
                issue_bf16x3<64, 1, 1>(t2, Z, H, 128, 0u);                                              // WG2: dW2 += dZ2^T H1
                wg::commit(); wg::wait<0>(); wg::reg_fence(d[0]); wg::reg_fence(d[1]); wg::reg_fence(t2);
                #pragma unroll
                for (int i = 0; i < 32; i++) dw2[i] += t2[i];
                stage(d);
                wait_full(a4_full, par);
                float g1[2][16];
                wg::fence();
                #pragma unroll
                for (int h = 0; h < 2; h++) issue_bf16x3<32, 0, 1>(g1[h], rows64(Z, h), W1, 64, 0u);  // G1 : dEnc = dZ1 W1
                float t1[16];
                issue_bf16x3<32, 1, 1>(t1, Z, E, 128, 0u);                                              // WG1: dW1 += dZ1^T Enc
                wg::commit(); wg::wait<0>(); wg::reg_fence(g1[0]); wg::reg_fence(g1[1]); wg::reg_fence(t1);
                #pragma unroll
                for (int i = 0; i < 16; i++) dw1[i] += t1[i];
                stage_frag<16>(g1, denc_w, 32, 0, 32, wl, lane);                                       // over the dZ tiles, now free
                // E(it+1), of this tile or the next, is already there (other half) or on its way.  Consuming its a1 phase BEFORE
                // releasing d4(it) keeps the encoders, who arrive for it+2 only after d4(it), from lapping this waiter.
                const uint32_t ntile = tile + gridDim.x;
                if (e + 1 < e_end || (ntile < a.tile1 && (uint64_t)ntile * T < m_pad)) wait_full(a1_full, par ^ 1u);
                mbar_arrive(d4_full);
            }
        }
        BWD_CLK_FLUSH(2, clock64() - clk_role); BWD_CLK_FLUSH(3, clk_wait);
#ifdef MI3D_FIELD_BWD_CLOCKS
        if (warp == 12 && lane == 0) atomicAdd(&g_field_bwd_clocks[7], (unsigned long long)it);
#endif
        // ---- flush the register-resident weight gradients: dW2 [64 x 64] and dW1 [64 x 32] (row = output feature) ----
        if (it > 0) {
            #pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                const int j = 16 * wl + (lane >> 2) + 8 * hh;
                #pragma unroll
                for (int n8 = 0; n8 < 8; n8++) {
                    const int c = 8 * n8 + 2 * (lane & 3);
                    atomicAdd(a.g_mlp.w2 + j * D_H + c, dw2[4 * n8 + 2 * hh]); atomicAdd(a.g_mlp.w2 + j * D_H + c + 1, dw2[4 * n8 + 2 * hh + 1]);
                }
                #pragma unroll
                for (int n8 = 0; n8 < 4; n8++) {
                    const int c = 8 * n8 + 2 * (lane & 3);
                    atomicAdd(a.g_mlp.w1 + j * D_IN + c, dw1[4 * n8 + 2 * hh]); atomicAdd(a.g_mlp.w1 + j * D_IN + c + 1, dw1[4 * n8 + 2 * hh + 1]);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// stand-alone hash-grid encoder (tcnn.Encoding drop-in used by the unfused B2 path and by parity tests)
// ---------------------------------------------------------------------------------------------------------
__global__ void k_hashgrid_fwd(const float* __restrict__ x, uint32_t E, const float* __restrict__ table, const mi3d_hashgrid hg,
                               float* __restrict__ out) {
    __shared__ LevelSm lv[16];
    if (threadIdx.x < 16) {
        LevelSm L; const int l = threadIdx.x;
        if (l < (int)hg.n_levels) {
            L.offset = hg.offsets[l]; L.size = hg.sizes[l]; L.res = hg.ress[l]; L.scale = hg.scales[l];
            L.hashed = (uint64_t)L.res * L.res * L.res > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        lv[l] = L;
    }
    __syncthreads();
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int nl = (int)hg.n_levels;
    encode_levels(table, lv, 0, nl, x[3 * (size_t)e], x[3 * (size_t)e + 1], x[3 * (size_t)e + 2], out + (size_t)e * 2 * nl, 1, 0);
}

__global__ void k_hashgrid_bwd(const float* __restrict__ x, uint32_t E, const float* __restrict__ g_out, const mi3d_hashgrid hg,
                               float* __restrict__ g_table) {
    __shared__ LevelSm lv[16];
    if (threadIdx.x < 16) {
        LevelSm L; const int l = threadIdx.x;
        if (l < (int)hg.n_levels) {
            L.offset = hg.offsets[l]; L.size = hg.sizes[l]; L.res = hg.ress[l]; L.scale = hg.scales[l];
            L.hashed = (uint64_t)L.res * L.res * L.res > (uint64_t)L.size ? 1u : 0u;
        } else { L.offset = 0; L.size = 8; L.res = 2; L.scale = 1.f; L.hashed = 0; }
        lv[l] = L;
    }
    __syncthreads();
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int nl = (int)hg.n_levels;
    scatter_levels(g_table, lv, 0, nl, x[3 * (size_t)e], x[3 * (size_t)e + 1], x[3 * (size_t)e + 2], g_out + (size_t)e * 2 * nl, 1, 0);
}

// ---------------------------------------------------------------------------------------------------------
// density-grid refresh (nerf/renderer.py:587-637): cell centres + jitter, EMA-max, mean, threshold
// ---------------------------------------------------------------------------------------------------------
// positions for cascade `cas`, Morton-ordered: cell index m -> coords (morton inverse) -> xyz
__global__ void k_grid_positions(uint32_t H, float cas_bound, const float* __restrict__ jitter, uint64_t seed, uint32_t cas,
                                 float* __restrict__ xyz) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = H * H * H;
    if (m >= n) return;
    const float half_grid = cas_bound / (float)H;
    const uint32_t c[3] = {mi3d_compact3(m), mi3d_compact3(m >> 1), mi3d_compact3(m >> 2)};
    float u[3];
    if (jitter) { u[0] = jitter[3 * (size_t)m]; u[1] = jitter[3 * (size_t)m + 1]; u[2] = jitter[3 * (size_t)m + 2]; }
    else {
        const uint4 r = mi3d_philox(make_uint4(m, cas, 0u, 0x67726964u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
        u[0] = mi3d_u01(r.x); u[1] = mi3d_u01(r.y); u[2] = mi3d_u01(r.z);
    }
    #pragma unroll
    for (int d = 0; d < 3; d++) {
        const float base = 2.f * (float)c[d] / (float)(H - 1) - 1.f;           // renderer.py:608
        float v = base * (cas_bound - half_grid);                              // :615
        v += (u[d] * 2.f - 1.f) * half_grid;                                   // :617
        xyz[3 * (size_t)m + d] = v;
    }
}

// grid[cas][m] = max(grid*decay, sigma) where grid >= 0 ; block partial sums of the valid cells for the mean
__global__ void k_grid_ema(float* __restrict__ grid, const float* __restrict__ sigmas, uint32_t n, float decay,
                           float* __restrict__ partial_sum, uint32_t* __restrict__ partial_cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float v = 0.f; uint32_t c = 0;
    if (i < n) {
        float g = grid[i];
        if (g >= 0.f) { g = fmaxf(g * decay, sigmas[i]); grid[i] = g; v = g; c = 1; }
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    __shared__ float sv[8]; __shared__ uint32_t sc[8];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; sc[threadIdx.x >> 5] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float tv = 0.f; uint32_t tc = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) { tv += sv[w]; tc += sc[w]; }
        partial_sum[blockIdx.x] = tv; partial_cnt[blockIdx.x] = tc;
    }
}

__global__ void k_grid_mean(const float* __restrict__ partial_sum, const uint32_t* __restrict__ partial_cnt, uint32_t nparts,
                            float* __restrict__ mean_out) {
    __shared__ double sv[256]; __shared__ unsigned long long sc[256];
    double v = 0; unsigned long long c = 0;
    for (uint32_t i = threadIdx.x; i < nparts; i += blockDim.x) { v += (double)partial_sum[i]; c += partial_cnt[i]; }
    sv[threadIdx.x] = v; sc[threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if ((int)threadIdx.x < o) { sv[threadIdx.x] += sv[threadIdx.x + o]; sc[threadIdx.x] += sc[threadIdx.x + o]; } __syncthreads(); }
    if (threadIdx.x == 0) *mean_out = sc[0] ? (float)(sv[0] / (double)sc[0]) : 0.f;
}

int g_num_sms = 0;
int num_sms() {
    if (g_num_sms == 0) {
        int dev = 0; cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) g_num_sms = 132;
    }
    return g_num_sms;
}

bool g_attr_set = false;
int ensure_attrs() {
    if (!g_attr_set) {
        MI3D_CHECK(cudaFuncSetAttribute(k_field_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdSmem));
        MI3D_CHECK(cudaFuncSetAttribute(k_field_fwd_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwdtc::kSmem));
        MI3D_CHECK(cudaFuncSetAttribute(k_field_bwd_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwdtc::kSmem));
        g_attr_set = true;
    }
    return MI3D_OK;
}

}  // namespace

extern "C" {

int mi3d_hashgrid_make(uint32_t n_levels, uint32_t base_resolution, double per_level_scale, uint32_t log2_hashmap_size, mi3d_hashgrid* out) {
    if (!out || n_levels == 0 || n_levels > 16 || log2_hashmap_size > 28) return MI3D_ERR_ARG;
    uint32_t off = 0;
    const uint64_t cap = (uint64_t)1 << log2_hashmap_size;
    for (uint32_t l = 0; l < 16; l++) { out->offsets[l] = 0; out->sizes[l] = 0; out->ress[l] = 0; out->scales[l] = 0.f; }
    for (uint32_t l = 0; l < n_levels; l++) {
        const float scale = exp2f((float)l * log2f((float)per_level_scale)) * (float)base_resolution - 1.0f;
        const uint32_t res = (uint32_t)ceilf(scale) + 1;
        const uint64_t dense = (uint64_t)res * res * res;
        uint64_t size = dense < cap ? dense : cap;
        size = (size + 7) / 8 * 8;
        if (size > cap) size = cap;
        out->offsets[l] = off; out->sizes[l] = (uint32_t)size; out->ress[l] = res; out->scales[l] = scale;
        off += (uint32_t)size;
    }
    out->n_levels = n_levels;
    out->n_entries = off;
    return MI3D_OK;
}

int mi3d_hashgrid_forward(const float* x, uint32_t E, const float* table, const mi3d_hashgrid* hg, float* out, mi3d_stream_t stream) {
    if (E == 0) return MI3D_OK;
    if (!hg) return MI3D_ERR_ARG;
    k_hashgrid_fwd<<<mi3d_ceil_div(E, 128), 128, 0, (cudaStream_t)stream>>>(x, E, table, *hg, out);
    MI3D_RETURN_LAUNCH();
}

int mi3d_hashgrid_backward(const float* x, uint32_t E, const float* grad_out, const mi3d_hashgrid* hg, float* grad_table, mi3d_stream_t stream) {
    if (E == 0) return MI3D_OK;
    if (!hg) return MI3D_ERR_ARG;
    k_hashgrid_bwd<<<mi3d_ceil_div(E, 128), 128, 0, (cudaStream_t)stream>>>(x, E, grad_out, *hg, grad_table);
    MI3D_RETURN_LAUNCH();
}

constexpr uint32_t kBwdChunkTiles = 8192;     // 1 048 576 samples per chunk: 1.74 GB of encoding staging

size_t mi3d_field_backward_workspace_bytes(void) { return (size_t)kBwdChunkTiles * 13 * T * 32 * sizeof(float); }

int mi3d_field_grid_ctas(int backward) { return num_sms() * (backward ? 1 : 2); }

int mi3d_field_forward(const mi3d_field_io* io, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                       const mi3d_field_cfg* cfg, float* sigmas, float* rgbs, float* normals, float* tape,
                       float* loss_partials, float* loss_orient, float* loss_smooth, mi3d_stream_t stream) {
    if (!io || !hg || !mlp || !cfg || !sigmas) return MI3D_ERR_ARG;
    if (cfg->n_evals != 1 && cfg->n_evals != 7 && cfg->n_evals != 13) return MI3D_ERR_ARG;
    if (hg->n_levels * 2 != D_IN) return MI3D_ERR_ARG;
    if ((loss_orient || loss_smooth) && !loss_partials) return MI3D_ERR_ARG;
    MI3D_CHECK((cudaError_t)ensure_attrs());
    FwdArgs a{};
    a.xyzs = io->xyzs; a.dirs = io->dirs; a.counter = io->counter; a.m_fixed = io->m_fixed; a.align = io->align; a.cap = io->cap;
    a.table = table; a.hg = *hg; a.mlp = *mlp;
    a.bound = cfg->bound; a.blob_density = cfg->blob_density; a.two_r2 = (float)(2.0 * (double)cfg->blob_radius * (double)cfg->blob_radius);
    a.n_evals = cfg->n_evals; a.shading = cfg->shading; a.ratio = cfg->ambient_ratio; a.light_d = cfg->light_d;
    a.smooth_noise = io->smooth_noise; a.seed = io->seed;
    a.sigmas = sigmas; a.rgbs = rgbs; a.normals = normals; a.tape = tape; a.loss_partials = loss_partials;
    a.enc_cache = io->enc_cache; a.enc_cache_tiles = io->enc_cache_tiles;
    a.segs = io->segs; a.noise_mode = io->noise_mode;
    if (io->segs && (io->n_views == 0 || io->n_views > MI3D_MAX_VIEWS)) return MI3D_ERR_ARG;
    const int grid = num_sms();
    k_field_fwd_tc<<<grid, fwdtc::kThreads, fwdtc::kSmem, (cudaStream_t)stream>>>(a);
    if (loss_orient || loss_smooth)
        k_loss_finalize<<<1, 32, 0, (cudaStream_t)stream>>>(loss_partials, grid, io->counter, io->m_fixed, io->align, io->cap, loss_orient, loss_smooth,
                                                             io->segs ? (int)io->n_views : 0);
    MI3D_RETURN_LAUNCH();
}

int mi3d_field_backward(const mi3d_field_io* io, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                        const mi3d_field_cfg* cfg, const float* tape, const float* grad_sigmas, const float* grad_rgbs,
                        const float* grad_normals, const float* grad_loss_orient, const float* grad_loss_smooth,
                        float* grad_table, const mi3d_mlp_grad* grad_mlp, void* workspace, mi3d_stream_t stream) {
    if (!io || !hg || !mlp || !cfg || !tape || !grad_table || !grad_mlp) return MI3D_ERR_ARG;
    if (cfg->n_evals != 1 && cfg->n_evals != 7 && cfg->n_evals != 13) return MI3D_ERR_ARG;
    if (hg->n_levels * 2 != D_IN) return MI3D_ERR_ARG;
    MI3D_CHECK((cudaError_t)ensure_attrs());
    BwdArgs a{};
    a.xyzs = io->xyzs; a.dirs = io->dirs; a.counter = io->counter; a.m_fixed = io->m_fixed; a.align = io->align; a.cap = io->cap;
    a.table = table; a.hg = *hg; a.mlp = *mlp;
    a.bound = cfg->bound; a.blob_density = cfg->blob_density; a.two_r2 = (float)(2.0 * (double)cfg->blob_radius * (double)cfg->blob_radius);
    a.n_evals = cfg->n_evals; a.shading = cfg->shading; a.ratio = cfg->ambient_ratio; a.light_d = cfg->light_d;
    a.smooth_noise = io->smooth_noise; a.seed = io->seed;
    a.tape = tape; a.g_sigmas = grad_sigmas; a.g_rgbs = grad_rgbs; a.g_normals = grad_normals;
    a.g_loss_orient = grad_loss_orient; a.g_loss_smooth = grad_loss_smooth;
    a.g_table = grad_table; a.g_mlp = *grad_mlp;
    a.enc_buf = nullptr; a.tile0 = 0; a.tile1 = 0xFFFFFFFFu;
    a.segs = io->segs; a.noise_mode = io->noise_mode;
    if (io->segs && (io->n_views == 0 || io->n_views > MI3D_MAX_VIEWS)) return MI3D_ERR_ARG;
    if (workspace) {
        // chunk by chunk (the sample count lives on the device: chunks past it return immediately): gather kernel, then the chain
        // kernel, whose encoder warps scatter d(enc) themselves from shared memory -- the RED stream is bound by the load / store unit,
        // the MMA / epilogue chain by its serial hand-offs, so they overlap in one kernel
        float* enc_tmp = (float*)workspace;
        const bool cached = io->enc_cache && io->enc_cache_valid;
        const uint32_t total_tiles = (io->cap + T - 1) / T;
        for (uint32_t t0 = 0; t0 < total_tiles; t0 += kBwdChunkTiles) {
            a.tile0 = t0; a.tile1 = t0 + kBwdChunkTiles;
            if (cached && (t0 + kBwdChunkTiles < total_tiles ? t0 + kBwdChunkTiles : total_tiles) <= io->enc_cache_tiles)
                a.enc_buf = io->enc_cache + (size_t)t0 * 13 * T * 32;   // saved by the forward
            else { a.enc_buf = enc_tmp; k_bwd_enc_scatter<<<num_sms() * 4, 512, 0, (cudaStream_t)stream>>>(a); }
            k_field_bwd_tc<<<num_sms(), bwdtc::kThreads, bwdtc::kSmem, (cudaStream_t)stream>>>(a);
            if (!io->counter && (uint64_t)(t0 + kBwdChunkTiles) * T >= io->m_fixed) break;
        }
    } else {
        k_field_bwd_tc<<<num_sms(), bwdtc::kThreads, bwdtc::kSmem, (cudaStream_t)stream>>>(a);
    }
    MI3D_RETURN_LAUNCH();
}

#ifdef MI3D_FIELD_BWD_CLOCKS
// the counters of g_field_bwd_clocks since the previous call (8 values), then zeroes them; profiling builds only
extern "C" int mi3d_field_bwd_clocks(unsigned long long* out) {
    MI3D_CHECK(cudaDeviceSynchronize());
    MI3D_CHECK(cudaMemcpyFromSymbol(out, g_field_bwd_clocks, sizeof(g_field_bwd_clocks)));
    const unsigned long long zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    MI3D_CHECK(cudaMemcpyToSymbol(g_field_bwd_clocks, zero, sizeof(zero)));
    return MI3D_OK;
}
#endif

size_t mi3d_field_enc_cache_bytes(uint32_t tiles) { return (size_t)tiles * 13 * T * 32 * sizeof(float); }

size_t mi3d_density_grid_workspace_bytes(uint32_t C, uint32_t H) {
    const size_t n = (size_t)H * H * H;
    const size_t nparts = (n + 255) / 256;
    return n * 3 * sizeof(float) + n * sizeof(float) + (size_t)C * nparts * (sizeof(float) + sizeof(uint32_t)) + 256;
}

// nerf/renderer.py:587-637 without the two .item() host syncs: the mean density and the packing threshold
// min(mean, density_thresh) stay on the device (mean_density_out is a device scalar the caller may read later).
int mi3d_density_grid_update(float* density_grid, uint8_t* bitfield, uint32_t C, uint32_t H, float bound, float decay,
                             float density_thresh, const float* table, const mi3d_hashgrid* hg, const mi3d_mlp* mlp,
                             const mi3d_field_cfg* cfg, const float* jitter, uint64_t seed, float* mean_density_out,
                             void* workspace, mi3d_stream_t stream) {
    if (!density_grid || !bitfield || !hg || !mlp || !cfg || !workspace || !mean_density_out || C == 0 || C > 8) return MI3D_ERR_ARG;
    if (hg->n_levels * 2 != D_IN) return MI3D_ERR_ARG;
    MI3D_CHECK((cudaError_t)ensure_attrs());
    cudaStream_t st = (cudaStream_t)stream;
    const uint32_t n = H * H * H;
    const uint32_t nparts = mi3d_ceil_div(n, 256);
    float* xyz = (float*)workspace;
    float* sig = xyz + (size_t)n * 3;
    float* psum = sig + n;
    uint32_t* pcnt = (uint32_t*)(psum + (size_t)nparts * C);
    for (uint32_t cas = 0; cas < C; cas++) {
        const float cas_bound = fminf((float)(1u << cas), bound);                 // renderer.py:612
        k_grid_positions<<<nparts, 256, 0, st>>>(H, cas_bound, jitter ? jitter + (size_t)cas * n * 3 : nullptr, seed, cas, xyz);
        k_field_fwd<<<mi3d_field_grid_ctas(0), NT, kFwdSmem, st>>>(xyz, n, table, *hg, *mlp, cfg->bound, cfg->blob_density,
                                                                   (float)(2.0 * (double)cfg->blob_radius * (double)cfg->blob_radius), sig);
        k_grid_ema<<<nparts, 256, 0, st>>>(density_grid + (size_t)cas * n, sig, n, decay, psum + (size_t)cas * nparts, pcnt + (size_t)cas * nparts);
    }
    k_grid_mean<<<1, 256, 0, st>>>(psum, pcnt, nparts * C, mean_density_out);
    MI3D_CHECK(cudaGetLastError());
    return mi3d_packbits(density_grid, C * (n / 8), density_thresh, mean_density_out, bitfield, stream);
}

}  // extern "C"
