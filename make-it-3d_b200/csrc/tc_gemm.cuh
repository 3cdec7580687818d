// tc_gemm.cuh -- the one tensor-core tile kernel behind every dense contraction of the SD guidance path
// (nerf/sd.py:117-174: U-Net convs / linears / attention products, VAE encoder forward and input-gradient).
//
// sm_90a: operands are staged by TMA (cp.async.bulk.tensor, 128B swizzle) into a multi-stage shared-memory ring and multiplied by
// wgmma.mma_async (fp16 in, fp32 accumulate in registers) by two consumer warpgroups, each owning 64 rows of the 128-row tile; the
// same warpgroups run the epilogue straight from their accumulator registers (bias / time-embedding / residual / GEGLU /
// transposed store) and write fp16 (or fp32) to HBM.
//
//   D[m, n] = sum_k A[m, k] * B[n, k]         A, B both K-major (K contiguous), fp16 in, fp32 accumulate
//
// Two A-operand addressing modes share the kernel:
//   PLAIN : A is a (K, M, Z1, Z2) tensor map; blockIdx.z selects (z % a_z1, z / a_z1)  (batched / per-head GEMMs)
//   CONV3 : implicit GEMM for a 3x3 stride-1 pad-1 convolution over an NHWC activation: A is a (C, W, H, N) tensor
//           map, the K loop runs over 9 taps x C/64 channel blocks, each stage is ONE 4-D TMA box shifted by the tap
//           offset; out-of-bounds rows/columns are zero-filled by the TMA unit (that is the padding).
//   CONV3_BLOCK (conv = 2, k_tc_gemm_vgg only): the same implicit conv for any H x W: a 128-row M tile is a conv_bw x conv_bh spatial
//           block of one image (m_blk -> image, block row, block column); the box may overhang the right / bottom edge (zero-filled
//           loads) and the epilogue stores only the in-image pixels, at NHWC row (n * H + y) * W + x.
//
// Warp roles (384 threads): warp 0 = TMA producer (warps 1..3 idle), warpgroups 1 and 2 = MMA + epilogue for tile rows 0..63 / 64..127.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "tc_host.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace tc {

constexpr int MMA_K = 16;
constexpr int kThreads = 384;

template <int BLOCK_N> struct Cfg {
    static constexpr int kStages = BLOCK_N == 256 ? 4 : (BLOCK_N == 128 ? 6 : (BLOCK_N == 160 ? 5 : 4));   // BN=64: 96 KB -> 2 CTAs/SM
    static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
    static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr size_t kSmemBytes = 1024 /*align slack*/ + (size_t)kStages * kStageBytes + 256;
    static constexpr int kMinBlocks = BLOCK_N == 64 ? 2 : 1;
    // 8-column groups whose epilogue inputs are loaded together: as many as the register budget holds without spilling
    // (BN = 256: the accumulator takes 128 of 168 registers; BN = 64: two CTAs per SM cap a thread at 85).  The QuickGELU
    // instantiation at BN = 256 holds one group (with two it spills).
    template <bool kQuickGelu> static constexpr int kEpiChunk = (BLOCK_N == 128 || BLOCK_N == 160) ? 4 : (kQuickGelu && BLOCK_N == 256 ? 1 : 2);
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float quick_gelu(float x) { return x / (1.f + __expf(-1.702f * x)); }
__device__ __forceinline__ float quick_gelu_grad(float x) { const float s = 1.f / (1.f + __expf(-1.702f * x)); return s * (1.f + 1.702f * x * (1.f - s)); }

// acc (+)= A[64 x 16] . B[BLOCK_N x 16]^T, both K-major
template <int BLOCK_N>
__device__ __forceinline__ void mma_tile(float (&acc)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (BLOCK_N == 64) wg::wgmma_f16_n64<0, 0>(acc, da, db, accumulate);
    else if constexpr (BLOCK_N == 128) wg::wgmma_f16_n128<0, 0>(acc, da, db, accumulate);
    else if constexpr (BLOCK_N == 160) wg::wgmma_f16_n160<0, 0>(acc, da, db, accumulate);
    else wg::wgmma_f16_n256<0, 0>(acc, da, db, accumulate);
}

// The kernel body.  kQuickGelu: the instantiation that also carries the EPI_QUICKGELU* epilogues; kVgg: the one that carries the
// CONV3_BLOCK mode and the EPI_RELU* epilogues; kGelu: the one that carries EPI_GELU.  Each is a compile-time switch, so the other
// modes compile exactly as without them.
template <int BLOCK_N, bool kQuickGelu, bool kVgg, bool kGelu = false>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& map_a, const CUtensorMap& map_b, const GemmParams& p) {
    using C = Cfg<BLOCK_N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    uint8_t* tiles = smem;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)C::kStages * C::kStageBytes);
    uint64_t* empty_bar = full_bar + C::kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&map_a); prefetch_tmap(&map_b);
        for (int s = 0; s < C::kStages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // empty: one arrive per consumer warp
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 0) {
        // ===================== TMA producer =====================
        // whole warp on the (uniform) loop and the barrier waits, one elected lane issues: see elect_one()
        int stage = 0; uint32_t phase = 0;
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
            const int sp = t % p.splits, tt = t / p.splits;
            const int n_blk = tt % p.n_tiles, rest = tt / p.n_tiles, m_blk = rest % p.m_tiles, z = rest / p.m_tiles;
            const int kb0 = sp * p.kb_per_split, kb1 = min(p.num_k_blocks, kb0 + p.kb_per_split);
            const int m0 = m_blk * BLOCK_M, n0 = n_blk * BLOCK_N;
            int cw = 0, ch = 0, cn = 0;
            if (kVgg && p.conv == 2) {
                const int bx = (p.conv_W + p.conv_bw - 1) / p.conv_bw, by = (p.conv_H + p.conv_bh - 1) / p.conv_bh;
                cn = m_blk / (bx * by); const int rem = m_blk - cn * bx * by;
                ch = rem / bx * p.conv_bh; cw = (rem % bx) * p.conv_bw;
            } else if (p.conv) {
                const int hw = p.conv_H * p.conv_W;
                cn = m0 / hw; const int rem = m0 - cn * hw;
                ch = rem / p.conv_W; cw = rem - ch * p.conv_W;
            }
            const int az0 = p.a_z1 > 0 ? z % p.a_z1 : 0, az1 = p.a_z1 > 0 ? z / p.a_z1 : 0;
            const int bz0 = p.b_batched ? (p.b_z1 > 0 ? z % p.b_z1 : 0) : 0, bz1 = p.b_batched ? (p.b_z1 > 0 ? z / p.b_z1 : 0) : 0;
            for (int kb = kb0; kb < kb1; kb++) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* sa = tiles + (size_t)stage * C::kStageBytes;
                uint8_t* sb = sa + C::kABytes;
                int c0 = kb * BLOCK_K, c1 = m0, c2 = az0, c3 = az1;
                if (p.conv) {
                    const int tap = kb / p.cin_blocks, cc = kb - tap * p.cin_blocks;
                    const int ky = tap / 3, kx = tap - ky * 3;
                    c0 = cc * BLOCK_K; c1 = cw + kx - 1; c2 = ch + ky - 1; c3 = cn;
                }
                if (elect_one()) {
                    mbar_arrive_expect_tx(&full_bar[stage], C::kStageBytes);
                    tma_load_4d(&map_a, &full_bar[stage], sa, c0, c1, c2, c3);
                    tma_load_4d(&map_b, &full_bar[stage], sb, kb * BLOCK_K, n0, bz0, bz1);
                }
                __syncwarp();
                if (++stage == C::kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup g owns tile rows 64 g .. 64 g + 63 =====================
        const int g = (warp >> 2) - 1, wl = warp & 3;
        const uint32_t tiles_u = smem_u32(tiles);
        int stage = 0; uint32_t phase = 0;
        float acc[BLOCK_N / 2];
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
            const int sp = t % p.splits, tt = t / p.splits;
            const int n_blk = tt % p.n_tiles, rest = tt / p.n_tiles, m_blk = rest % p.m_tiles, z = rest / p.m_tiles;
            const int kb0 = sp * p.kb_per_split, kb1 = min(p.num_k_blocks, kb0 + p.kb_per_split);
            #pragma unroll
            for (int i = 0; i < BLOCK_N / 2; i++) acc[i] = 0.f;          // an empty K-range (never planned) still stores zeros
            int prev = -1;
            for (int kb = kb0; kb < kb1; kb++) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t sa = tiles_u + (uint32_t)stage * (uint32_t)C::kStageBytes;
                const uint64_t da = wg::desc_sw128(sa + (uint32_t)g * 8192u);            // 64 rows x 128 B further down the A tile
                wg::fence();
                const uint64_t db = wg::desc_sw128(sa + C::kABytes);
                #pragma unroll
                for (int k = 0; k < BLOCK_K / MMA_K; k++)                                  // +32 B inside the swizzle row (>>4 => +2)
                    mma_tile<BLOCK_N>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > kb0 || k > 0) ? 1u : 0u);
                wg::commit();
                wg::wait<1>();                                   // the previous stage's MMAs have retired: hand its buffers back
                if (prev >= 0 && lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty_bar[prev])) : "memory");
                prev = stage;
                if (++stage == C::kStages) { stage = 0; phase ^= 1; }
            }
            wg::wait<0>();
            wg::reg_fence(acc);
            if (prev >= 0 && lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty_bar[prev])) : "memory");

            // epilogue: this thread holds rows r0 and r0 + 8, columns 8 j + 2 (lane % 4) + {0, 1}
            const size_t zoff = (size_t)(z % p.out_z1) * p.out_s_lo + (size_t)(z / p.out_z1) * p.out_s_hi;
            #pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                int m = m_blk * BLOCK_M + g * 64 + wl * 16 + (lane >> 2) + 8 * hh;
                if (kVgg && p.conv == 2) {
                    // tile row -> pixel of the spatial block; rows over the right / bottom edge are not stored
                    const int bx = (p.conv_W + p.conv_bw - 1) / p.conv_bw, by = (p.conv_H + p.conv_bh - 1) / p.conv_bh;
                    const int r = m - m_blk * BLOCK_M, n = m_blk / (bx * by), rem = m_blk - n * bx * by;
                    const int y = rem / bx * p.conv_bh + r / p.conv_bw, x = (rem % bx) * p.conv_bw + r % p.conv_bw;
                    if (x >= p.conv_W || y >= p.conv_H) continue;
                    m = (n * p.conv_H + y) * p.conv_W + x;
                }
                const bool row_ok = m < p.m_valid;
                if (!row_ok) continue;
                const float* rb = p.row_bias ? p.row_bias + (size_t)(((long long)z * p.M + m) / p.rows_per_group) * p.N : nullptr;
                if (p.splits > 1) {
                    // split-K partial: fp32 RED into the workspace; bias / residual / conversion happen in k_splitk_finish
                    #pragma unroll
                    for (int j = 0; j < BLOCK_N / 8; j++)
                        atomicAdd(reinterpret_cast<float2*>(p.splitk_ws + (size_t)m * p.N + n_blk * BLOCK_N + 8 * j + 2 * (lane & 3)),
                                  make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]));
                    continue;
                }
                // the epilogue's bias and fp16 input (residual / aux) of kEpiChunk 8-column groups are loaded before any of their outputs
                // is stored: a load placed after a store waits for it (the pointers may alias), which made every group pay a full load
                // latency (the row bias, on the deep-K time-embedding convs only, is still read in place)
                const __half* in16 = nullptr;                  // the fp16 input of the mode, same row / column as the output
                long long ld_in = p.ldc;
                if (p.epi_mode == EPI_PLAIN && p.residual) { in16 = p.residual; ld_in = p.ld_res; }
                else if ((kQuickGelu && p.epi_mode == EPI_QUICKGELU_BWD) || (kVgg && p.epi_mode == EPI_RELU_BWD)) in16 = p.aux;
                constexpr int kChunk = C::template kEpiChunk<kQuickGelu>;
                #pragma unroll
                for (int j0 = 0; j0 < BLOCK_N / 8; j0 += kChunk) {
                    float2 bias_v[kChunk];
                    __half2 in_v[kChunk];
                    #pragma unroll
                    for (int c = 0; c < kChunk; c++) {
                        const int n = n_blk * BLOCK_N + 8 * (j0 + c) + 2 * (lane & 3);
                        if (p.bias) bias_v[c] = __ldg(reinterpret_cast<const float2*>(p.bias + n));
                        if (in16) in_v[c] = *reinterpret_cast<const __half2*>(in16 + zoff + (size_t)m * ld_in + n);
                    }
                    #pragma unroll
                    for (int c = 0; c < kChunk; c++) {
                        const int j = j0 + c;
                        const int n = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);
                        float f0 = acc[4 * j + 2 * hh], f1 = acc[4 * j + 2 * hh + 1];
                        f0 *= p.alpha; f1 *= p.alpha;
                        if (p.bias) { f0 += bias_v[c].x; f1 += bias_v[c].y; }
                        if (rb) { const float2 bv = __ldg(reinterpret_cast<const float2*>(rb + n)); f0 += bv.x; f1 += bv.y; }
                        if (p.epi_mode == EPI_GEGLU) {
                            // weight rows were interleaved (value, gate) at plan time: out[:, n/2] = value * gelu(gate)
                            p.out[zoff + (size_t)m * p.ldc + (n >> 1)] = __float2half_rn(f0 * gelu_erf(f1));
                        } else if (p.epi_mode == EPI_TRANSPOSED) {
                            __half* o = p.out + zoff + (size_t)n * p.ldc + m;
                            o[0] = __float2half_rn(f0); o[p.ldc] = __float2half_rn(f1);
                        } else if (kQuickGelu && p.epi_mode == EPI_QUICKGELU) {
                            const size_t o = zoff + (size_t)m * p.ldc + n;
                            if (p.aux) *reinterpret_cast<__half2*>(p.aux + o) = __floats2half2_rn(f0, f1);
                            *reinterpret_cast<__half2*>(p.out + o) = __floats2half2_rn(quick_gelu(f0), quick_gelu(f1));
                        } else if (kQuickGelu && p.epi_mode == EPI_QUICKGELU_BWD) {
                            const __half2 pre = in_v[c];
                            *reinterpret_cast<__half2*>(p.out + zoff + (size_t)m * p.ldc + n) =
                                __floats2half2_rn(f0 * quick_gelu_grad(__low2float(pre)), f1 * quick_gelu_grad(__high2float(pre)));
                        } else if (kVgg && p.epi_mode == EPI_RELU) {
                            *reinterpret_cast<__half2*>(p.out + zoff + (size_t)m * p.ldc + n) = __floats2half2_rn(fmaxf(f0, 0.f), fmaxf(f1, 0.f));
                        } else if (kVgg && p.epi_mode == EPI_RELU_BWD) {
                            const __half2 a = in_v[c];
                            *reinterpret_cast<__half2*>(p.out + zoff + (size_t)m * p.ldc + n) =
                                __floats2half2_rn(__low2float(a) > 0.f ? f0 : 0.f, __high2float(a) > 0.f ? f1 : 0.f);
                        } else if (kGelu && p.epi_mode == EPI_GELU) {
                            *reinterpret_cast<__half2*>(p.out + zoff + (size_t)m * p.ldc + n) = __floats2half2_rn(gelu_erf(f0), gelu_erf(f1));
                        } else {
                            if (in16) { f0 += __low2float(in_v[c]); f1 += __high2float(in_v[c]); }
                            if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + zoff + (size_t)m * p.ldc + n) = make_float2(f0, f1);
                            else *reinterpret_cast<__half2*>(p.out + zoff + (size_t)m * p.ldc + n) = __floats2half2_rn(f0, f1);
                        }
                    }
                }
            }
        }
    }
}

template <int BLOCK_N, bool kQuickGelu = false>
__global__ void __launch_bounds__(kThreads, Cfg<BLOCK_N>::kMinBlocks)
k_tc_gemm(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
    tc_gemm_body<BLOCK_N, kQuickGelu, false>(map_a, map_b, p);
}

// VGG19's convs (cx_engine.cu): CONV3_BLOCK tiles, EPI_RELU / EPI_RELU_BWD epilogues
template <int BLOCK_N>
__global__ void __launch_bounds__(kThreads, Cfg<BLOCK_N>::kMinBlocks)
k_tc_gemm_vgg(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
    tc_gemm_body<BLOCK_N, false, true>(map_a, map_b, p);
}

// the SD-2 text encoder's MLP input GEMM (sd_text_engine.cu): EPI_GELU epilogue
template <int BLOCK_N>
__global__ void __launch_bounds__(kThreads, Cfg<BLOCK_N>::kMinBlocks)
k_tc_gemm_gelu(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
    tc_gemm_body<BLOCK_N, false, false, true>(map_a, map_b, p);
}

// split-K epilogue: out = alpha * ws + bias + row_bias (+ residual) -> fp16 ; 8 elements per thread
static __global__ void k_splitk_finish(const float* __restrict__ ws, const GemmParams p) {
    const size_t total = (size_t)p.m_valid * p.N / 8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e0 = i * 8; const int m = (int)(e0 / p.N), n0 = (int)(e0 % p.N);
        const float4 a = *reinterpret_cast<const float4*>(ws + e0), b = *reinterpret_cast<const float4*>(ws + e0 + 4);
        float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        const float* rb = p.row_bias ? p.row_bias + (size_t)(m / p.rows_per_group) * p.N : nullptr;
        #pragma unroll
        for (int k = 0; k < 8; k++) { f[k] *= p.alpha; if (p.bias) f[k] += p.bias[n0 + k]; if (rb) f[k] += rb[n0 + k]; }
        if (p.residual) {
            const uint4 rv = *reinterpret_cast<const uint4*>(p.residual + (size_t)m * p.ld_res + n0);
            const __half* rh = reinterpret_cast<const __half*>(&rv);
            #pragma unroll
            for (int k = 0; k < 8; k++) f[k] += __half2float(rh[k]);
        }
        __align__(16) __half h[8];
        #pragma unroll
        for (int k = 0; k < 8; k++) h[k] = __float2half_rn(f[k]);
        *reinterpret_cast<uint4*>(p.out + (size_t)m * p.ldc + n0) = *reinterpret_cast<const uint4*>(h);
    }
}

}  // namespace tc
