// attn.cuh -- fused multi-head attention (softmax(Q K^T / sqrt(d)) V) for the U-Net transformer blocks and the CLIP-style towers,
// head_dim d in {40, 64, 80, 160} (SD-2.x and the towers: 64; SD-1.x: 40, 80, 160).
//
// Replaces the three-launch form (batched QK^T tile GEMM -> softmax over the materialised [B*heads, T, Tk] fp16 score tensor ->
// batched PV tile GEMM) that stood in for diffusers' attention processor under nerf/sd.py:146.  At 64x64 latents one layer's
// score tensor is 335 MB; here scores never leave the SM: S and O live in registers, P goes straight from the S accumulator
// registers into the A operand of the second product.
//
// One CTA = one 128-query tile of one (batch, head).  288 threads:
//   warpgroups 0, 1  query rows 0..63 / 64..127 of the tile: S = Q K_j^T (wgmma m64 nKB k16, both K-major from shared memory),
//                    online softmax in registers, O += P_j V_j (wgmma m64 n<=64 k16 per 64-column chunk of the head, P from
//                    registers, V MN-major as loaded)
//   warp 8           TMA producer: Q once, K and V double-buffered (4D maps: d, token, head, batch; 128B swizzle)
// A head is loaded as ceil(d / 64) boxes of 64 columns; TMA zero-fills the columns past d, so every chunk is an ordinary
// 128B-swizzled 64-column tile.  Q K^T issues ceil(d / 16) k16 steps (the zero tail of a chunk takes part only up to the next
// multiple of 16); P V issues one product per chunk, 64 wide or exactly the tail's width, so O holds d columns per row.
//   d = 40, 64: 1 chunk,  KB = 128 keys per block,  81 KB shared memory;  S 64, P 32, O 20 / 32 registers per thread
//   d = 80:     2 chunks, KB = 128,                161 KB;                  S 64, P 32, O 40
//   d = 160:    3 chunks, KB = 64,                 145 KB;                  S 32, P 16, O 80  (128-key blocks would need 240 KB)
// Every instantiation fits one CTA per SM without spills.
#pragma once
#include <cmath>
#include "tc_host.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace attn {
using namespace tc;

constexpr int kThreads = 288;
constexpr int kTile = 16384;                                 // 128 rows x 128 B: one 64-column chunk of the 128-query tile

template <int D> struct Shape {
    static constexpr int kChunks = (D + 63) / 64;            // 64-column chunks of a head
    static constexpr int kTail = D - 64 * (kChunks - 1);      // columns of the last chunk: 40, 64, 16, 32
    static constexpr int kKeys = D > 128 ? 64 : 128;          // keys per K / V block
    static constexpr int kKeysLog2 = D > 128 ? 6 : 7;
    static constexpr int kSteps = (D + 15) / 16;              // k16 steps of Q K^T
    static constexpr int kKVBytes = kChunks * kKeys * 128;    // one stage of K or of V
    static constexpr size_t kSmemBytes = 1024 + (size_t)kChunks * kTile + 4 * (size_t)kKVBytes + 256;   // Q, K0, K1, V0, V1 + barriers
    static_assert(D % 8 == 0 && D >= 16 && kChunks <= 3 && (kTail == 64 || kTail == 40 || kTail == 32 || kTail == 16), "head_dim");
    static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

struct Params {
    int T;              // queries per (batch, head)
    int kv_valid;       // keys per (batch, head) that take part (77 of the 128 padded context rows for cross attention)
    int ldo;            // row stride of o (elements)
    float scale_log2e;  // (1 / sqrt(d)) * log2(e)
    __half* o;          // [B*T, ldo], head h at column h * d
};

__device__ __forceinline__ float ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }   // one MUFU, no range fix-up
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}
// O[:, 0:N) of one chunk += P (16 keys, registers) . V (16 keys x N columns, MN-major)
template <int N> __device__ __forceinline__ void pv(float* o, const uint32_t (&a)[4], uint64_t dv) {
    if constexpr (N == 64) wg::wgmma_f16_rs_n64<1>(*reinterpret_cast<float(*)[32]>(o), a, dv, 1u);
    else if constexpr (N == 40) wg::wgmma_f16_rs_n40<1>(*reinterpret_cast<float(*)[20]>(o), a, dv, 1u);
    else if constexpr (N == 32) wg::wgmma_f16_rs_n32<1>(*reinterpret_cast<float(*)[16]>(o), a, dv, 1u);
    else wg::wgmma_f16_rs_n16<1>(*reinterpret_cast<float(*)[8]>(o), a, dv, 1u);
}

template <int D>
static __global__ void __launch_bounds__(kThreads, 1)
k_flash_attn(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
             const Params p) {
    using Sh = Shape<D>;
    constexpr int NC = Sh::kChunks, KB = Sh::kKeys, KVB = Sh::kKVBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    uint8_t* sQ = smem;                  // NC chunks of kTile
    uint8_t* sK = sQ + NC * kTile;       // two stages of NC chunks of KB rows
    uint8_t* sV = sK + 2 * KVB;          // two stages
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * KVB);
    uint64_t* q_full = bars + 0;
    uint64_t* k_full = bars + 1;         // [2]
    uint64_t* k_empty = bars + 3;        // [2]
    uint64_t* v_full = bars + 5;         // [2]
    uint64_t* v_empty = bars + 7;        // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 128, head = blockIdx.y, batch = blockIdx.z;
    const int nkv = (p.kv_valid + KB - 1) >> Sh::kKeysLog2;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&map_q); prefetch_tmap(&map_k); prefetch_tmap(&map_v);
        mbar_init(q_full, 1);
        for (int s = 0; s < 2; s++) { mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 8); mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===================== TMA producer =====================
        // whole warp on the (uniform) loop and the barrier waits, one elected lane issues: see tc::elect_one()
        if (elect_one()) {
            mbar_arrive_expect_tx(q_full, NC * kTile);
            #pragma unroll
            for (int c = 0; c < NC; c++) tma_load_4d(&map_q, q_full, sQ + c * kTile, 64 * c, q0, head, batch);
        }
        __syncwarp();
        for (int j = 0; j < nkv; j++) {
            const int st = j & 1;
            const uint32_t par = (((uint32_t)j >> 1) & 1u) ^ 1u;
            mbar_wait(&k_empty[st], par);
            if (elect_one()) {
                mbar_arrive_expect_tx(&k_full[st], KVB);
                #pragma unroll
                for (int c = 0; c < NC; c++) tma_load_4d(&map_k, &k_full[st], sK + st * KVB + c * KB * 128, 64 * c, j * KB, head, batch);
            }
            __syncwarp();
            mbar_wait(&v_empty[st], par);
            if (elect_one()) {
                mbar_arrive_expect_tx(&v_full[st], KVB);
                #pragma unroll
                for (int c = 0; c < NC; c++) tma_load_4d(&map_v, &v_full[st], sV + st * KVB + c * KB * 128, 64 * c, j * KB, head, batch);
            }
            __syncwarp();
        }
    } else {
        // ===================== warpgroup g: query rows 64 g .. 64 g + 63 of the tile =====================
        // this thread holds rows r and r + 8 (r = 16 wl + lane / 4), columns 8 j + 2 (lane % 4) + {0, 1} of every n8 block j
        // (of S: key j of the block; of O: column 8 j of the head, chunk c's n8 blocks at o[32 c ..])
        const int g = warp >> 2, wl = warp & 3;
        const float c = p.scale_log2e;
        const uint32_t sq_u = smem_u32(sQ) + (uint32_t)g * 8192u, sk_u = smem_u32(sK), sv_u = smem_u32(sV);
        float o[D / 2];
        #pragma unroll
        for (int i = 0; i < D / 2; i++) o[i] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        mbar_wait(q_full, 0);
        for (int j = 0; j < nkv; j++) {
            const int st = j & 1;
            const uint32_t par = ((uint32_t)j >> 1) & 1u;
            float s[KB / 2];
            mbar_wait(&k_full[st], par);
            wg::fence();
            {
                const uint64_t dq = wg::desc_sw128(sq_u), dk = wg::desc_sw128(sk_u + (uint32_t)(st * KVB));
                #pragma unroll
                for (int k = 0; k < Sh::kSteps; k++) {    // chunk k / 4, +32 B per k16 step inside its 128-byte rows
                    const uint64_t oq = (uint64_t)((k >> 2) * (kTile >> 4) + 2 * (k & 3)), ok = (uint64_t)((k >> 2) * (KB * 8) + 2 * (k & 3));
                    if constexpr (KB == 128) wg::wgmma_f16_n128<0, 0>(s, dq + oq, dk + ok, k > 0 ? 1u : 0u);
                    else wg::wgmma_f16_n64<0, 0>(s, dq + oq, dk + ok, k > 0 ? 1u : 0u);
                }
            }
            wg::commit();
            wg::wait<0>();
            wg::reg_fence(s);
            if (lane == 0) mbar_arrive(&k_empty[st]);
            const int kbase = j * KB;
            if (kbase + KB > p.kv_valid) {
                #pragma unroll
                for (int jj = 0; jj < KB / 8; jj++) {
                    const int col = kbase + 8 * jj + 2 * (lane & 3);
                    if (col >= p.kv_valid) { s[4 * jj] = -INFINITY; s[4 * jj + 2] = -INFINITY; }
                    if (col + 1 >= p.kv_valid) { s[4 * jj + 1] = -INFINITY; s[4 * jj + 3] = -INFINITY; }
                }
            }
            float mx0 = -INFINITY, mx1 = -INFINITY;
            #pragma unroll
            for (int jj = 0; jj < KB / 8; jj++) {
                mx0 = fmaxf(mx0, fmaxf(s[4 * jj], s[4 * jj + 1]));
                mx1 = fmaxf(mx1, fmaxf(s[4 * jj + 2], s[4 * jj + 3]));
            }
            #pragma unroll
            for (int off = 1; off <= 2; off <<= 1) {           // the four lanes of a row
                mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
                mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
            }
            // every key block holds at least one valid key, so the new maxima are finite
            const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
            const float al0 = ex2((m0 - mn0) * c), al1 = ex2((m1 - mn1) * c);      // 0 on the first block (m = -inf)
            m0 = mn0; m1 = mn1;
            l0 *= al0; l1 *= al1;
            #pragma unroll
            for (int jj = 0; jj < D / 8; jj++) { o[4 * jj] *= al0; o[4 * jj + 1] *= al0; o[4 * jj + 2] *= al1; o[4 * jj + 3] *= al1; }
            const float mc0 = m0 * c, mc1 = m1 * c;
            // P = ex2(s c - m c) -> fp16 A fragments: k16 block kk of P is n8 blocks 2 kk, 2 kk + 1 of S
            uint32_t a[KB / 16][4];
            #pragma unroll
            for (int kk = 0; kk < KB / 16; kk++) {
                float pr[8];
                #pragma unroll
                for (int i = 0; i < 8; i++) pr[i] = ex2(fmaf(s[8 * kk + i], c, (i & 2) ? -mc1 : -mc0));
                l0 += (pr[0] + pr[1]) + (pr[4] + pr[5]);
                l1 += (pr[2] + pr[3]) + (pr[6] + pr[7]);
                a[kk][0] = pack_h2(pr[0], pr[1]); a[kk][1] = pack_h2(pr[2], pr[3]);
                a[kk][2] = pack_h2(pr[4], pr[5]); a[kk][3] = pack_h2(pr[6], pr[7]);
            }
            mbar_wait(&v_full[st], par);
            wg::fence();
            {
                const uint32_t sv_st = sv_u + (uint32_t)(st * KVB);
                #pragma unroll
                for (int ch = 0; ch < NC - 1; ch++) {
                    const uint64_t dv = wg::desc_sw128(sv_st + (uint32_t)(ch * KB * 128), 8192u);
                    #pragma unroll
                    for (int kk = 0; kk < KB / 16; kk++) pv<64>(o + 32 * ch, a[kk], dv + (uint64_t)(128 * kk));   // 16 keys = 2048 B
                }
                const uint64_t dv = wg::desc_sw128(sv_st + (uint32_t)((NC - 1) * KB * 128), 8192u);
                #pragma unroll
                for (int kk = 0; kk < KB / 16; kk++) pv<Sh::kTail>(o + 32 * (NC - 1), a[kk], dv + (uint64_t)(128 * kk));
            }
            wg::commit();
            wg::wait<0>();
            wg::reg_fence(o);
            if (lane == 0) mbar_arrive(&v_empty[st]);
        }
        #pragma unroll
        for (int off = 1; off <= 2; off <<= 1) { l0 += __shfl_xor_sync(0xffffffffu, l0, off); l1 += __shfl_xor_sync(0xffffffffu, l1, off); }
        const float inv0 = 1.f / l0, inv1 = 1.f / l1;
        const int r = q0 + g * 64 + wl * 16 + (lane >> 2);
        #pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            if (r + 8 * hh >= p.T) continue;
            const float inv = hh ? inv1 : inv0;
            __half* dst = p.o + ((size_t)batch * p.T + r + 8 * hh) * p.ldo + head * D + 2 * (lane & 3);
            #pragma unroll
            for (int jj = 0; jj < D / 8; jj++)
                *reinterpret_cast<__half2*>(dst + 8 * jj) = __floats2half2_rn(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
        }
    }
}

}  // namespace attn
