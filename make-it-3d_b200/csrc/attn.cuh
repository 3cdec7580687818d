// attn.cuh -- fused multi-head attention (softmax(Q K^T / sqrt(d)) V) for the SD-2.0 U-Net transformer blocks, d = 64.
//
// Replaces the three-launch form (batched QK^T tile GEMM -> softmax over the materialised [B*heads, T, Tk] fp16 score tensor ->
// batched PV tile GEMM) that stood in for diffusers' attention processor under nerf/sd.py:146.  At 64x64 latents one layer's
// score tensor is 335 MB; here scores never leave the SM: S and O live in registers, P goes straight from the S accumulator
// registers into the A operand of the second product.
//
// One CTA = one 128-query tile of one (batch, head).  288 threads:
//   warpgroups 0, 1  query rows 0..63 / 64..127 of the tile: S = Q K_j^T (wgmma m64 n128 k16, both K-major from shared memory),
//                    online softmax in registers, O += P_j V_j (wgmma m64 n64 k16, P from registers, V MN-major as loaded)
//   warp 8           TMA producer: Q once, K and V double-buffered (4D maps: d, token, head, batch; 128B swizzle)
// 81 KB shared memory per CTA; S (64 registers), P (32) and O (32) per thread leave room for one CTA per SM without spills.
#pragma once
#include "tc_host.cuh"

namespace attn {
using namespace tc;

constexpr int kThreads = 288;
constexpr int kTile = 16384;                                 // 128 rows x 128 B
constexpr size_t kSmemBytes = 1024 + 5 * (size_t)kTile + 256;   // Q, K0, K1, V0, V1 + barriers

struct Params {
    int T;              // queries per (batch, head)
    int kv_valid;       // keys per (batch, head) that take part (77 of the 128 padded context rows for cross attention)
    int ldo;            // row stride of o (elements)
    float scale_log2e;  // (1 / sqrt(d)) * log2(e)
    __half* o;          // [B*T, ldo], head h at column h * 64
};

__device__ __forceinline__ float ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }   // one MUFU, no range fix-up
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

static __global__ void __launch_bounds__(kThreads, 1)
k_flash_attn(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
             const Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + kTile;            // two stages
    uint8_t* sV = sK + 2 * kTile;        // two stages
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * kTile);
    uint64_t* q_full = bars + 0;
    uint64_t* k_full = bars + 1;         // [2]
    uint64_t* k_empty = bars + 3;        // [2]
    uint64_t* v_full = bars + 5;         // [2]
    uint64_t* v_empty = bars + 7;        // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 128, head = blockIdx.y, batch = blockIdx.z;
    const int nkv = (p.kv_valid + 127) >> 7;

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
            mbar_arrive_expect_tx(q_full, kTile);
            tma_load_4d(&map_q, q_full, sQ, 0, q0, head, batch);
        }
        __syncwarp();
        for (int j = 0; j < nkv; j++) {
            const int st = j & 1;
            const uint32_t par = (((uint32_t)j >> 1) & 1u) ^ 1u;
            mbar_wait(&k_empty[st], par);
            if (elect_one()) {
                mbar_arrive_expect_tx(&k_full[st], kTile);
                tma_load_4d(&map_k, &k_full[st], sK + st * kTile, 0, j * 128, head, batch);
            }
            __syncwarp();
            mbar_wait(&v_empty[st], par);
            if (elect_one()) {
                mbar_arrive_expect_tx(&v_full[st], kTile);
                tma_load_4d(&map_v, &v_full[st], sV + st * kTile, 0, j * 128, head, batch);
            }
            __syncwarp();
        }
    } else {
        // ===================== warpgroup g: query rows 64 g .. 64 g + 63 of the tile =====================
        // this thread holds rows r and r + 8 (r = 16 wl + lane / 4), columns 8 j + 2 (lane % 4) + {0, 1} of every n8 block j
        const int g = warp >> 2, wl = warp & 3;
        const float c = p.scale_log2e;
        const uint32_t sq_u = smem_u32(sQ) + (uint32_t)g * 8192u, sk_u = smem_u32(sK), sv_u = smem_u32(sV);
        float o[32];
        #pragma unroll
        for (int i = 0; i < 32; i++) o[i] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        mbar_wait(q_full, 0);
        for (int j = 0; j < nkv; j++) {
            const int st = j & 1;
            const uint32_t par = ((uint32_t)j >> 1) & 1u;
            float s[64];
            mbar_wait(&k_full[st], par);
            wg::fence();
            {
                const uint64_t dq = wg::desc_sw128(sq_u), dk = wg::desc_sw128(sk_u + (uint32_t)(st * kTile));
                #pragma unroll
                for (int k = 0; k < 4; k++) wg::wgmma_f16_n128<0, 0>(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
            }
            wg::commit();
            wg::wait<0>();
            wg::reg_fence(s);
            if (lane == 0) mbar_arrive(&k_empty[st]);
            const int kbase = j * 128;
            if (kbase + 128 > p.kv_valid) {
                #pragma unroll
                for (int jj = 0; jj < 16; jj++) {
                    const int col = kbase + 8 * jj + 2 * (lane & 3);
                    if (col >= p.kv_valid) { s[4 * jj] = -INFINITY; s[4 * jj + 2] = -INFINITY; }
                    if (col + 1 >= p.kv_valid) { s[4 * jj + 1] = -INFINITY; s[4 * jj + 3] = -INFINITY; }
                }
            }
            float mx0 = -INFINITY, mx1 = -INFINITY;
            #pragma unroll
            for (int jj = 0; jj < 16; jj++) {
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
            for (int jj = 0; jj < 8; jj++) { o[4 * jj] *= al0; o[4 * jj + 1] *= al0; o[4 * jj + 2] *= al1; o[4 * jj + 3] *= al1; }
            const float mc0 = m0 * c, mc1 = m1 * c;
            // P = ex2(s c - m c) -> fp16 A fragments: k16 block kk of P is n8 blocks 2 kk, 2 kk + 1 of S
            uint32_t a[8][4];
            #pragma unroll
            for (int kk = 0; kk < 8; kk++) {
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
                const uint64_t dv = wg::desc_sw128(sv_u + (uint32_t)(st * kTile), 8192u);
                #pragma unroll
                for (int kk = 0; kk < 8; kk++) wg::wgmma_f16_rs_n64<1>(o, a[kk], dv + (uint64_t)(128 * kk), 1u);    // 16 keys = 2048 B
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
            __half* dst = p.o + ((size_t)batch * p.T + r + 8 * hh) * p.ldo + head * 64 + 2 * (lane & 3);
            #pragma unroll
            for (int jj = 0; jj < 8; jj++)
                *reinterpret_cast<__half2*>(dst + 8 * jj) = __floats2half2_rn(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
        }
    }
}

struct Maps { CUtensorMap q, k, v; };

// token matrices: x[(b * tokens + t) * ld + h * 64 + i]
inline int make_maps(Maps* m, const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv,
                     int B, int T, int Tk, int heads) {
    const uint32_t box[4] = {64, 128, 1, 1};
    auto one = [&](CUtensorMap* map, const __half* base, long long ld, int tokens) {
        const uint64_t dims[4] = {64, (uint64_t)tokens, (uint64_t)heads, (uint64_t)B};
        const uint64_t str[4] = {2, (uint64_t)ld * 2, 128, (uint64_t)tokens * (uint64_t)ld * 2};
        return make_map_f16(map, base, dims, str, box);
    };
    int r = one(&m->q, q, ldq, T);
    if (r) return r;
    r = one(&m->k, k, ldk, Tk);
    if (r) return r;
    return one(&m->v, v, ldv, Tk);
}

static inline int launch(const Maps& m, __half* o, long long ldo, int B, int T, int kv_valid, int heads, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        MI3D_CHECK(cudaFuncSetAttribute(k_flash_attn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        attr = true;
    }
    if (kv_valid < 1 || T < 1) return MI3D_ERR_ARG;
    Params p; p.T = T; p.kv_valid = kv_valid; p.ldo = (int)ldo; p.scale_log2e = 0.125f * 1.4426950408889634f; p.o = o;
    dim3 grid((unsigned)((T + 127) / 128), (unsigned)heads, (unsigned)B);
    k_flash_attn<<<grid, kThreads, kSmemBytes, st>>>(m.q, m.k, m.v, p);
    return (int)cudaGetLastError();
}

}  // namespace attn
