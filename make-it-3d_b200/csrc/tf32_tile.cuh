// tf32_tile.cuh -- helpers for hand-written wgmma tf32 tiles with a 3-term hi/lo split (fp32-class accuracy):
//   x = hi + lo (hi = tf32-rounded x):  A.B ~= A_hi.B_hi + A_lo.B_hi + A_hi.B_lo
// Storage convention for every operand tile: column blocks of [rows][32 fp32] (128-byte rows, 8-row / 1024-byte swizzle
// atoms, block stride = rows * 128 B), written by ordinary threads through sw_off().  tf32 wgmma reads both operands K-major:
// rows = M or N index, columns = K (descriptor: SBO = 1024 B, K advances by +32 B inside the row).
#pragma once
#include <cuda_runtime.h>
#include "tma.cuh"
#include "wgmma.cuh"

namespace ftc {

// byte offset of element (row, k) inside one [rows x 32 fp32] block (block base 1024-aligned)
__device__ __forceinline__ uint32_t sw_off(int row, int k) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 2) ^ (row & 7)) & 7) << 4) + ((k & 3) << 2));
}
__device__ __forceinline__ float tf32_hi(float x) {
    uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return __uint_as_float(r);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(tc::smem_u32(bar)) : "memory");
}
// D[64 x N] (+)= A[64 x K] . B[N x K]^T with the 3-term split (both operands K-major hi / lo column blocks, K % 32 == 0).
// a_hi .. b_lo: shared addresses of the first column block; *_blk: byte distance between column blocks.  Issue only: the caller
// commits and waits.  `acc` = 0: the first MMA overwrites D.
template <int N>
__device__ __forceinline__ void issue_3tf32(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t a_blk, uint32_t b_hi, uint32_t b_lo,
                                            uint32_t b_blk, int K, uint32_t acc) {
    #pragma unroll
    for (int k8 = 0; k8 < K / 8; k8++) {
        const uint32_t oa = (uint32_t)(k8 >> 2) * a_blk + (uint32_t)(k8 & 3) * 32u, ob = (uint32_t)(k8 >> 2) * b_blk + (uint32_t)(k8 & 3) * 32u;
        const uint64_t dah = wg::desc_sw128(a_hi + oa), dal = wg::desc_sw128(a_lo + oa);
        const uint64_t dbh = wg::desc_sw128(b_hi + ob), dbl = wg::desc_sw128(b_lo + ob);
        if constexpr (N == 16) { wg::wgmma_tf32_n16(d, dah, dbh, acc); wg::wgmma_tf32_n16(d, dal, dbh, 1u); wg::wgmma_tf32_n16(d, dah, dbl, 1u); }
        else if constexpr (N == 32) { wg::wgmma_tf32_n32(d, dah, dbh, acc); wg::wgmma_tf32_n32(d, dal, dbh, 1u); wg::wgmma_tf32_n32(d, dah, dbl, 1u); }
        else { wg::wgmma_tf32_n64(d, dah, dbh, acc); wg::wgmma_tf32_n64(d, dal, dbh, 1u); wg::wgmma_tf32_n64(d, dah, dbl, 1u); }
        acc = 1u;
    }
}

}  // namespace ftc

// ---------------------------------------------------------------------------------------------------------------------
// bf16 3-way split tiles (wgmma bf16): x = h + m + l (each bf16, together ~24 bits) -> fp32-class products,
// used by the fused field BACKWARD because 16-bit operands may be consumed MN-major (tf32 wgmma is K-major only;
// the MN-major operands are held element-wise to fp64 by the field backward's parity tests).
// Storage: [rows][64 bf16] = 128-byte rows, 8-row swizzle atoms; the same tile is read K-major (rows = M/N, +32 B per
// K = 16 step) or MN-major (rows = K, +2048 B per K = 16 step, LBO = distance to the next 64-column block).
// ---------------------------------------------------------------------------------------------------------------------
#include <cuda_bf16.h>
namespace fbf {
using ftc::mbar_arrive;

// byte offset of element (row, c) inside a [rows x 64 bf16] tile
__device__ __forceinline__ uint32_t sw_off16(int row, int c) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((c >> 3) ^ (row & 7)) & 7) << 4) + ((c & 7) << 1));
}
// 3-way split: x = h + m + l exactly to ~24 bits (fp32-class), each part bf16
__device__ __forceinline__ void split3(float x, __nv_bfloat16& h, __nv_bfloat16& m, __nv_bfloat16& l) {
    h = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(h);
    m = __float2bfloat16_rn(r1);
    l = __float2bfloat16_rn(r1 - __bfloat162float(m));
}
// Two values at a time: one packed conversion (F2FP.BF16.F32.PACK_AB, full-rate ALU) per part instead of two scalar F2F.BF16.F32, which
// issue at a quarter of that rate -- the chain kernel's owners convert 576 values per evaluation and were bound by that pipe.
// Same round-to-nearest-even as split3: bit-identical parts.  x0 lands in the low half (the lower column / K index).
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ void split3x2(float x0, float x1, uint32_t& h, uint32_t& m, uint32_t& l) {
    h = pack_bf16x2(x0, x1);
    const float r0 = x0 - __uint_as_float(h << 16), r1 = x1 - __uint_as_float(h & 0xffff0000u);
    m = pack_bf16x2(r0, r1);
    l = pack_bf16x2(r0 - __uint_as_float(m << 16), r1 - __uint_as_float(m & 0xffff0000u));
}
// pack 8 floats into one 16-byte chunk per part
__device__ __forceinline__ void split8(const float (&x)[8], uint4& ph, uint4& pm, uint4& pl) {
    uint32_t h[4], m[4], l[4];
    #pragma unroll
    for (int i = 0; i < 4; i++) split3x2(x[2 * i], x[2 * i + 1], h[i], m[i], l[i]);
    ph = make_uint4(h[0], h[1], h[2], h[3]); pm = make_uint4(m[0], m[1], m[2], m[3]); pl = make_uint4(l[0], l[1], l[2], l[3]);
}
// one operand: three part tiles laid out back to back (h, m, l at +0, +part_stride, +2 part_stride); lbo: MN-major distance between
// 64-column blocks
struct Operand { uint32_t base; uint32_t part_stride; uint32_t lbo; };

// D[64 x N] (+)= A . B over K elements (K % 16 == 0; K-major operands: K <= 64).  TA / TB = 1: operand is MN-major.  Six MMAs per
// K = 16 step keep every product term down to 2^-16 of the leading one: hh, hm, mh, hl, lh, mm  -> fp32-class accuracy.
// Issue only: the caller commits and waits.
template <int N, int TA, int TB>
__device__ __forceinline__ void issue_bf16x3(float (&d)[N / 2], const Operand& A, const Operand& B, int K, uint32_t acc) {
    const uint64_t a0 = wg::desc_sw128(A.base, TA ? A.lbo : 16u), b0 = wg::desc_sw128(B.base, TB ? B.lbo : 16u);
    #pragma unroll
    for (int k16 = 0; k16 < K / 16; k16++) {
        const uint32_t oa = (TA ? (uint32_t)k16 * 2048u : (uint32_t)k16 * 32u) >> 4;
        const uint32_t ob = (TB ? (uint32_t)k16 * 2048u : (uint32_t)k16 * 32u) >> 4;
        uint64_t da[3], db[3];
        #pragma unroll
        for (int q = 0; q < 3; q++) { da[q] = a0 + oa + q * (A.part_stride >> 4); db[q] = b0 + ob + q * (B.part_stride >> 4); }
        auto mma = [&](uint64_t x, uint64_t y, uint32_t s) {
            if constexpr (N == 32) wg::wgmma_bf16_n32<TA, TB>(d, x, y, s); else wg::wgmma_bf16_n64<TA, TB>(d, x, y, s);
        };
        mma(da[0], db[0], acc); acc = 1u;
        mma(da[0], db[1], 1u);
        mma(da[1], db[0], 1u);
        mma(da[0], db[2], 1u);
        mma(da[2], db[0], 1u);
        mma(da[1], db[1], 1u);
    }
}
}  // namespace fbf
