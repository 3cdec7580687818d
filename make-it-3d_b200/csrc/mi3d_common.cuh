// mi3d_common.cuh -- shared helpers for the sm_90a kernels behind include/mi3d.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <float.h>

#define MI3D_OK 0
#define MI3D_ERR_ARG 1000001

// Launch-error check only (never synchronises): the C ABI reports bad launches, the caller
// (a torch.autograd.Function) raises.  Asynchronous faults surface at the caller's next sync.
#define MI3D_RETURN_LAUNCH()                      \
    do {                                          \
        cudaError_t e__ = cudaGetLastError();     \
        return e__ == cudaSuccess ? MI3D_OK : (int)e__; \
    } while (0)

#define MI3D_CHECK(call)                          \
    do {                                          \
        cudaError_t e__ = (call);                 \
        if (e__ != cudaSuccess) return (int)e__;  \
    } while (0)

static inline __host__ __device__ uint32_t mi3d_ceil_div(uint32_t a, uint32_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float mi3d_clampf(float v, float lo, float hi) { return fminf(hi, fmaxf(lo, v)); }

// 10-bit-per-axis Morton code (same bit layout as the reference's density grid so that
// checkpoints' density_grid / density_bitfield stay interchangeable: raymarching.cu:56-81).
__host__ __device__ __forceinline__ uint32_t mi3d_spread3(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__host__ __device__ __forceinline__ uint32_t mi3d_morton(uint32_t x, uint32_t y, uint32_t z) {
    return mi3d_spread3(x) | (mi3d_spread3(y) << 1) | (mi3d_spread3(z) << 2);
}
__host__ __device__ __forceinline__ uint32_t mi3d_compact3(uint32_t x) {
    x &= 0x49249249u;
    x = (x | (x >> 2)) & 0xc30c30c3u;
    x = (x | (x >> 4)) & 0x0f00f00fu;
    x = (x | (x >> 8)) & 0xff0000ffu;
    x = (x | (x >> 16)) & 0x0000ffffu;
    return x;
}

// Philox4x32-10 counter RNG (in-kernel noise: march jitter, smooth-loss perturbation, density-grid jitter)
__device__ __forceinline__ uint4 mi3d_philox(uint4 ctr, uint2 key) {
    #pragma unroll
    for (int r = 0; r < 10; r++) {
        uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
        uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += 0x9E3779B9u; key.y += 0xBB67AE85u;
    }
    return ctr;
}
__device__ __forceinline__ float mi3d_u01(uint32_t v) { return (float)(v >> 8) * (1.0f / 16777216.0f); }   // [0,1)
