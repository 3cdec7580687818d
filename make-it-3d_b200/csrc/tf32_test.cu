// tf32_test.cu -- C-ABI unit-test entry for the hand-written wgmma tf32 tiles used by the fused field forward kernel:
// validates the thread-written 128B-swizzle layout, the 3-term split accuracy and the K-major operand descriptors.
#include "tf32_tile.cuh"
#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

// stage X [R x C] (fp32 row-major, global) into hi/lo column blocks of [R x 32]
__device__ void stage(const float* __restrict__ X, int R, int C, uint8_t* hi, uint8_t* lo, int tid, int nthreads) {
    for (int i = tid; i < R * C; i += nthreads) {
        const int r = i / C, c = i % C;
        const float v = X[i], h = ftc::tf32_hi(v);
        const uint32_t o = (uint32_t)(c >> 5) * (uint32_t)R * 128u + ftc::sw_off(r, c & 31);
        *reinterpret_cast<float*>(hi + o) = h; *reinterpret_cast<float*>(lo + o) = v - h;
    }
}

// D = A[128 x K] . B[N x K]^T, both K-major; one warpgroup, two m64 halves
template <int N>
__global__ void __launch_bounds__(128, 1) k_tf32_tile_test(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ D, int K) {
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* sm = smem_dyn + ((1024u - (tc::smem_u32(smem_dyn) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS / LDS, not generic ST / LD)
    const uint32_t a_bytes = 128u * (uint32_t)K * 4u, b_bytes = (uint32_t)N * (uint32_t)K * 4u;
    uint8_t *a_hi = sm, *a_lo = sm + a_bytes, *b_hi = sm + 2 * a_bytes, *b_lo = sm + 2 * a_bytes + b_bytes;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    stage(A, 128, K, a_hi, a_lo, tid, blockDim.x);
    stage(B, N, K, b_hi, b_lo, tid, blockDim.x);
    tc::fence_proxy_async();                 // tiles were written through the generic proxy, wgmma reads through the async proxy
    __syncthreads();
    float d[2][N / 2];
    wg::fence();
    #pragma unroll
    for (int h = 0; h < 2; h++)
        ftc::issue_3tf32<N>(d[h], tc::smem_u32(a_hi) + 8192u * h, tc::smem_u32(a_lo) + 8192u * h, 128u * 128u,
                            tc::smem_u32(b_hi), tc::smem_u32(b_lo), (uint32_t)N * 128u, K, 0u);
    wg::commit();
    wg::wait<0>();
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        wg::reg_fence(d[h]);
        #pragma unroll
        for (int j = 0; j < N / 8; j++)
            #pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                const int row = 64 * h + 16 * warp + (lane >> 2) + 8 * hh, col = 8 * j + 2 * (lane & 3);
                D[(size_t)row * N + col] = d[h][4 * j + 2 * hh];
                D[(size_t)row * N + col + 1] = d[h][4 * j + 2 * hh + 1];
            }
    }
}

}  // namespace

extern "C" int mi3d_tf32_tile_test(const float* a, const float* b, float* d, int N, int K, int mode, mi3d_stream_t stream) {
    if ((N != 16 && N != 32 && N != 64) || K % 32 || K > 128 || K < 32 || mode != 0) return MI3D_ERR_ARG;
    const size_t smem = 1024 + 2 * (size_t)128 * K * 4 + 2 * (size_t)N * K * 4;
    const cudaStream_t st = (cudaStream_t)stream;
    if (N == 16) {
        MI3D_CHECK(cudaFuncSetAttribute(k_tf32_tile_test<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_tf32_tile_test<16><<<1, 128, smem, st>>>(a, b, d, K);
    } else if (N == 32) {
        MI3D_CHECK(cudaFuncSetAttribute(k_tf32_tile_test<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_tf32_tile_test<32><<<1, 128, smem, st>>>(a, b, d, K);
    } else {
        MI3D_CHECK(cudaFuncSetAttribute(k_tf32_tile_test<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_tf32_tile_test<64><<<1, 128, smem, st>>>(a, b, d, K);
    }
    MI3D_RETURN_LAUNCH();
}
