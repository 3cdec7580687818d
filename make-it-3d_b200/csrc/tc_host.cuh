// tc_host.cuh -- host side of the tensor-core tile kernel: TMA descriptor encoding + launch
#pragma once
#include "tc_gemm.cuh"
#include "mi3d_common.cuh"
#include <cudaTypedefs.h>

namespace tc {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// libcuda is not linked (the .so must load on a CPU-only box); the entry point is fetched through the runtime.
inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// fp16 tensor, up to 4 dims (dim 0 innermost/contiguous), 128B swizzle, zero OOB fill.
// dims[i] extents, strides_bytes[i] for i >= 1, box[i] box extents (box[0] must be 64).
inline int make_map_f16(CUtensorMap* map, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[4], const uint32_t box[4]) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return MI3D_ERR_ARG;
    cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
    cuuint64_t gstr[3] = {strides_bytes[1], strides_bytes[2], strides_bytes[3]};
    cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? MI3D_OK : 2000000 + (int)r;
}

// Plain K-major matrix [rows][K] (optionally batched: z1 x z2 with element strides sz1, sz2), row stride ld (elements).
inline int make_map_matrix(CUtensorMap* map, const __half* base, uint64_t K, uint64_t rows, uint64_t ld, uint32_t box_rows,
                           uint64_t z1 = 1, uint64_t sz1 = 0, uint64_t z2 = 1, uint64_t sz2 = 0) {
    const uint64_t dims[4] = {K, rows, z1, z2};
    const uint64_t str[4] = {2, ld * 2, (sz1 ? sz1 : ld * rows) * 2, (sz2 ? sz2 : (sz1 ? sz1 : ld * rows) * z1) * 2};
    const uint32_t box[4] = {BLOCK_K, box_rows, 1, 1};
    return make_map_f16(map, base, dims, str, box);
}

// NHWC activation for the implicit 3x3 conv: dims (C, W, H, N), box (64, bw, bh, bn) with bw*bh*bn = 128
inline int make_map_nhwc(CUtensorMap* map, const __half* base, int C, int W, int H, int N, int bw, int bh, int bn) {
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    const uint64_t str[4] = {2, (uint64_t)C * 2, (uint64_t)C * W * 2, (uint64_t)C * W * H * 2};
    const uint32_t box[4] = {BLOCK_K, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
    return make_map_f16(map, base, dims, str, box);
}

// Only the plain kernel has a 160-wide instantiation (launch() below): epilogues PLAIN, GEGLU, TRANSPOSED, conv 0 or 1.
inline bool has_block_n_160(int epi_mode, int conv) { return conv != 2 && (epi_mode == EPI_PLAIN || epi_mode == EPI_GEGLU || epi_mode == EPI_TRANSPOSED); }

inline int pick_block_n(int N, long long m_tiles_times_batch, int num_sms, bool allow_160 = true) {
    // largest tile that divides N; prefer 256 only when the grid still fills the machine
    if (N % 256 == 0 && m_tiles_times_batch * (N / 256) >= num_sms) return 256;
    if (N % 128 == 0 && m_tiles_times_batch * (N / 128) >= num_sms) return 128;
    if (allow_160 && N % 160 == 0 && N % 128 != 0 && m_tiles_times_batch * (N / 160) >= num_sms / 2) return 160;   // N = 320: 2.5x the MACs per operand byte of BN = 64
    if (N % 64 == 0) return 64;
    return 0;
}

template <int BN, bool kQuickGelu = false, bool kVgg = false, bool kGelu = false>
inline int launch_bn(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, int batch, cudaStream_t st) {
    static bool attr = false;
    auto kernel = [] {
        if constexpr (kVgg) return k_tc_gemm_vgg<BN>;
        else if constexpr (kGelu) return k_tc_gemm_gelu<BN>;
        else return k_tc_gemm<BN, kQuickGelu>;
    }();
    if (!attr) {
        MI3D_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<BN>::kSmemBytes));
        attr = true;
    }
    GemmParams q = p;
    q.m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M; q.n_tiles = p.N / BN;
    if (q.splits <= 1) { q.splits = 1; q.kb_per_split = q.num_k_blocks; }
    q.num_tiles = q.m_tiles * q.n_tiles * batch * q.splits;
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    const int resident = (Cfg<BN>::kSmemBytes <= 110 * 1024) ? 2 : 1;       // persistent grid: one (or two) CTAs per SM loop over the tiles
    const int grid = q.num_tiles < sms * resident ? q.num_tiles : sms * resident;
    kernel<<<grid, kThreads, Cfg<BN>::kSmemBytes, st>>>(ma, mb, q);
    return (int)cudaGetLastError();
}

inline int launch(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, int block_n, int batch, cudaStream_t st) {
    if (p.K % BLOCK_K || p.N % block_n || p.out_z1 < 1) return MI3D_ERR_ARG;
    if (((uintptr_t)p.bias | (uintptr_t)p.row_bias | (uintptr_t)p.splitk_ws) & 15) return MI3D_ERR_ARG;     // read / RED-added 16 bytes at a time
    if (p.conv == 2 || p.epi_mode == EPI_RELU || p.epi_mode == EPI_RELU_BWD) {
        if (p.splits > 1 || (p.epi_mode == EPI_RELU_BWD && !p.aux)) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, false, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, false, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, false, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    if (p.epi_mode == EPI_QUICKGELU || p.epi_mode == EPI_QUICKGELU_BWD) {
        if (p.splits > 1) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    if (p.epi_mode == EPI_GELU) {
        if (p.splits > 1 || p.conv || !p.out) return MI3D_ERR_ARG;
        switch (block_n) {
            case 64: return launch_bn<64, false, false, true>(ma, mb, p, batch, st);
            case 128: return launch_bn<128, false, false, true>(ma, mb, p, batch, st);
            case 256: return launch_bn<256, false, false, true>(ma, mb, p, batch, st);
        }
        return MI3D_ERR_ARG;
    }
    switch (block_n) {
        case 64: return launch_bn<64>(ma, mb, p, batch, st);
        case 128: return launch_bn<128>(ma, mb, p, batch, st);
        case 160: return launch_bn<160>(ma, mb, p, batch, st);
        case 256: return launch_bn<256>(ma, mb, p, batch, st);
    }
    return MI3D_ERR_ARG;
}

// Split-K for the deep U-Net / VAE levels (M = 128 .. 512 rows): a handful of output tiles with K = 3 000 .. 23 000 would otherwise
// run on a handful of SMs.  ws: fp32 [M][N] scratch (zeroed here).  Only plain fp16-output GEMMs / convs with batch == 1.
inline int plan_splits(long long tiles, int num_k_blocks, int num_sms) {
    if (tiles * 2 > num_sms || num_k_blocks < 48) return 1;      // the zero-fill + finish passes are two more launches: only deep K pays
    int s = (int)(num_sms / tiles);
    if (s > 8) s = 8;
    while (s > 1 && num_k_blocks / s < 8) s--;
    return s;
}
inline int launch_splitk(const CUtensorMap& ma, const CUtensorMap& mb, GemmParams p, int block_n, int splits, float* ws, cudaStream_t st) {
    p.kb_per_split = (p.num_k_blocks + splits - 1) / splits;
    p.splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;          // every K-range non-empty
    p.splitk_ws = ws;
    MI3D_CHECK(cudaMemsetAsync(ws, 0, (size_t)p.M * p.N * sizeof(float), st));
    int r = launch(ma, mb, p, block_n, 1, st);
    if (r) return r;
    p.splits = 1;
    const size_t total = (size_t)p.m_valid * p.N / 8;
    k_splitk_finish<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ws, p);
    return (int)cudaGetLastError();
}

}  // namespace tc
