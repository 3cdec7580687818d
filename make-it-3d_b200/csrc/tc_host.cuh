// tc_host.cuh -- host side of the tensor-core tile kernel (tc_gemm.cuh) and the fused attention (attn.cuh): their parameter types,
// TMA descriptor encoding and tile planning.  Includable anywhere: the kernels and their launchers are compiled once, in plan.cu.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "mi3d_common.cuh"
#include <cudaTypedefs.h>

namespace tc {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 fp16 = 128 B = one swizzle-128B atom row

// EPI_QUICKGELU: out = y * sigmoid(1.702 y) (CLIP's MLP activation), y = alpha * acc + bias; the pre-activation y is also stored to aux
//                when aux is set (the input-gradient pass needs it).
// EPI_QUICKGELU_BWD: out = y * QuickGELU'(aux), aux = the saved pre-activation (same layout as out).
// EPI_RELU: out = max(y, 0) (VGG's convs).  EPI_RELU_BWD: out = y * (aux > 0), aux = the saved post-ReLU input of the conv whose
//                input gradient this is (same layout as out).  Both only in k_tc_gemm_vgg.
// EPI_GELU: out = 0.5 y (1 + erf(y / sqrt 2)) (exact GELU, the SD-2 text encoder's MLP activation), y = alpha * acc + bias, in fp32,
//                stored fp16.  Forward only; only in k_tc_gemm_gelu.
enum EpiMode : int { EPI_PLAIN = 0, EPI_GEGLU = 1, EPI_TRANSPOSED = 2, EPI_QUICKGELU = 3, EPI_QUICKGELU_BWD = 4, EPI_RELU = 5, EPI_RELU_BWD = 6,
                     EPI_GELU = 7 };

struct GemmParams {
    int M, N, K;                 // per-batch extents; N multiple of BLOCK_N, K multiple of 64, M multiple of 128 (rows may be padded)
    int num_k_blocks;
    int conv;                    // 0 plain, 1 implicit 3x3 conv, 2 implicit 3x3 conv over spatial blocks (k_tc_gemm_vgg)
    int conv_H, conv_W, conv_bw, conv_bh, cin_blocks;
    int a_z1, b_z1;              // batch decomposition of blockIdx.z for A and B maps; b_batched = 0 -> weights shared
    int b_batched;
    // epilogue
    __half* out;                 // fp16 output or nullptr
    float* out_f32;              // fp32 output or nullptr
    long long ldc;               // row stride (elements) of out
    int out_z1;                  // blockIdx.z -> out offset (z % out_z1) * out_s_lo + (z / out_z1) * out_s_hi (elements)
    long long out_s_lo, out_s_hi;
    const float* bias;           // [N] fp32 or nullptr
    const float* row_bias;       // [M / rows_per_group][N] fp32 (time-embedding term) or nullptr
    int rows_per_group;
    const __half* residual;      // same layout as out, or nullptr
    long long ld_res;
    int epi_mode;
    float alpha;                 // scales the accumulator before bias
    int m_valid;                 // rows >= m_valid (per batch) are not stored
    int splits, kb_per_split;     // split-K: work item t -> (t % splits) K-range, partial sums RED-added (fp32) into splitk_ws[M][N]
    float* splitk_ws;
    int m_tiles, n_tiles, num_tiles;   // persistent tile loop: tile t -> n_blk = t % n_tiles, m_blk = (t / n_tiles) % m_tiles, z = t / (n_tiles * m_tiles)
    __half* aux;                 // QuickGELU modes: pre-activation, same layout as out; EPI_RELU_BWD: the ReLU mask source
};

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

// Only the plain kernel has a 160-wide instantiation (tc::launch in plan.cu): epilogues PLAIN, GEGLU, TRANSPOSED, conv 0 or 1.
inline bool has_block_n_160(int epi_mode, int conv) { return conv != 2 && (epi_mode == EPI_PLAIN || epi_mode == EPI_GEGLU || epi_mode == EPI_TRANSPOSED); }

inline int pick_block_n(int N, long long m_tiles_times_batch, int num_sms, bool allow_160 = true) {
    // largest tile that divides N; prefer 256 only when the grid still fills the machine
    if (N % 256 == 0 && m_tiles_times_batch * (N / 256) >= num_sms) return 256;
    if (N % 128 == 0 && m_tiles_times_batch * (N / 128) >= num_sms) return 128;
    if (allow_160 && N % 160 == 0 && N % 128 != 0 && m_tiles_times_batch * (N / 160) >= num_sms / 2) return 160;   // N = 320: 2.5x the MACs per operand byte of BN = 64
    if (N % 64 == 0) return 64;
    return 0;
}

// Split-K for the deep U-Net / VAE levels (M = 128 .. 512 rows): a handful of output tiles with K = 3 000 .. 23 000 would otherwise
// run on a handful of SMs.  Only plain fp16-output GEMMs / convs with batch == 1.
inline int plan_splits(long long tiles, int num_k_blocks, int num_sms) {
    if (tiles * 2 > num_sms || num_k_blocks < 48) return 1;      // the zero-fill + finish passes are two more launches: only deep K pays
    int s = (int)(num_sms / tiles);
    if (s > 8) s = 8;
    while (s > 1 && num_k_blocks / s < 8) s--;
    return s;
}

}  // namespace tc

// The fused attention's Q / K / V maps; head_dim d: 40, 64, 80 or 160.
namespace attn {

inline bool supported(int d) { return d == 40 || d == 64 || d == 80 || d == 160; }

struct Maps { CUtensorMap q, k, v; int d = 64; };

// token matrices: x[(b * tokens + t) * ld + h * d + i]; every ld and the head stride 2 d bytes are multiples of 16 bytes
inline int make_maps(Maps* m, const __half* q, long long ldq, const __half* k, long long ldk, const __half* v, long long ldv,
                     int B, int T, int Tk, int heads, int d) {
    if (!supported(d)) return MI3D_ERR_ARG;
    m->d = d;
    const uint32_t kv_rows = d > 128 ? 64 : 128;          // Shape<d>::kKeys
    auto one = [&](CUtensorMap* map, const __half* base, long long ld, int tokens, uint32_t rows) {
        const uint64_t dims[4] = {(uint64_t)d, (uint64_t)tokens, (uint64_t)heads, (uint64_t)B};
        const uint64_t str[4] = {2, (uint64_t)ld * 2, (uint64_t)d * 2, (uint64_t)tokens * (uint64_t)ld * 2};
        const uint32_t box[4] = {64, rows, 1, 1};
        return tc::make_map_f16(map, base, dims, str, box);
    };
    int r = one(&m->q, q, ldq, T, 128);
    if (r) return r;
    r = one(&m->k, k, ldk, Tk, kv_rows);
    if (r) return r;
    return one(&m->v, v, ldv, Tk, kv_rows);
}

}  // namespace attn
