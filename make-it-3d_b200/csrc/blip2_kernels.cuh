// blip2_kernels.cuh -- the kernels of the BLIP-2 captioner (blip2_engine.cu) that the tile GEMM and the shared memory-bound kernels
// do not cover: the weight-streaming GEMM for <= 64 activation rows (OPT's decoder linears and lm_head), attention for any head_dim
// (EVA's 88, OPT's 80, the Q-Former's 64; causal or not), the 14x14 patch gather, the decoder's token / query embedding and the
// device-side greedy step.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2k {
namespace {   // internal linkage, as the other engines' kernel headers

// ------------------------------------------------------------------------------------------------------------
// Weight-streaming GEMM: part[s][m][n] = sum over k in split s of X[m][k] W[n][k], m < M <= 64.
//
// At <= 64 rows a linear is a read of its weight matrix, so the grid is cut over N (128 weight rows per CTA, 16 per warp) AND over K
// (`kc` columns per split) until every SM streams weights.  Each warp keeps its next 256 K-columns of weights in flight in registers
// (16 x 16 B per thread) while the CTA stages the matching [64 x 256] slice of X in shared memory; the products run on mma.sync
// m16n8k16 with W as the A operand (16 weight rows) and X as B (8 activation rows per n8 tile).  K is permuted inside every 32-column
// step so that one 16-byte load of W or X feeds two k16 MMAs (thread t owns columns 8t..8t+7 of the step; the same permutation on
// both operands leaves the sum unchanged).  The partial sums of the splits go to `part` and k_stream_reduce adds them in split order:
// no atomics, so the output is bit-identical from call to call.
// ------------------------------------------------------------------------------------------------------------
constexpr int kStreamRows = 128;          // weight rows per CTA
constexpr int kStreamChunk = 256;         // K-columns per staged X slice
constexpr int kStreamXLd = kStreamChunk + 32;   // 576-byte rows: the 8 lanes of an LDS.128 phase hit 32 distinct banks

__device__ __forceinline__ uint4 ldg_stream(const __half* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(256, 2)
k_stream_gemm(const __half* __restrict__ X, long long ldx, int M, const __half* __restrict__ W, int N, int K, int kc, float* __restrict__ part) {
    __shared__ __align__(16) __half xs[64 * kStreamXLd];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int n0 = blockIdx.x * kStreamRows + warp * 16;
    const int r0 = min(n0 + g, N - 1), r1 = min(n0 + g + 8, N - 1);      // rows past N load a valid row and are never stored
    const __half* w0 = W + (size_t)r0 * K + 8 * t;
    const __half* w1 = W + (size_t)r1 * K + 8 * t;
    const int k_begin = blockIdx.y * kc, k_end = min(K, k_begin + kc);
    float acc[8][4];
    #pragma unroll
    for (int j = 0; j < 8; j++) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
    for (int kb = k_begin; kb < k_end; kb += kStreamChunk) {
        const int len = min(kStreamChunk, k_end - kb);
        uint4 wa[8], wb[8];
        #pragma unroll
        for (int s = 0; s < 8; s++) {
            if (32 * s < len) { wa[s] = ldg_stream(w0 + kb + 32 * s); wb[s] = ldg_stream(w1 + kb + 32 * s); }
        }
        __syncthreads();                                  // the previous slice's readers are done
        #pragma unroll
        for (int i = 0; i < 8; i++) {
            const int idx = tid + 256 * i, m = idx >> 5, c = (idx & 31) * 8;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (m < M && c < len) v = *reinterpret_cast<const uint4*>(X + (size_t)m * ldx + kb + c);
            *reinterpret_cast<uint4*>(xs + m * kStreamXLd + c) = v;
        }
        __syncthreads();
        #pragma unroll
        for (int s = 0; s < 8; s++) {
            if (32 * s < len) {
                #pragma unroll
                for (int j = 0; j < 8; j++) {
                    const uint4 xv = *reinterpret_cast<const uint4*>(xs + (8 * j + g) * kStreamXLd + 32 * s + 8 * t);
                    mma16816(acc[j], wa[s].x, wb[s].x, wa[s].y, wb[s].y, xv.x, xv.y);
                    mma16816(acc[j], wa[s].z, wb[s].z, wa[s].w, wb[s].w, xv.z, xv.w);
                }
            }
        }
    }
    // acc[j]: (weight row g, activation rows 8j + 2t, +1), (weight row g + 8, the same activation rows)
    float* ps = part + (size_t)blockIdx.y * M * N;
    #pragma unroll
    for (int j = 0; j < 8; j++) {
        #pragma unroll
        for (int e = 0; e < 4; e++) {
            const int m = 8 * j + 2 * t + (e & 1), n = n0 + g + ((e & 2) ? 8 : 0);
            if (m < M && n < N) ps[(size_t)m * N + n] = acc[j][e];
        }
    }
}

// out[m][n] = act(sum_s part[s][m][n] + bias[n] (+ residual[m][n])), the splits added in order 0..S-1; act: 0 none, 1 ReLU.
// fp16 out (ldo) or fp32 out32 (ldo).  One thread per output element.
__global__ void k_stream_reduce(const float* __restrict__ part, int S, int M, int N, const float* __restrict__ bias, const __half* __restrict__ residual,
                                long long ld_res, int act, __half* __restrict__ out, float* __restrict__ out32, long long ldo) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    const int m = (int)(i / N), n = (int)(i % N);
    float v = 0.f;
    for (int s = 0; s < S; s++) v += part[(size_t)s * M * N + i];
    if (bias) v += bias[n];
    if (residual) v += __half2float(residual[(size_t)m * ld_res + n]);
    if (act == 1) v = fmaxf(v, 0.f);
    if (out32) out32[(size_t)m * ldo + n] = v;
    else out[(size_t)m * ldo + n] = __float2half_rn(v);
}

// ------------------------------------------------------------------------------------------------------------
// Attention for head_dim d (d % 8 == 0, d <= 128): o[b*T + i, h*d + c] = sum_j softmax_j(scale q_i . k_j) v_j[c] over the first
// kv_valid keys (causal: j <= i as well).  One warp per query row, 8 rows of one head per CTA; scores and statistics in fp32, the
// reductions in a fixed order (bit-identical run to run).  Query rows >= T are not written.
// ------------------------------------------------------------------------------------------------------------
constexpr int kAttnMaxKeys = 512;

__global__ void __launch_bounds__(256)
k_attn_rows(const __half* __restrict__ q, long long ldq, const __half* __restrict__ k, long long ldk, const __half* __restrict__ v, long long ldv,
            __half* __restrict__ o, long long ldo, int T, int Tk, int kv_valid, int d, float scale, int causal) {
    __shared__ float sp[8][kAttnMaxKeys];
    __shared__ __align__(16) __half sq[8][128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * 8 + warp, h = blockIdx.y, b = blockIdx.z;
    if (i >= T) return;
    const __half* qr = q + ((size_t)b * T + i) * ldq + (size_t)h * d;
    for (int c = lane * 8; c < d; c += 256) *reinterpret_cast<uint4*>(&sq[warp][c]) = *reinterpret_cast<const uint4*>(qr + c);
    __syncwarp();
    const int nk = causal ? min(i + 1, kv_valid) : kv_valid;
    const __half* kb = k + (size_t)b * Tk * ldk + (size_t)h * d;
    const __half* vb = v + (size_t)b * Tk * ldv + (size_t)h * d;
    float mx = -INFINITY;
    for (int j = lane; j < nk; j += 32) {
        const __half* kr = kb + (size_t)j * ldk;
        float s = 0.f;
        for (int c = 0; c < d; c += 8) {
            const uint4 kv4 = *reinterpret_cast<const uint4*>(kr + c);
            const uint4 qv4 = *reinterpret_cast<const uint4*>(&sq[warp][c]);
            const __half2* kh = reinterpret_cast<const __half2*>(&kv4);
            const __half2* qh = reinterpret_cast<const __half2*>(&qv4);
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const float2 a = __half22float2(kh[e]), bq = __half22float2(qh[e]);
                s = fmaf(a.x, bq.x, s); s = fmaf(a.y, bq.y, s);
            }
        }
        s *= scale;
        sp[warp][j] = s;
        mx = fmaxf(mx, s);
    }
    #pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.f;
    for (int j = lane; j < nk; j += 32) { const float e = __expf(sp[warp][j] - mx); sp[warp][j] = e; sum += e; }
    #pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    __syncwarp();
    const float inv = 1.f / sum;
    __half* orow = o + ((size_t)b * T + i) * ldo + (size_t)h * d;
    for (int c = 2 * lane; c < d; c += 64) {
        float a0 = 0.f, a1 = 0.f;
        for (int j = 0; j < nk; j++) {
            const float p = sp[warp][j];
            const float2 vv = __half22float2(*reinterpret_cast<const __half2*>(vb + (size_t)j * ldv + c));
            a0 = fmaf(p, vv.x, a0); a1 = fmaf(p, vv.y, a1);
        }
        *reinterpret_cast<__half2*>(orow + c) = __floats2half2_rn(a0 * inv, a1 * inv);
    }
}

// ------------------------------------------------------------------------------------------------------------
// EVA patch embedding: pixel_values fp32 [1,3,S,S] -> col fp16 [np][Kpad], col[p][c*P*P + ky*P + kx] (the conv weight's flattening),
// columns >= 3 P P zero.  The patch GEMM then runs on the tile kernel.
// ------------------------------------------------------------------------------------------------------------
__global__ void k_patch_cols(const float* __restrict__ img, int S, int P, int Kpad, __half* __restrict__ col) {
    const int g = S / P, np = g * g, K = 3 * P * P;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)np * Kpad; i += (size_t)gridDim.x * blockDim.x) {
        const int p = (int)(i / Kpad), kk = (int)(i % Kpad);
        float v = 0.f;
        if (kk < K) {
            const int c = kk / (P * P), r = kk % (P * P), ky = r / P, kx = r % P, py = p / g, px = p % g;
            v = img[((size_t)c * S + py * P + ky) * S + px * P + kx];
        }
        col[i] = __float2half_rn(v);
    }
}

// x[0] = cls + pos[0]; x[1 + p] = patch[p] + pos[1 + p] (fp32 sums, one rounding)
__global__ void k_vision_embed(const __half* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, __half* __restrict__ x,
                               int np, int C) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)(np + 1) * C; i += (size_t)gridDim.x * blockDim.x) {
        const int t = (int)(i / C), c = (int)(i % C);
        const float base = t == 0 ? cls[c] : __half2float(patch[(size_t)(t - 1) * C + c]);
        x[i] = __float2half_rn(base + pos[i]);
    }
}

// ------------------------------------------------------------------------------------------------------------
// OPT decoder input over the fixed row window: x[t] = (t < nq ? proj[t] : tok_emb[ids[t]]) + pos_emb[t + 2], t < rows.
// ------------------------------------------------------------------------------------------------------------
__global__ void k_decoder_embed(const long long* __restrict__ ids, const __half* __restrict__ proj, const __half* __restrict__ tok,
                                const __half* __restrict__ pos, __half* __restrict__ x, int rows, int nq, int C, int V) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)rows * C; i += (size_t)gridDim.x * blockDim.x) {
        const int t = (int)(i / C), c = (int)(i % C);
        float e;
        if (t < nq) e = __half2float(proj[(size_t)t * C + c]);
        else { long long id = ids[t]; id = id < 0 ? 0 : (id >= V ? V - 1 : id); e = __half2float(tok[(size_t)id * C + c]); }
        x[i] = __float2half_rn(e + __half2float(pos[(size_t)(t + 2) * C + c]));
    }
}

// Decoder state on the device: st[0] = rows filled (prompt + generated), st[1] = tokens generated, st[2] = stopped (eos seen),
// st[3] = steps run.
// The prompt: ids = [image_token] x nq + [bos], st = {nq + 1, 0, 0, 0}.
__global__ void k_decoder_start(long long* __restrict__ ids, int* __restrict__ st, int rows, int nq, long long image_token, long long bos) {
    for (int t = threadIdx.x; t < rows; t += blockDim.x) ids[t] = t < nq ? image_token : bos;
    if (threadIdx.x == 0) { st[0] = nq + 1; st[1] = 0; st[2] = 0; st[3] = 0; }
}

// y[0] = x[st[0] - 1]: the last filled row, the only one lm_head reads
__global__ void k_last_row(const __half* __restrict__ x, const int* __restrict__ st, __half* __restrict__ y, int C) {
    const __half* src = x + (size_t)(st[0] - 1) * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) y[c] = src[c];
}

// Greedy step, one CTA: the argmax of logits[0..V) (the lowest index among equal maxima, torch.argmax's rule; the padding rows of the
// vocab are never read), appended at row st[0] unless the decode has stopped.  *use_forced != 0: forced[st[3]] is appended instead
// (teacher forcing).  The step's logits are copied to all_logits[st[3]][V].  *eos < 0: no early stop.
__global__ void __launch_bounds__(1024) k_greedy_pick(const float* __restrict__ logits, int V, long long* __restrict__ ids, int* __restrict__ st,
                                                      const long long* __restrict__ eos_p, const long long* __restrict__ forced_p,
                                                      const int* __restrict__ use_forced, float* __restrict__ all_logits) {
    const long long eos = *eos_p;
    const long long* forced = *use_forced ? forced_p : nullptr;
    __shared__ float sv[32]; __shared__ int si[32];
    const int step = st[3];
    float best = -INFINITY; int bi = 0x7fffffff;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const float x = logits[v];
        all_logits[(size_t)step * V + v] = x;
        if (x > best) { best = x; bi = v; }               // v increases along a thread's sweep: the first maximum is kept
    }
    #pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off); const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); w++)
            if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
        if (bi == 0x7fffffff) bi = 0;                     // all logits NaN: no maximum, token 0
        const long long tok = forced ? forced[step] : (long long)bi;
        if (!st[2]) {
            ids[st[0]] = tok;
            st[0] += 1; st[1] += 1;
            if (eos >= 0 && tok == eos) st[2] = 1;
        }
        st[3] = step + 1;
    }
}

// fp16 -> fp32 copy of a tap
__global__ void k_f16_to_f32(const __half* __restrict__ src, float* __restrict__ dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = __half2float(src[i]);
}

// fp32 [N][K] -> fp16 [N][Kpad], columns >= K zero (the patch conv's weight, K = 3 P P)
__global__ void k_f32_to_f16_padk(const float* __restrict__ src, __half* __restrict__ dst, int N, int K, int Kpad) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)N * Kpad; i += (size_t)gridDim.x * blockDim.x) {
        const int n = (int)(i / Kpad), k = (int)(i % Kpad);
        dst[i] = __float2half_rn(k < K ? src[(size_t)n * K + k] : 0.f);
    }
}

}  // namespace
}  // namespace b2k
