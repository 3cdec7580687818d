// adan.cu -- the parameter update that follows the hot path every step (SURVEY.md 8f-1), for sm_90a (C ABI: include/mi3d.h)
//
// Replaces, in ONE elementwise pass over a (shard of a) flat parameter vector, what the reference runs as ~25 separate torch ops per
// tensor plus two host synchronisations:
//     nn.utils.clip_grad_norm(model.parameters(), max_norm=10)            nerf/utils.py:984
//     Adan.step(): global-norm clip (max_grad_norm = 5.0, .item() sync)   optimizer.py:102-131
//                  _single_tensor_adan (foreach=False, main.py:132)        optimizer.py:201-256
// Both clip factors derive from the one global gradient norm, which stays on the device (total_sumsq): no .item().
// HBM-bound: 6 streams in (p, g, m, n, d, prev) and 5 out per element = 44 B/element; 12.2 M parameters -> 0.54 GB -> ~0.16 ms at
// the H100 SXM data-sheet 3.35 TB/s.  With G ranks every rank updates 1/G of the table (reduce-scatter -> this kernel -> all-gather).
#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kThreads = 256;

// deterministic two-stage sum of squares: per-block partials (fixed order), then one block folds them in fp64
__global__ void __launch_bounds__(kThreads) k_sumsq_partial(const float* __restrict__ g, uint64_t n, double* __restrict__ partials) {
    double acc = 0.0;
    const uint64_t stride = (uint64_t)gridDim.x * kThreads * 4;
    for (uint64_t i = ((uint64_t)blockIdx.x * kThreads + threadIdx.x) * 4; i < n; i += stride) {
        if (i + 3 < n) {
            const float4 v = *reinterpret_cast<const float4*>(g + i);
            acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
        } else {
            for (uint64_t j = i; j < n; j++) acc += (double)g[j] * g[j];
        }
    }
    __shared__ double sm[kThreads];
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) partials[blockIdx.x] = sm[0];
}

__global__ void __launch_bounds__(kThreads) k_sumsq_final(const double* __restrict__ partials, int n_part, float* __restrict__ out, int accumulate) {
    __shared__ double sm[kThreads];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n_part; i += kThreads) acc += partials[i];
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) *out = (accumulate ? *out : 0.f) + (float)sm[0];
}

struct AdanScalars {       // python-float (double) expressions of optimizer.py evaluated on the host in double, rounded once to fp32
    float beta1, beta2, beta3, om_beta1, om_beta2, om_beta3, eps;
    float bias_correction3_sqrt, step_size, step_size_diff, decay_mul /* 1 - lr*wd */, decay_div /* 1 + lr*wd */;
    float max_grad_norm, clip_grad_norm;
    int no_prox, first_step;
};

// one IEEE rounding per reference op, in the reference's order (optimizer.py:228-256), so the update tracks torch's to ~1 ulp
__global__ void __launch_bounds__(kThreads)
k_adan(float* __restrict__ param, float* __restrict__ grad, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
       float* __restrict__ exp_avg_diff, float* __restrict__ neg_pre_grad, uint64_t n, const float* __restrict__ total_sumsq, const AdanScalars s) {
    // clip_grad_norm_(max_norm): coef = min(1, max_norm / (norm + 1e-6)) (torch.nn.utils.clip_grad_norm_), applied to .grad in place
    float coef = 1.f;
    float norm = total_sumsq ? sqrtf(*total_sumsq) : 0.f;
    if (s.clip_grad_norm > 0.f && total_sumsq) { coef = fminf(1.f, s.clip_grad_norm / (norm + 1e-6f)); norm = norm * coef; }
    // Adan's own global clip on the already clipped gradients: clamp(max_grad_norm / (norm + eps), max = 1)   optimizer.py:112-129
    float clip = 1.f;
    if (s.max_grad_norm > 0.f && total_sumsq) clip = fminf(1.f, s.max_grad_norm / (norm + s.eps));
    const float step_size_diff = s.step_size_diff, step_size = s.step_size;
    const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    float g = grad[i] * coef;
    float prev = s.first_step ? g * (-clip) : neg_pre_grad[i];          // optimizer.py:160-162 (clone().mul_(-clip) of the unclipped-by-Adan grad)
    g = g * clip;                                                        // grad.mul_(clip)
    float diff = prev + g;                                               // neg_grad_or_diff.add_(grad)
    const float m = exp_avg[i] * s.beta1 + g * s.om_beta1;
    const float d = exp_avg_diff[i] * s.beta2 + diff * s.om_beta2;
    diff = diff * s.beta2 + g;                                           // neg_grad_or_diff.mul_(beta2).add_(grad)
    const float v = exp_avg_sq[i] * s.beta3 + s.om_beta3 * (diff * diff);
    const float denom = sqrtf(v) / s.bias_correction3_sqrt + s.eps;
    float p = param[i];
    if (s.no_prox) {
        p = p * s.decay_mul;
        p = p + (-step_size) * (m / denom);
        p = p + (-step_size_diff) * (d / denom);
    } else {
        p = p + (-step_size) * (m / denom);
        p = p + (-step_size_diff) * (d / denom);
        p = p / s.decay_div;
    }
    param[i] = p; grad[i] = g; exp_avg[i] = m; exp_avg_sq[i] = v; exp_avg_diff[i] = d; neg_pre_grad[i] = -g;
}

}  // namespace

extern "C" {

size_t mi3d_sumsq_workspace_bytes(void) { return 1024 * sizeof(double); }

int mi3d_sumsq(const float* g, uint64_t n, float* out, int accumulate, void* workspace, mi3d_stream_t stream) {
    if (!out || !workspace || (n && !g) || (((uintptr_t)g) & 15)) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    int blocks = (int)((n / 4 + kThreads - 1) / kThreads);
    if (blocks < 1) blocks = 1;
    if (blocks > 1024) blocks = 1024;
    k_sumsq_partial<<<blocks, kThreads, 0, st>>>(g, n, (double*)workspace);
    k_sumsq_final<<<1, kThreads, 0, st>>>((const double*)workspace, blocks, out, accumulate);
    MI3D_RETURN_LAUNCH();
}

int mi3d_adan_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* exp_avg_diff, float* neg_pre_grad, uint64_t n,
                   const float* total_sumsq, const mi3d_adan_cfg* c, mi3d_stream_t stream) {
    if (n == 0) return MI3D_OK;
    if (!param || !grad || !exp_avg || !exp_avg_sq || !exp_avg_diff || !neg_pre_grad || !c || c->step < 1) return MI3D_ERR_ARG;
    if ((c->max_grad_norm > 0.f || c->clip_grad_norm > 0.f) && !total_sumsq) return MI3D_ERR_ARG;
    AdanScalars s;
    const double b1 = c->beta1, b2 = c->beta2, b3 = c->beta3, lr = c->lr, wd = c->weight_decay;
    const double bc1 = 1.0 - pow(b1, (double)c->step), bc2 = 1.0 - pow(b2, (double)c->step), bc3 = 1.0 - pow(b3, (double)c->step);   // optimizer.py:145-147
    s.beta1 = (float)b1; s.beta2 = (float)b2; s.beta3 = (float)b3; s.om_beta1 = (float)(1.0 - b1); s.om_beta2 = (float)(1.0 - b2); s.om_beta3 = (float)(1.0 - b3);
    s.eps = (float)c->eps; s.bias_correction3_sqrt = (float)sqrt(bc3);
    s.step_size = (float)(lr / bc1); s.step_size_diff = (float)(lr * b2 / bc2);                                                       // optimizer.py:243-244
    s.decay_mul = (float)(1.0 - lr * wd); s.decay_div = (float)(1.0 + lr * wd);
    s.max_grad_norm = c->max_grad_norm; s.clip_grad_norm = c->clip_grad_norm; s.no_prox = c->no_prox; s.first_step = c->step == 1 || c->reset_prev;
    const uint64_t blocks = (n + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffull) return MI3D_ERR_ARG;
    k_adan<<<(unsigned)blocks, kThreads, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, exp_avg_diff, neg_pre_grad, n, total_sumsq, s);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
