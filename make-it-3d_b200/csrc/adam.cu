// adam.cu -- torch.optim.Adam's step with the Trainer's gradient clip folded in, for sm_90a (C ABI: include/mi3d.h)
//
// Replaces, in ONE elementwise pass per parameter tensor, what the reference runs for `--optim adam|adamw` (main.py:133-134):
//     nn.utils.clip_grad_norm(model.parameters(), max_norm=10)            nerf/utils.py:984
//     torch.optim.Adam(..., betas=(0.9, 0.99), eps=1e-15).step()          torch's _multi_tensor_adam, capturable=False
// The global gradient norm comes from mi3d_sumsq (adan.cu) and stays on the device: no host synchronisation.
// The clip coefficient is formed as _clip_grads_with_norm_ forms it in fp32: clamp(max_norm / (norm + 1e-6), max=1), where the
// python-float-over-tensor division is torch's reciprocal() * max_norm.  The per-element update is adam_update.cuh, shared with
// the refine Adam.  Compiled with -fmad=false (see adam_update.cuh).
// HBM-bound: p g m v in, p g m v out (g only when clipping) = 32 B / element, plus mi3d_sumsq's 4 B.
#include "adam_update.cuh"
#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kThreads = 256;

// torch.clamp(coef, max=1) keeps a NaN coefficient (a non-finite norm), so the clipped gradients turn NaN as torch's do
__device__ __forceinline__ float clip_coef(const float* total_sumsq, float max_norm) {
    const float coef = (1.0f / (sqrtf(*total_sumsq) + 1e-6f)) * max_norm;
    return coef > 1.0f ? 1.0f : coef;
}

// VEC: every pointer 16-byte aligned; thread t owns elements [4t, 4t + 4)
template <bool VEC>
__global__ void __launch_bounds__(kThreads)
k_adam(float* __restrict__ param, float* __restrict__ grad, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, uint64_t n,
       const float* __restrict__ total_sumsq, float max_norm, const mi3d_adam::Scalars a) {
    const bool clip = max_norm > 0.f;
    const float coef = clip ? clip_coef(total_sumsq, max_norm) : 1.f;
    const uint64_t t = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
    if (VEC && t * 4 + 3 < n) {
        float4 p = *reinterpret_cast<const float4*>(param + t * 4), g = *reinterpret_cast<const float4*>(grad + t * 4);
        float4 m = *reinterpret_cast<const float4*>(exp_avg + t * 4), v = *reinterpret_cast<const float4*>(exp_avg_sq + t * 4);
        if (clip) {
            g.x = g.x * coef; g.y = g.y * coef; g.z = g.z * coef; g.w = g.w * coef;
            *reinterpret_cast<float4*>(grad + t * 4) = g;
        }
        mi3d_adam::update(p.x, m.x, v.x, g.x, a);
        mi3d_adam::update(p.y, m.y, v.y, g.y, a);
        mi3d_adam::update(p.z, m.z, v.z, g.z, a);
        mi3d_adam::update(p.w, m.w, v.w, g.w, a);
        *reinterpret_cast<float4*>(param + t * 4) = p;
        *reinterpret_cast<float4*>(exp_avg + t * 4) = m;
        *reinterpret_cast<float4*>(exp_avg_sq + t * 4) = v;
        return;
    }
    for (uint64_t i = VEC ? t * 4 : t; i < (VEC ? t * 4 + 4 : t + 1) && i < n; i++) {
        float p = param[i], g = grad[i], m = exp_avg[i], v = exp_avg_sq[i];
        if (clip) { g = g * coef; grad[i] = g; }
        mi3d_adam::update(p, m, v, g, a);
        param[i] = p; exp_avg[i] = m; exp_avg_sq[i] = v;
    }
}

}  // namespace

extern "C" {

int mi3d_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, uint64_t n, const float* total_sumsq,
                   const mi3d_adam_cfg* c, mi3d_stream_t stream) {
    if (n == 0) return MI3D_OK;
    if (!param || !grad || !exp_avg || !exp_avg_sq || !c || c->step < 1 || !(c->clip_grad_norm >= 0.f)) return MI3D_ERR_ARG;
    if (c->clip_grad_norm > 0.f && !total_sumsq) return MI3D_ERR_ARG;
    const mi3d_adam::Scalars a = mi3d_adam::host_scalars(c->lr, c->beta1, c->beta2, c->eps, c->step);
    const bool vec = ((((uintptr_t)param) | ((uintptr_t)grad) | ((uintptr_t)exp_avg) | ((uintptr_t)exp_avg_sq)) & 15) == 0;
    const uint64_t threads = vec ? (n + 3) / 4 : n;
    const uint64_t blocks = (threads + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffull) return MI3D_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (vec)
        k_adam<true><<<(unsigned)blocks, kThreads, 0, st>>>(param, grad, exp_avg, exp_avg_sq, n, total_sumsq, c->clip_grad_norm, a);
    else
        k_adam<false><<<(unsigned)blocks, kThreads, 0, st>>>(param, grad, exp_avg, exp_avg_sq, n, total_sumsq, c->clip_grad_norm, a);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
