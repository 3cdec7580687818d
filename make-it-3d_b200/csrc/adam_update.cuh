// adam_update.cuh -- one element of torch.optim.Adam's step (foreach path, capturable=False, no weight decay, amsgrad off), in
// torch's operation order.  Shared by k_refine_adam (refine.cu) and k_adam (adam.cu), which are both compiled with -fmad=false:
// every op rounds once, like torch's separate kernels, and where torch's own kernels contract to an FMA (lerp, addcmul, addcdiv) the
// fmaf is written out.
#pragma once
#include <math.h>

namespace mi3d_adam {

struct Scalars {
    float w1;          // 1 - beta1: lerp weight
    float beta2, omb2; // beta2, 1 - beta2
    float step_size;   // -(lr / (1 - beta1^t))
    float bc2_sqrt;    // (1 - beta2^t)^0.5
    float eps;
};

// torch.optim.Adam's host scalars, computed as it computes them (Python floats are C doubles; ** is pow), rounded once to fp32
inline Scalars host_scalars(double lr, double beta1, double beta2, double eps, int step) {
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    Scalars a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.omb2 = (float)(1.0 - beta2);
    a.step_size = (float)((lr / bc1) * -1.0);
    a.bc2_sqrt = (float)pow(bc2, 0.5);
    a.eps = (float)eps;
    return a;
}

// exp_avg.lerp_(g, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(g, g, 1 - beta2);
// param.addcdiv_(exp_avg, sqrt(exp_avg_sq) / bc2_sqrt + eps, step_size)
__device__ __forceinline__ void update(float& p, float& m, float& v, const float g, const Scalars& a) {
    m = fmaf(a.w1, g - m, m);
    v = fmaf(a.omb2, g * g, v * a.beta2);
    const float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
    p = fmaf(a.step_size, m / denom, p);
}

}  // namespace mi3d_adam
