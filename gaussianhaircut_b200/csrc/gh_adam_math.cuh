// torch.optim.Adam's per-element update and its device-side bias-correction set-up, shared by the Gaussian optimizer
// (gh_adam.cu) and the per-camera optimizer (gh_camera.cu) so that both apply the same arithmetic.
#pragma once
#include <cuda_runtime.h>

// MUFU-based square root / reciprocal (about 1 ulp each): the update is bandwidth bound only if the
// per-element arithmetic stays short.  The result differs from torch's IEEE sqrt + divide by a few
// ulp of the UPDATE, i.e. ~1e-7 * lr relative to the parameter.
static __device__ __forceinline__ float gh_sqrt_approx(float x) { float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
static __device__ __forceinline__ float gh_rcp_approx(float x) { float r; asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

struct GhAdamConst { float beta1, beta2, omb1, omb2, eps, inv_bc2s, step_size; };

static __device__ __forceinline__ void gh_adam_elem(float& p, float gr, float& m, float& v, const GhAdamConst& c) {
    m = fmaf(c.omb1, gr - m, m);                           // exp_avg.lerp_(grad, 1 - beta1)
    v = fmaf(v, c.beta2, (c.omb2 * gr) * gr);              // mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = fmaf(gh_sqrt_approx(v), c.inv_bc2s, c.eps);   // sqrt(v) / sqrt(bias_correction2) + eps
    p = fmaf(-(c.step_size * m), gh_rcp_approx(denom), p);            // addcdiv_(exp_avg, denom, -lr / bias_correction1)
}

// bias corrections for a device-resident step count (the count AFTER this step, >= 1): 1 - beta1^step and
// sqrt(1 - beta2^step)
static __device__ __forceinline__ float gh_adam_bc1(float beta1, int step) { return 1.0f - powf(beta1, (float)step); }
static __device__ __forceinline__ float gh_adam_bc2_sqrt(float beta2, int step) { return sqrtf(1.0f - powf(beta2, (float)step)); }

static __device__ __forceinline__ GhAdamConst gh_adam_const(float beta1, float beta2, float eps, float lr, float bc1,
                                                           float bc2_sqrt) {
    GhAdamConst c;
    c.beta1 = beta1; c.beta2 = beta2; c.omb1 = 1.0f - beta1; c.omb2 = 1.0f - beta2; c.eps = eps;
    c.inv_bc2s = 1.0f / bc2_sqrt; c.step_size = lr / bc1;
    return c;
}
