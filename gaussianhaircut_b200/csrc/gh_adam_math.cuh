// torch.optim.Adam's per-element update and its device-side bias-correction set-up, shared by the Gaussian optimizer
// (gh_adam.cu) and the per-camera optimizer (gh_camera.cu) so that both apply the same arithmetic.
#pragma once
#include <cuda_runtime.h>

// MUFU-based square root / reciprocal: the update is bandwidth bound only if the per-element arithmetic stays short.
// The PTX ISA bounds sqrt.approx.f32 by 2^-23 relative and rcp.approx.f32 by 1 ulp, so each adds at most 2^-23 of
// the update to what torch's IEEE sqrt + divide would give.  tests/test_gpu_adam64.py checks every element against a
// float64 replay of torch's step to 8 units of 2^-24 of the update (plus half an ulp of the parameter).
static __device__ __forceinline__ float gh_sqrt_approx(float x) { float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
static __device__ __forceinline__ float gh_rcp_approx(float x) { float r; asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

struct GhAdamConst { float beta2, omb1, omb2, eps, inv_bc2s, step_size; };

static __device__ __forceinline__ void gh_adam_elem(float& p, float gr, float& m, float& v, const GhAdamConst& c) {
    m = fmaf(c.omb1, gr - m, m);                           // exp_avg.lerp_(grad, 1 - beta1)
    v = fmaf(v, c.beta2, (c.omb2 * gr) * gr);              // mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = fmaf(gh_sqrt_approx(v), c.inv_bc2s, c.eps);   // sqrt(v) / sqrt(bias_correction2) + eps
    p = fmaf(-(c.step_size * m), gh_rcp_approx(denom), p);            // addcdiv_(exp_avg, denom, -lr / bias_correction1)
}

// torch.optim.Adam (foreach and single-tensor) holds beta1, beta2, lr and eps as Python doubles, forms 1 - beta1,
// 1 - beta2, lr / (1 - beta1^step) and sqrt(1 - beta2^step) in double and rounds each to float only where its kernel
// takes it; so do we.  lr and eps arrive as float: the float of torch's double.

// bias corrections for step `step` (the count AFTER this step, >= 1): 1 - beta1^step and 1 / (float)sqrt(1 - beta2^step)
struct GhAdamBias { double bc1; float inv_bc2s; };

// beta1^step and beta2^step by binary powering in double: at most 2 log2(step) roundings, i.e. a relative error of a
// few 1e-15, far below the float rounding that follows, and a short dependent chain where pow() would be a long one
// (one thread per CTA derives the constants while the others wait)
static __device__ __forceinline__ void gh_adam_pow2(double b1, double b2, int step, double& p1, double& p2) {
    p1 = 1.0; p2 = 1.0;
    for (unsigned int e = (unsigned int)step; e != 0u; e >>= 1) {
        if (e & 1u) { p1 *= b1; p2 *= b2; }
        b1 *= b1; b2 *= b2;
    }
}

static __device__ __forceinline__ GhAdamBias gh_adam_bias(double beta1, double beta2, int step) {
    double p1, p2;
    gh_adam_pow2(beta1, beta2, step, p1, p2);
    GhAdamBias b;
    b.bc1 = 1.0 - p1;
    b.inv_bc2s = (float)(1.0 / (double)(float)sqrt(1.0 - p2));
    return b;
}

static __device__ __forceinline__ GhAdamConst gh_adam_const(double beta1, double beta2, float eps, float lr,
                                                           const GhAdamBias& b) {
    GhAdamConst c;
    c.beta2 = (float)beta2; c.omb1 = (float)(1.0 - beta1); c.omb2 = (float)(1.0 - beta2); c.eps = eps;
    c.inv_bc2s = b.inv_bc2s;
    c.step_size = (float)((double)lr / b.bc1);
    return c;
}
