// Device code shared by the image-space kernels (gh_image_loss.cu: the training losses; gh_render_maps.cu: the render
// scripts' maps and the evaluation metrics; gh_eval_ssim.cu: the evaluation SSIM): the dir -> angle epilogue, the
// SSIM window and per-pixel expression, and the fixed-order block sum.
#pragma once
#include <cmath>
#include "gh_common.cuh"

#define GH_PI_F 3.14159265358979323846f
#define GH_ORIENT_LO (-1.f + 1e-3f)     // clamp range of dir.y before acos
#define GH_ORIENT_HI (1.f - 1e-3f)

// ------------------------------------------------------------------------------------------------------------ SSIM
// loss_utils.ssim (SRC/utils/loss_utils.py:72-121): an 11x11 Gaussian window, sigma 1.5, zero padding 5, and
// C1 = 0.01^2, C2 = 0.03^2 as float32 constants.
#define GH_SSIM_R 5                     // window radius: 11 taps
#define GH_SSIM_C1 (0.01f * 0.01f)
#define GH_SSIM_C2 (0.03f * 0.03f)

// gaussian(11, 1.5) as the reference builds it: float32 taps, float32 normalisation (host code; the kernels take the
// taps as arguments)
inline void gh_ssim_window(float (&w)[11])
{
    float g[11], sum = 0.f;
    for (int k = 0; k < 11; k++) { g[k] = (float)std::exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)); sum += g[k]; }
    for (int k = 0; k < 11; k++) w[k] = g[k] / sum;
}

// One pixel of ssim_map from the five window sums mu1 = conv(x), mu2 = conv(y), e11 = conv(x^2), e22 = conv(y^2),
// e12 = conv(x y): S = (a1 a2) / (b1 b2).  The intermediate values are what the training loss differentiates through.
// ROUNDED == false (the training loss): S = a1 * a2 * (1 / (b1 b2)) with a correctly rounded reciprocal, the compiler
//   free to contract products and sums into FMAs.
// ROUNDED == true (the evaluation SSIM): every operation rounded on its own and S a correctly rounded quotient (ib is
//   not formed), so that a pixel whose two windows hold the same values gives a1 == b1, a2 == b2 and S == 1 exactly,
//   as the reference's tensor arithmetic does; a contracted mu1^2 + mu2^2 would leave a bias of a few units there.
struct GhSsimPixel {
    float a1, a2;    // 2 mu1 mu2 + C1, 2 sigma12 + C2
    float b1, b2;    // mu1^2 + mu2^2 + C1, sigma1^2 + sigma2^2 + C2
    float ib;        // 1 / (b1 b2)
    float S;         // ssim_map
};

template <bool ROUNDED = false>
__device__ __forceinline__ GhSsimPixel gh_ssim_pixel(float mu1, float mu2, float e11, float e22, float e12)
{
    GhSsimPixel p;
    if constexpr (ROUNDED) {
        const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu12 = __fmul_rn(mu1, mu2);
        const float sg1 = __fsub_rn(e11, mu1_sq), sg2 = __fsub_rn(e22, mu2_sq), sg12 = __fsub_rn(e12, mu12);
        p.a1 = __fadd_rn(2.f * mu12, GH_SSIM_C1); p.a2 = __fadd_rn(2.f * sg12, GH_SSIM_C2);
        p.b1 = __fadd_rn(__fadd_rn(mu1_sq, mu2_sq), GH_SSIM_C1); p.b2 = __fadd_rn(__fadd_rn(sg1, sg2), GH_SSIM_C2);
        p.ib = 0.f;
        p.S = __fdiv_rn(__fmul_rn(p.a1, p.a2), __fmul_rn(p.b1, p.b2));
        return p;
    }
    const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
    const float sg1 = e11 - mu1_sq, sg2 = e22 - mu2_sq, sg12 = e12 - mu12;
    p.a1 = 2.f * mu12 + GH_SSIM_C1; p.a2 = 2.f * sg12 + GH_SSIM_C2;
    p.b1 = mu1_sq + mu2_sq + GH_SSIM_C1; p.b2 = sg1 + sg2 + GH_SSIM_C2;
    p.ib = __frcp_rn(p.b1 * p.b2);
    p.S = p.a1 * p.a2 * p.ib;
    return p;
}

// The reference's epilogue on channels 5, 6 of the raw image (SRC/gaussian_renderer/__init__.py:100-105):
// dir = normalize(c5, c6) (F.normalize eps 1e-12), mirrored so that dir.x >= 0, angle = acos(clamp(dir.y) * mirror) / pi.
// The intermediate values are what the training loss differentiates through.
struct GhOrientAngle {
    float nrm;       // |(c5, c6)|
    float diry;      // dir.y before the clamp
    float mirror;    // -1 where dir.x < 0, else 1
    float t;         // clamp(dir.y) * mirror
    float ang;       // acos(t) / pi, in [0, 1]
};

__device__ __forceinline__ GhOrientAngle gh_orient_angle(float c5, float c6)
{
    GhOrientAngle o;
    o.nrm = sqrtf(c5 * c5 + c6 * c6);
    const float den = fmaxf(o.nrm, 1e-12f);                  // F.normalize eps
    const float dirx = c5 / den;
    o.diry = c6 / den;
    o.mirror = (dirx < 0.f) ? -1.f : 1.f;
    const float tcl = fminf(fmaxf(o.diry, GH_ORIENT_LO), GH_ORIENT_HI);
    o.t = tcl * o.mirror;
    o.ang = acosf(o.t) / GH_PI_F;
    return o;
}

// K sums of a 256-thread CTA grid without floating-point atomics: warp shuffle tree, the 8 warps in warp order, then
// the CTA's total goes to its own slot part[k * gridDim + CTA].  The last CTA to finish (ticket: a uint32 in
// sums[ticket_slot], zeroed by the caller) adds the slots in CTA order into sums[idx[k]], staging 256 slots at a time in
// shared memory; that is one of the orders a per-CTA atomicAdd could produce, now the only one, so the sums are
// reproducible run to run.
template <int K>
__device__ __forceinline__ void gh_block_sum_fixed(double (&v)[K], double* __restrict__ part, double* sums,
                                                   const int (&idx)[K], int ticket_slot) {
    __shared__ double s_part[K][8];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
#pragma unroll
    for (int k = 0; k < K; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    __syncthreads();
    if ((tid & 31) == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) s_part[k][tid >> 5] = v[k];
    }
    __syncthreads();
    const unsigned G = gridDim.x * gridDim.y, b = blockIdx.y * gridDim.x + blockIdx.x;
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) {
            double t = 0.0;
            for (int w = 0; w < 8; w++) t += s_part[k][w];
            part[(size_t)k * G + b] = t;
        }
        __threadfence();
        s_last = atomicAdd(reinterpret_cast<unsigned*>(sums + ticket_slot), 1u) == G - 1u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ double s_stage[K][256];
    double t = 0.0;                     // thread k: sum k
    for (unsigned c0 = 0; c0 < G; c0 += 256) {
        const unsigned m = min(256u, G - c0);
#pragma unroll
        for (int k = 0; k < K; k++)
            if ((unsigned)tid < m) s_stage[k][tid] = __ldcg(part + (size_t)k * G + c0 + tid);
        __syncthreads();
        if (tid < K)
            for (unsigned i = 0; i < m; i++) t += s_stage[tid][i];
        __syncthreads();
    }
    if (tid < K) {
        int d = idx[0];
#pragma unroll
        for (int k = 1; k < K; k++) d = (tid == k) ? idx[k] : d;
        sums[d] = t;
    }
}
