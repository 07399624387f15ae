// Device code shared by the image-space kernels (gh_image_loss.cu: the training losses; gh_render_maps.cu: the render
// scripts' maps and the evaluation metrics): the dir -> angle epilogue and the fixed-order block sum.
#pragma once
#include "gh_common.cuh"

#define GH_PI_F 3.14159265358979323846f
#define GH_ORIENT_LO (-1.f + 1e-3f)     // clamp range of dir.y before acos
#define GH_ORIENT_HI (1.f - 1e-3f)

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
