// Strand geometry of GaussianModelCurves (src/scene/gaussian_model_strands.py:435-454) around the strand instantiation
// of the projection kernels (gh_project.cu, flag bit 10).  The model's only geometric parameter is the polyline's
// segment vectors d (S, L, 3); the reference rebuilds every per-Gaussian tensor from them in PyTorch each iteration:
//   p_0 = origin_s,  p_{k+1} = origin_s + sum_{j<=k} d_{s,j}   (torch.cumsum)
//   xyz[s L + k] = 0.5 (p_k + p_{k+1})                         (segment midpoints)
// plus scales and rotations, which the projection kernels now derive from d in registers.  Here:
//   gh_strand_midpoints_kernel  the midpoints, one thread per (strand, component) summing the segments in order:
//                               bit-identical to torch.cumsum + the reference's midpoint expression (any L >= 1)
//   gh_strand_backward_kernel   dL/dd_k = direct_k + 0.5 gx_k + sum_{j>k} gx_j, with gx = dL/dxyz (the chain rule of the
//                               cumsum and the midpoint average), one warp per strand, suffix scan from the tip;
//                               written in place over the direct terms the projection backward left in d_dirs.
// Bytes per Gaussian: midpoints read 12 (d) and write 12 (xyz); the backward reads 24 (gx, direct) and writes 12.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_ST_THREADS 128
#define GH_ST_WARPS (GH_ST_THREADS / 32)

// One thread per (strand, component).  The running sum is accumulated in segment order, which is the order of
// torch.cumsum along a dimension that is not the innermost one (one sequential loop per output column), and the
// midpoint is formed as the reference forms it, ((o + c_k) + (o + c_{k-1})) * 0.5 with c_{-1} = 0: the midpoints are
// bit-identical to initialize_gaussians_hair()'s.  That matters beyond the last bit: the rasterizer sorts by view
// depth, and opaque segments of different strands at near-equal depth swap places on a one-ulp change of position.
__global__ void __launch_bounds__(GH_ST_THREADS)
gh_strand_midpoints_kernel(int S, int L, const float* __restrict__ origins, const float* __restrict__ dirs,
                           float* __restrict__ xyz)
{
    const int t = blockIdx.x * GH_ST_THREADS + threadIdx.x;
    if (t >= 3 * S) return;
    const int s = t / 3, c = t - 3 * s;
    const float o = origins[t];                       // origins (S,1,3): element (s, 0, c)
    const float* d = dirs + (size_t)s * L * 3 + c;
    float* out = xyz + (size_t)s * L * 3 + c;
    float acc = 0.f, prev = o + 0.f;                  // p_0 = origin + 0
#pragma unroll 4
    for (int k = 0; k < L; k++) {
        acc += d[3 * (size_t)k];
        const float p = o + acc;                      // p_{k+1}
        out[3 * (size_t)k] = (p + prev) * 0.5f;
        prev = p;
    }
}

__global__ void __launch_bounds__(GH_ST_THREADS)
gh_strand_backward_kernel(int S, int L, const float* __restrict__ d_xyz, float* __restrict__ d_dirs,
                          unsigned int* __restrict__ nan_flag)
{
    const int s = blockIdx.x * GH_ST_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (s >= S) return;
    const float* gx = d_xyz + (size_t)s * L * 3;
    float* gd = d_dirs + (size_t)s * L * 3;
    float cx = 0.f, cy = 0.f, cz = 0.f;               // sum of gx over the segments beyond this chunk
    bool bad = false;
    const int nchunks = (L + 31) / 32;
    for (int c = nchunks - 1; c >= 0; c--) {
        const int k = c * 32 + lane;
        float x = 0.f, y = 0.f, z = 0.f;
        if (k < L) { x = gx[3 * (size_t)k]; y = gx[3 * (size_t)k + 1]; z = gx[3 * (size_t)k + 2]; }
        const float hx = 0.5f * x, hy = 0.5f * y, hz = 0.5f * z;
        // inclusive suffix sums within the chunk
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float ux = __shfl_down_sync(0xffffffffu, x, o), uy = __shfl_down_sync(0xffffffffu, y, o), uz = __shfl_down_sync(0xffffffffu, z, o);
            if (lane + o < 32) { x += ux; y += uy; z += uz; }
        }
        // exclusive: the segments after k (the next lane's inclusive sum, the carry for the chunk's last lane)
        float ex = __shfl_down_sync(0xffffffffu, x, 1), ey = __shfl_down_sync(0xffffffffu, y, 1), ez = __shfl_down_sync(0xffffffffu, z, 1);
        if (lane == 31) { ex = 0.f; ey = 0.f; ez = 0.f; }
        if (k < L) {
            const float tx = gd[3 * (size_t)k] + hx + (cx + ex);
            const float ty = gd[3 * (size_t)k + 1] + hy + (cy + ey);
            const float tz = gd[3 * (size_t)k + 2] + hz + (cz + ez);
            gd[3 * (size_t)k] = tx; gd[3 * (size_t)k + 1] = ty; gd[3 * (size_t)k + 2] = tz;
            bad |= (tx != tx) || (ty != ty) || (tz != tz);
        }
        cx += __shfl_sync(0xffffffffu, x, 0); cy += __shfl_sync(0xffffffffu, y, 0); cz += __shfl_sync(0xffffffffu, z, 0);
    }
    // the optimizer's NaN guard (train_strands.py:154-157 checks _dirs) sees the totals, not only the direct terms
    if (nan_flag != nullptr && __any_sync(0xffffffffu, bad) && lane == 0) atomicOr(nan_flag, 1u);
}

int gh_strand_check(int S, int L, const char* who)
{
    if (S <= 0 || L <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: S and L must be positive", who);
    if ((unsigned long long)S * L * 3 > 0x7fffffffull) return gh_set_error(GH_E_INVALID_ARG, "%s: 3 * S * L must stay below 2^31", who);
    return GH_OK;
}

}  // namespace

// the two kernels for entry points outside this file (gh_hair_strands_*_capturable); S, L checked by the caller
void gh_launch_strand_midpoints(int S, int L, const float* origins, const float* dirs, float* xyz, cudaStream_t stream)
{
    gh_strand_midpoints_kernel<<<(3 * S + GH_ST_THREADS - 1) / GH_ST_THREADS, GH_ST_THREADS, 0, stream>>>(S, L, origins, dirs, xyz);
}

void gh_launch_strand_backward(int S, int L, const float* d_xyz, float* d_dirs, unsigned int* nan_flag, cudaStream_t stream)
{
    gh_strand_backward_kernel<<<(S + GH_ST_WARPS - 1) / GH_ST_WARPS, GH_ST_THREADS, 0, stream>>>(S, L, d_xyz, d_dirs, nan_flag);
}

extern "C" int gh_strand_midpoints(int S, int L, const float* origins, const float* dirs, float* xyz, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    const int rc = gh_strand_check(S, L, "gh_strand_midpoints");
    if (rc != GH_OK) return rc;
    if (!origins || !dirs || !xyz) return gh_set_error(GH_E_INVALID_ARG, "gh_strand_midpoints: missing pointer");
    gh_strand_midpoints_kernel<<<(3 * S + GH_ST_THREADS - 1) / GH_ST_THREADS, GH_ST_THREADS, 0, stream>>>(S, L, origins, dirs, xyz);
    return gh_launch_status("gh_strand_midpoints", 1);
}

extern "C" int gh_strand_backward(int S, int L, const float* d_xyz, float* d_dirs, unsigned int* nan_flag, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    const int rc = gh_strand_check(S, L, "gh_strand_backward");
    if (rc != GH_OK) return rc;
    if (!d_xyz || !d_dirs) return gh_set_error(GH_E_INVALID_ARG, "gh_strand_backward: missing pointer");
    gh_strand_backward_kernel<<<(S + GH_ST_WARPS - 1) / GH_ST_WARPS, GH_ST_THREADS, 0, stream>>>(S, L, d_xyz, d_dirs, nan_flag);
    return gh_launch_status("gh_strand_backward", 1);
}
