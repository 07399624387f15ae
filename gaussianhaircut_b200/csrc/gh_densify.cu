// "Next" row 3 (SURVEY.md 8f-3): adaptive density control as ONE classification pass and ONE compaction pass.
//
// The reference's `GaussianModel.densify_and_prune` (src/scene/gaussian_model.py:723-737, run every 100 iterations,
// src/train_gaussians.py:160-171) is densify_and_clone (:708-721) + densify_and_split (:682-706) + prune_points
// (:613-630), each of which re-allocates every parameter tensor AND both Adam moments with boolean-mask gathers and
// torch.cat (cat_tensors_to_optimizer :632-654, _prune_optimizer :595-611): ~25 tensors x 3 rounds of
// gather / concatenate kernels, and finishes with torch.cuda.empty_cache().
//
// The outcome of the three rounds is a pure function of per-Gaussian decisions, so it is computed directly:
//   classify  (one thread per Gaussian): g = grad_accum / denom (NaN -> 0), s_max = max exp(log-scale),
//             clone = g >= thr and s_max <= percent_dense * extent        (:710-712)
//             split = g >= thr and s_max >  percent_dense * extent        (:687-689; clones have padded grad 0)
//             the final prune (:728-733) per resulting row: opacity < min_opacity, or world-size s_max > 0.1 * extent
//             (the screen-size test never fires: densification_postfix zeroes max_radii2D before it is read, :674);
//             children of a split use the shrunk scale s / (0.8 * 2)      (:695), which torch on the device forms as
//             s * fl(1 / fl(1.6)) = s * 0.625f (a tensor divided by a Python scalar is multiplied by its reciprocal);
//             s_max and the children's max are NaN when any component is, as torch.max is: no NaN row is cloned,
//             split or pruned on its size
//             -> keep flags A (original survives: not split, not pruned), B (its clone survives), C (its two children survive)
//   scan      exclusive prefix sums of the three flags (device-wide; done by the caller)
//   scatter   (one thread per source Gaussian): rows go to their final position in the reference's order
//             [surviving originals | surviving clones | first children | second children], parameters and both Adam
//             moments in the same pass; clones and children start with zero moments (:640-641); child position =
//             R(q) * sample + xyz with the caller's N(0, s) samples (:690-694), child log-scale = log(s * 0.625f).
// Everything is written exactly once; nothing is re-allocated in between.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_DN_MAX_TENSORS 8

struct GhDensifyTensors {
    const float* src[GH_DN_MAX_TENSORS];      // parameter tensors, row-major (P, row[k])
    const float* m1[GH_DN_MAX_TENSORS];       // exp_avg  (NULL: this tensor has no optimizer state)
    const float* m2[GH_DN_MAX_TENSORS];       // exp_avg_sq
    float* dst[GH_DN_MAX_TENSORS];
    float* dm1[GH_DN_MAX_TENSORS];
    float* dm2[GH_DN_MAX_TENSORS];
    int row[GH_DN_MAX_TENSORS];               // floats per Gaussian
    int n;
    int xyz_index, scaling_index, rotation_index;
};

// torch.max(dim=1) propagates a NaN component; fmaxf would drop it
__device__ __forceinline__ float gh_max_nan(float a, float b) { return (a != a || a > b) ? a : b; }

// a split child's scale, get_scaling / (0.8 * 2), bit-identical to torch's s * (1.0f / 1.6f) with 1.0f / 1.6f = 0.625f
__device__ __forceinline__ float gh_child_scale(float s) { return s * 0.625f; }

__global__ void __launch_bounds__(256)
gh_densify_classify_kernel(int P, const float* __restrict__ grad_accum, const float* __restrict__ denom,
                           const float* __restrict__ log_scaling, const float* __restrict__ opacity_logit,
                           float grad_threshold, float dense_extent, float min_opacity, float ws_limit,
                           int* __restrict__ flags)       // (P, 4): keep original, keep clone, keep children, split (before the prune)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float g = grad_accum[i] / denom[i];
    if (g != g) g = 0.f;                                               // grads[grads.isnan()] = 0.0
    const float s0 = expf(log_scaling[3 * (size_t)i]), s1 = expf(log_scaling[3 * (size_t)i + 1]), s2 = expf(log_scaling[3 * (size_t)i + 2]);
    const float smax = gh_max_nan(s0, gh_max_nan(s1, s2));
    const bool hot = (fabsf(g) >= grad_threshold);
    const bool clone = hot && (smax <= dense_extent);
    const bool split = (g >= grad_threshold) && (smax > dense_extent);
    const float op = 1.0f / (1.0f + expf(-opacity_logit[i]));
    const bool prune_self = (op < min_opacity) || (ws_limit > 0.f && smax > ws_limit);
    // children: new log-scale = log(s * 0.625f); their get_scaling is exp of that
    const float cmax = gh_max_nan(expf(logf(gh_child_scale(s0))), gh_max_nan(expf(logf(gh_child_scale(s1))), expf(logf(gh_child_scale(s2)))));
    const bool prune_child = (op < min_opacity) || (ws_limit > 0.f && cmax > ws_limit);
    reinterpret_cast<int4*>(flags)[i] = make_int4((!split && !prune_self) ? 1 : 0, (clone && !prune_self) ? 1 : 0,
                                                  (split && !prune_child) ? 1 : 0, split ? 1 : 0);
}

// prefix: INCLUSIVE prefix sums of `flags` (P, 4) -- exclusive = inclusive - flag.  Column 3 ranks the Gaussians that
// are split BEFORE the final prune: the caller draws the normal samples for every one of them, like the reference.
__global__ void __launch_bounds__(128)
gh_densify_scatter_kernel(int P, GhDensifyTensors T, const int* __restrict__ flags, const int* __restrict__ prefix,
                          int nA, int nB, int nC, const float* __restrict__ samples, int n_split_all)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int4 f = reinterpret_cast<const int4*>(flags)[i], pf = reinterpret_cast<const int4*>(prefix)[i];
    const int fA = f.x, fB = f.y, fC = f.z;
    if (!(fA | fB | fC)) return;
    const int dA = pf.x - fA;
    const int dB = nA + pf.y - fB;
    const int dC0 = nA + nB + pf.z - fC, dC1 = dC0 + nC;

    float child0[3] = {0.f, 0.f, 0.f}, child1[3] = {0.f, 0.f, 0.f}, cscale[3] = {0.f, 0.f, 0.f};
    if (fC) {
        const float* q = T.src[T.rotation_index] + 4 * (size_t)i;
        const float* ls = T.src[T.scaling_index] + 3 * (size_t)i;
        const float* x = T.src[T.xyz_index] + 3 * (size_t)i;
        const float qn = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);      // build_rotation normalises
        const float r = q[0] * qn, a = q[1] * qn, b = q[2] * qn, c = q[3] * qn;
        // general_utils.py:79-109 layout: R[0][0]=1-2(yy+zz) R[1][0]=2(xy-rz) R[2][0]=2(xz+ry) R[0][1]=2(xy+rz) ...
        const float R00 = 1.f - 2.f * (b * b + c * c), R10 = 2.f * (a * b - r * c), R20 = 2.f * (a * c + r * b);
        const float R01 = 2.f * (a * b + r * c), R11 = 1.f - 2.f * (a * a + c * c), R21 = 2.f * (b * c - r * a);
        const float R02 = 2.f * (a * c - r * b), R12 = 2.f * (b * c + r * a), R22 = 1.f - 2.f * (a * a + b * b);
        const int slot = pf.w - 1;                                           // rank among ALL split Gaussians
        const float* sA = samples + 3 * (size_t)slot;                       // stds.repeat(N,1): first copy block, then second
        const float* sB = samples + 3 * ((size_t)n_split_all + slot);
        // new_xyz = bmm(rots, samples) + xyz : row k of R times the sample
        child0[0] = R00 * sA[0] + R01 * sA[1] + R02 * sA[2] + x[0];
        child0[1] = R10 * sA[0] + R11 * sA[1] + R12 * sA[2] + x[1];
        child0[2] = R20 * sA[0] + R21 * sA[1] + R22 * sA[2] + x[2];
        child1[0] = R00 * sB[0] + R01 * sB[1] + R02 * sB[2] + x[0];
        child1[1] = R10 * sB[0] + R11 * sB[1] + R12 * sB[2] + x[1];
        child1[2] = R20 * sB[0] + R21 * sB[1] + R22 * sB[2] + x[2];
#pragma unroll
        for (int k = 0; k < 3; k++) cscale[k] = logf(gh_child_scale(expf(ls[k])));   // scaling_inverse_activation(get_scaling / (0.8 * N))
    }
    for (int t = 0; t < T.n; t++) {
        const int row = T.row[t];
        const float* s = T.src[t] + (size_t)row * i;
        const bool has_m = (T.m1[t] != nullptr);
        if (fA) {
            float* d = T.dst[t] + (size_t)row * dA;
            for (int e = 0; e < row; e++) d[e] = s[e];
            if (has_m) {
                const float* a1 = T.m1[t] + (size_t)row * i; const float* a2 = T.m2[t] + (size_t)row * i;
                float* d1 = T.dm1[t] + (size_t)row * dA; float* d2 = T.dm2[t] + (size_t)row * dA;
                for (int e = 0; e < row; e++) { d1[e] = a1[e]; d2[e] = a2[e]; }
            }
        }
        if (fB) {
            float* d = T.dst[t] + (size_t)row * dB;
            for (int e = 0; e < row; e++) d[e] = s[e];
            if (has_m) {
                float* d1 = T.dm1[t] + (size_t)row * dB; float* d2 = T.dm2[t] + (size_t)row * dB;
                for (int e = 0; e < row; e++) { d1[e] = 0.f; d2[e] = 0.f; }
            }
        }
        if (fC) {
            float* c0 = T.dst[t] + (size_t)row * dC0; float* c1 = T.dst[t] + (size_t)row * dC1;
            if (t == T.xyz_index) { for (int e = 0; e < 3; e++) { c0[e] = child0[e]; c1[e] = child1[e]; } }
            else if (t == T.scaling_index) { for (int e = 0; e < 3; e++) { c0[e] = cscale[e]; c1[e] = cscale[e]; } }
            else { for (int e = 0; e < row; e++) { c0[e] = s[e]; c1[e] = s[e]; } }
            if (has_m) {
                float* p0 = T.dm1[t] + (size_t)row * dC0; float* p1 = T.dm1[t] + (size_t)row * dC1;
                float* q0 = T.dm2[t] + (size_t)row * dC0; float* q1 = T.dm2[t] + (size_t)row * dC1;
                for (int e = 0; e < row; e++) { p0[e] = 0.f; p1[e] = 0.f; q0[e] = 0.f; q1[e] = 0.f; }
            }
        }
    }
}

}  // namespace

extern "C" int gh_densify_classify(int P, const float* grad_accum, const float* denom, const float* log_scaling,
                                   const float* opacity_logit, float grad_threshold, float dense_extent,
                                   float min_opacity, float ws_limit, int* flags, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (P < 0 || (P > 0 && (!grad_accum || !denom || !log_scaling || !opacity_logit || !flags)))
        return gh_set_error(GH_E_INVALID_ARG, "gh_densify_classify: bad P or missing pointer");
    if (P == 0) return GH_OK;
    gh_densify_classify_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, grad_accum, denom, log_scaling, opacity_logit,
                                                                   grad_threshold, dense_extent, min_opacity, ws_limit, flags);
    return gh_launch_status("gh_densify_classify", 1);
}

extern "C" int gh_densify_scatter(int P, int n_tensors, const float* const* src, const float* const* exp_avg,
                                  const float* const* exp_avg_sq, float* const* dst, float* const* dst_exp_avg,
                                  float* const* dst_exp_avg_sq, const int* row_floats,
                                  int xyz_index, int scaling_index, int rotation_index,
                                  const int* flags, const int* inclusive_prefix, int n_keep, int n_clone, int n_split_kept,
                                  const float* samples, int n_split_all, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (P < 0 || n_tensors <= 0 || n_tensors > GH_DN_MAX_TENSORS || !src || !dst || !row_floats || !exp_avg || !exp_avg_sq ||
        !dst_exp_avg || !dst_exp_avg_sq)
        return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: bad tensor table");
    if (xyz_index < 0 || xyz_index >= n_tensors || scaling_index < 0 || scaling_index >= n_tensors ||
        rotation_index < 0 || rotation_index >= n_tensors)
        return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: xyz / scaling / rotation index out of range");
    if (P == 0) return GH_OK;
    if (!flags || !inclusive_prefix || (n_split_kept > 0 && !samples) || ((size_t)flags & 15) || ((size_t)inclusive_prefix & 15))
        return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: missing flags / prefix / samples");
    GhDensifyTensors T;
    T.n = n_tensors; T.xyz_index = xyz_index; T.scaling_index = scaling_index; T.rotation_index = rotation_index;
    for (int k = 0; k < GH_DN_MAX_TENSORS; k++) {
        const bool on = k < n_tensors;
        T.src[k] = on ? src[k] : nullptr; T.dst[k] = on ? dst[k] : nullptr; T.row[k] = on ? row_floats[k] : 0;
        T.m1[k] = on ? exp_avg[k] : nullptr; T.m2[k] = on ? exp_avg_sq[k] : nullptr;
        T.dm1[k] = on ? dst_exp_avg[k] : nullptr; T.dm2[k] = on ? dst_exp_avg_sq[k] : nullptr;
        if (on && (!src[k] || (!dst[k] && (n_keep + n_clone + n_split_kept) > 0) || row_floats[k] <= 0))
            return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: NULL tensor or bad row size");
        if (on && ((exp_avg[k] == nullptr) != (exp_avg_sq[k] == nullptr) ||
                   (exp_avg[k] != nullptr && (n_keep + n_clone + n_split_kept) > 0 && (!dst_exp_avg[k] || !dst_exp_avg_sq[k]))))
            return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: optimizer moments must come in pairs with destinations");
    }
    if (T.row[xyz_index] != 3 || T.row[scaling_index] != 3 || T.row[rotation_index] != 4)
        return gh_set_error(GH_E_INVALID_ARG, "gh_densify_scatter: xyz / scaling must have 3 and rotation 4 floats per Gaussian");
    gh_densify_scatter_kernel<<<(P + 127) / 128, 128, 0, stream>>>(P, T, flags, inclusive_prefix, n_keep, n_clone, n_split_kept,
                                                                  samples, n_split_all);
    return gh_launch_status("gh_densify_scatter", 1);
}
