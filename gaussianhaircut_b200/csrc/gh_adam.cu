// "Next" row 2 (SURVEY.md 8f): the optimiser step that follows the rasterizer backward.
// One launch updates every parameter group with torch.optim.Adam's arithmetic
// (reference: torch.optim.Adam(l, lr=0.0, eps=1e-15), SRC/scene/gaussian_model.py:431-448) and the
// reference's NaN guard (SRC/train_gaussians.py:174-181: skip the step if any gradient has a NaN,
// done there with seven blocking `.isnan().any()` host syncs) is a device-side flag: no host sync.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_adam_math.cuh"
#include "../../include/gh_rasterizer.h"

namespace {

struct GhAdamGroups {
    float* param[GH_ADAM_MAX_GROUPS];
    const float* grad[GH_ADAM_MAX_GROUPS];
    float* exp_avg[GH_ADAM_MAX_GROUPS];
    float* exp_avg_sq[GH_ADAM_MAX_GROUPS];
    unsigned long long end[GH_ADAM_MAX_GROUPS];   // exclusive prefix of element counts
    float lr[GH_ADAM_MAX_GROUPS];
    int n;
};

// grid = (blocks, groups): blockIdx.y is the parameter group, float4 per thread when the group's four
// arrays are 16-byte aligned (torch allocations are), scalar tail / fallback otherwise.
__global__ void __launch_bounds__(256)
gh_adam_nan_kernel(GhAdamGroups g, unsigned int* __restrict__ flag)
{
    const int k = blockIdx.y;
    const unsigned long long n = g.end[k] - (k ? g.end[k - 1] : 0ull);
    const float* __restrict__ gr = g.grad[k];
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long nthreads = (unsigned long long)gridDim.x * blockDim.x;
    bool bad = false;
    unsigned long long done = 0;
    if ((reinterpret_cast<size_t>(gr) & 15) == 0) {
        const unsigned long long n4 = n >> 2;
        const float4* g4 = reinterpret_cast<const float4*>(gr);
        for (unsigned long long i = tid; i < n4; i += nthreads) {
            const float4 x = g4[i];
            bad |= (x.x != x.x) | (x.y != x.y) | (x.z != x.z) | (x.w != x.w);
        }
        done = n4 << 2;
    }
    for (unsigned long long i = done + tid; i < n; i += nthreads) { const float x = gr[i]; bad |= (x != x); }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1u);
}

// DEV_LR: the learning rates are read from device memory (lr_dev[group]) instead of the launch argument.
// `step` (1-based) is used when step_state is NULL.
template <bool DEV_LR>
__device__ __forceinline__ void
gh_adam_update_body(const GhAdamGroups& g, const float* __restrict__ lr_dev, double beta1, double beta2, float eps,
                    int step, const unsigned int* __restrict__ flag,
                    const unsigned int* __restrict__ skip_flag, int* step_state)
{
    // thread 0 reads the flags and the step count and derives the constants once per CTA; nothing else reads them
    __shared__ GhAdamConst c_sh;
    __shared__ int skip_sh;
    const int k = blockIdx.y;
    if (threadIdx.x == 0) {
        // independent loads, issued together
        const unsigned int nan_seen = flag != nullptr ? *flag : 0u, skip_seen = skip_flag != nullptr ? *skip_flag : 0u;
        const int taken = step_state != nullptr ? step_state[0] : 0;
        const float lr = DEV_LR ? lr_dev[k] : g.lr[k];
        // a gradient held a NaN, or the producer of the gradients reported a failure: skip this step entirely
        skip_sh = (nan_seen | skip_seen) != 0u;
        // device-resident step count (only advanced by steps that were not skipped, like torch's state['step'])
        if (step_state != nullptr) step = taken + 1;
        if (!skip_sh) c_sh = gh_adam_const(beta1, beta2, eps, lr, gh_adam_bias(beta1, beta2, step));
    }
    __syncthreads();
    if (skip_sh) return;
    const GhAdamConst c = c_sh;
    const unsigned long long n = g.end[k] - (k ? g.end[k - 1] : 0ull);
    float* __restrict__ P = g.param[k];
    const float* __restrict__ G = g.grad[k];
    float* __restrict__ M = g.exp_avg[k];
    float* __restrict__ V = g.exp_avg_sq[k];
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long nthreads = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long done = 0;
    if (((reinterpret_cast<size_t>(P) | reinterpret_cast<size_t>(G) | reinterpret_cast<size_t>(M) | reinterpret_cast<size_t>(V)) & 15) == 0) {
        const unsigned long long n4 = n >> 2;
        for (unsigned long long i = tid; i < n4; i += nthreads) {
            float4 p = reinterpret_cast<float4*>(P)[i];
            const float4 gr = reinterpret_cast<const float4*>(G)[i];
            float4 m = reinterpret_cast<float4*>(M)[i], v = reinterpret_cast<float4*>(V)[i];
            gh_adam_elem(p.x, gr.x, m.x, v.x, c); gh_adam_elem(p.y, gr.y, m.y, v.y, c);
            gh_adam_elem(p.z, gr.z, m.z, v.z, c); gh_adam_elem(p.w, gr.w, m.w, v.w, c);
            reinterpret_cast<float4*>(P)[i] = p;
            reinterpret_cast<float4*>(M)[i] = m;
            reinterpret_cast<float4*>(V)[i] = v;
        }
        done = n4 << 2;
    }
    for (unsigned long long i = done + tid; i < n; i += nthreads) {
        float p = P[i], m = M[i], v = V[i];
        gh_adam_elem(p, G[i], m, v, c);
        P[i] = p; M[i] = m; V[i] = v;
    }
    if (step_state != nullptr) {
        // the last CTA to finish advances the counter: every CTA's thread 0 read it before the __syncthreads() above,
        // and this one waits for the whole CTA before it counts itself done
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned int t = atomicAdd(reinterpret_cast<unsigned int*>(step_state + 1), 1u);
            if (t == gridDim.x * gridDim.y - 1) { step_state[0] += 1; step_state[1] = 0; }
        }
    }
}

__global__ void __launch_bounds__(256)
gh_adam_update_kernel(GhAdamGroups g, double beta1, double beta2, float eps, int step,
                      const unsigned int* __restrict__ flag, const unsigned int* __restrict__ skip_flag, int* step_state)
{
    gh_adam_update_body<false>(g, nullptr, beta1, beta2, eps, step, flag, skip_flag, step_state);
}

// gh_adam_step_capturable: learning rates from device memory, step count always on the device
__global__ void __launch_bounds__(256)
gh_adam_update_dev_lr_kernel(GhAdamGroups g, const float* __restrict__ lrs, double beta1, double beta2, float eps,
                             const unsigned int* __restrict__ flag, const unsigned int* __restrict__ skip_flag,
                             int* step_state)
{
    gh_adam_update_body<true>(g, lrs, beta1, beta2, eps, 0, flag, skip_flag, step_state);
}

}  // namespace

// the kernel-argument view of the caller's HOST arrays (no launch); GH_OK or GH_E_INVALID_ARG
// one grid row per group; enough CTAs per row for the largest group to fill the machine
static int gh_adam_groups(const char* who, int n_groups, float* const* params, const float* const* grads,
                          float* const* exp_avg, float* const* exp_avg_sq, const unsigned long long* sizes,
                          const float* lrs_host, GhAdamGroups& g, unsigned long long& total, dim3& grid)
{
    total = 0;
    for (int k = 0; k < GH_ADAM_MAX_GROUPS; k++) {
        const bool on = k < n_groups;
        g.param[k] = on ? params[k] : nullptr; g.grad[k] = on ? grads[k] : nullptr;
        g.exp_avg[k] = on ? exp_avg[k] : nullptr; g.exp_avg_sq[k] = on ? exp_avg_sq[k] : nullptr;
        g.lr[k] = (on && lrs_host) ? lrs_host[k] : 0.f;
        if (on) {
            if (!params[k] || !grads[k] || !exp_avg[k] || !exp_avg_sq[k])
                return gh_set_error(GH_E_INVALID_ARG, "%s: NULL parameter / gradient / moment pointer", who);
            total += sizes[k];
        }
        g.end[k] = total;
    }
    g.n = n_groups;
    unsigned long long largest = 0;
    for (int k = 0; k < n_groups; k++) largest = sizes[k] > largest ? sizes[k] : largest;
    const unsigned long long want = (largest / 4 + 255) / 256;
    grid = dim3((unsigned int)(want < 1 ? 1 : (want > 132ull * 8 ? 132ull * 8 : want)), (unsigned int)n_groups);
    return GH_OK;
}

extern "C" int gh_adam_step(int n_groups, float* const* params, const float* const* grads,
                            float* const* exp_avg, float* const* exp_avg_sq,
                            const unsigned long long* sizes, const float* lrs,
                            double beta1, double beta2, float eps, int step, int* step_state,
                            unsigned int* nan_flag, const unsigned int* skip_flag, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (n_groups <= 0 || n_groups > GH_ADAM_MAX_GROUPS || (step < 1 && step_state == nullptr) || !params || !grads || !exp_avg || !exp_avg_sq || !sizes || !lrs)
        return gh_set_error(GH_E_INVALID_ARG, "gh_adam_step: bad group count / step or missing array");
    GhAdamGroups g;
    unsigned long long total;
    dim3 grid;
    const int rc = gh_adam_groups("gh_adam_step", n_groups, params, grads, exp_avg, exp_avg_sq, sizes, lrs, g, total, grid);
    if (rc != GH_OK || total == 0) return rc;
    if (nan_flag) {
        const cudaError_t e = cudaMemsetAsync(nan_flag, 0, sizeof(unsigned int), stream);
        if (e != cudaSuccess) return gh_cuda_status("gh_adam_step", "memset(NaN flag)", e);
        gh_adam_nan_kernel<<<grid, 256, 0, stream>>>(g, nan_flag);
    }
    gh_adam_update_kernel<<<grid, 256, 0, stream>>>(g, beta1, beta2, eps, step, nan_flag, skip_flag, step_state);
    return gh_launch_status("gh_adam_step", nan_flag ? 2 : 1);
}

extern "C" int gh_adam_step_capturable(int n_groups, float* const* params, const float* const* grads,
                                       float* const* exp_avg, float* const* exp_avg_sq,
                                       const unsigned long long* sizes, const float* lrs,
                                       double beta1, double beta2, float eps, int* step_state,
                                       unsigned int* nan_flag, const unsigned int* skip_flag, int debug, gh_stream_t stream_)
{
    const char* who = "gh_adam_step_capturable";
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc != GH_OK) return rc;
    if (n_groups <= 0 || n_groups > GH_ADAM_MAX_GROUPS || !params || !grads || !exp_avg || !exp_avg_sq || !sizes)
        return gh_set_error(GH_E_INVALID_ARG, "%s: bad group count or missing array", who);
    if (!lrs) return gh_set_error(GH_E_INVALID_ARG, "%s: lrs (device float[n_groups]) is required", who);
    if (!step_state) return gh_set_error(GH_E_INVALID_ARG, "%s: step_state (device int[2]) is required", who);
    GhAdamGroups g;
    unsigned long long total;
    dim3 grid;
    rc = gh_adam_groups(who, n_groups, params, grads, exp_avg, exp_avg_sq, sizes, nullptr, g, total, grid);
    if (rc != GH_OK || total == 0) return rc;
    if (nan_flag) {
        rc = gh_cuda_status(who, "memset(NaN flag)", cudaMemsetAsync(nan_flag, 0, sizeof(unsigned int), stream));
        if (rc != GH_OK) return rc;
        gh_adam_nan_kernel<<<grid, 256, 0, stream>>>(g, nan_flag);
    }
    gh_adam_update_dev_lr_kernel<<<grid, 256, 0, stream>>>(g, lrs, beta1, beta2, eps, nan_flag, skip_flag, step_state);
    return gh_launch_status(who, nan_flag ? 2 : 1);
}
