// Trainable cameras on the device (DESIGN §17): the reference's BARF camera model (src/scene/cameras.py:95-152) and its
// own Adam (src/train_gaussians.py:45-63, 183-196) as three single-CTA kernels.  A camera costs a few hundred flops, so
// what matters is that nothing synchronises with the host and every call can be captured in a CUDA graph: the camera
// index is read from device memory, so one captured graph serves every view.  The arithmetic is gh_camera_math.h.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_adam_math.cuh"
#include "gh_camera_math.h"
#include "../../include/gh_rasterizer.h"

namespace {

// the device index, or -1 (and GH_STATUS_CAMERA_INDEX in *status) when it lies outside [0, n)
__device__ __forceinline__ int gh_camera_index(const int* index, int n, unsigned int* status) {
    const int i = *index;
    if (i < 0 || i >= n) {
        if (status != nullptr) atomicOr(status, GH_STATUS_CAMERA_INDEX);
        return -1;
    }
    return i;
}

__global__ void __launch_bounds__(32)
gh_camera_forward_kernel(int n, const float* __restrict__ residuals, const float* __restrict__ base,
                         const int* __restrict__ index, float* __restrict__ viewmatrix, float* __restrict__ projmatrix,
                         float* __restrict__ campos, float* __restrict__ tan_fov, unsigned int* status)
{
    if (threadIdx.x != 0) return;
    const int i = gh_camera_index(index, n, status);
    if (i < 0) return;
    float r[GH_CAM_ROW], b[GH_CAM_BASE], v[16], p[16], c[3], t[2];
    for (int k = 0; k < GH_CAM_ROW; k++) r[k] = residuals[(size_t)i * GH_CAM_ROW + k];
    for (int k = 0; k < GH_CAM_BASE; k++) b[k] = base[(size_t)i * GH_CAM_BASE + k];
    gh_camera_forward_math(b, r, v, p, c, t);
    for (int k = 0; k < 16; k++) { viewmatrix[k] = v[k]; projmatrix[k] = p[k]; }
    campos[0] = c[0]; campos[1] = c[1]; campos[2] = c[2];
    tan_fov[0] = t[0]; tan_fov[1] = t[1];
}

__global__ void __launch_bounds__(32)
gh_camera_backward_kernel(int n, const float* __restrict__ residuals, const float* __restrict__ base,
                          const int* __restrict__ index, int intrinsics, const float* __restrict__ d_camera,
                          float* __restrict__ grad, int* __restrict__ touched, unsigned int* nan_flag,
                          unsigned int* status)
{
    if (threadIdx.x != 0) return;
    const int i = gh_camera_index(index, n, status);
    if (i < 0) return;
    float r[GH_CAM_ROW], b[GH_CAM_BASE], g[GH_CAM_DCAMERA], dr[GH_CAM_ROW];
    for (int k = 0; k < GH_CAM_ROW; k++) r[k] = residuals[(size_t)i * GH_CAM_ROW + k];
    for (int k = 0; k < GH_CAM_BASE; k++) b[k] = base[(size_t)i * GH_CAM_BASE + k];
    for (int k = 0; k < GH_CAM_DCAMERA; k++) g[k] = d_camera[k];
    gh_camera_backward_math(b, r, g, intrinsics, dr);
    bool bad = false;
    for (int k = 0; k < GH_CAM_ROW; k++) {
        grad[(size_t)i * GH_CAM_ROW + k] += dr[k];
        bad |= dr[k] != dr[k];
    }
    touched[i] = 1;
    if (bad && nan_flag != nullptr) atomicOr(nan_flag, 1u);
}

// one CTA: every touched row takes torch.optim.Adam's step with its own step count; rows 0-2 / 3-5 / 6-7 use the
// rotation / translation / fov learning rate (lrs[0..2]).  Skipped as a whole -- moments and step counts unchanged --
// when *skip_flag or *nan_flag is set.  Either way the touched rows' gradients and marks are cleared, and so is the
// NaN flag (after every thread has read it).
__global__ void __launch_bounds__(256)
gh_camera_adam_kernel(int n, int cols, float* __restrict__ residuals, float* __restrict__ grad, int* __restrict__ touched,
                      float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, int* __restrict__ steps,
                      const float* __restrict__ lrs, double beta1, double beta2, float eps, unsigned int* nan_flag,
                      const unsigned int* skip_flag)
{
    const bool skip = (nan_flag != nullptr && *nan_flag != 0u) || (skip_flag != nullptr && *skip_flag != 0u);
    const float lr[3] = {lrs[0], lrs[1], lrs[2]};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (touched[i] == 0) continue;
        const size_t o = (size_t)i * GH_CAM_ROW;
        if (!skip) {
            const int step = steps[i] + 1;
            const GhAdamBias b = gh_adam_bias(beta1, beta2, step);
            for (int k = 0; k < cols; k++) {
                const GhAdamConst c = gh_adam_const(beta1, beta2, eps, lr[k < 3 ? 0 : (k < 6 ? 1 : 2)], b);
                float p = residuals[o + k], m = exp_avg[o + k], v = exp_avg_sq[o + k];
                gh_adam_elem(p, grad[o + k], m, v, c);
                residuals[o + k] = p; exp_avg[o + k] = m; exp_avg_sq[o + k] = v;
            }
            steps[i] = step;
        }
        for (int k = 0; k < GH_CAM_ROW; k++) grad[o + k] = 0.0f;
        touched[i] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0 && nan_flag != nullptr) *nan_flag = 0u;
}

}  // namespace

static bool gh_misaligned(const void* p) { return ((size_t)p & 3) != 0; }

static int gh_camera_check(const char* who, int n, int debug, const void* const* ptrs, int count)
{
    const int rc = gh_check_capturable(who, debug);
    if (rc != GH_OK) return rc;
    if (n <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: n must be positive", who);
    for (int k = 0; k < count; k++) {
        if (ptrs[k] == nullptr) return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
        if (gh_misaligned(ptrs[k])) return gh_set_error(GH_E_INVALID_ARG, "%s: pointers must be 4-byte aligned", who);
    }
    return GH_OK;
}

extern "C" int gh_camera_forward(int n, const float* residuals, const float* base, const int* index,
                                 float* viewmatrix, float* projmatrix, float* campos, float* tan_fov,
                                 unsigned int* status, int debug, gh_stream_t stream_)
{
    const char* who = "gh_camera_forward";
    gh_clear_error();
    const void* ptrs[] = {residuals, base, index, viewmatrix, projmatrix, campos, tan_fov, status};
    const int rc = gh_camera_check(who, n, debug, ptrs, 8);
    if (rc != GH_OK) return rc;
    gh_camera_forward_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>(n, residuals, base, index, viewmatrix, projmatrix,
                                                                  campos, tan_fov, status);
    return gh_launch_status(who, 1);
}

extern "C" int gh_camera_backward(int n, const float* residuals, const float* base, const int* index, int intrinsics,
                                  const float* d_camera, float* grad, int* touched, unsigned int* nan_flag,
                                  unsigned int* status, int debug, gh_stream_t stream_)
{
    const char* who = "gh_camera_backward";
    gh_clear_error();
    const void* ptrs[] = {residuals, base, index, d_camera, grad, touched, nan_flag, status};
    const int rc = gh_camera_check(who, n, debug, ptrs, 8);
    if (rc != GH_OK) return rc;
    gh_camera_backward_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>(n, residuals, base, index, intrinsics != 0, d_camera,
                                                                   grad, touched, nan_flag, status);
    return gh_launch_status(who, 1);
}

extern "C" int gh_camera_adam_step(int n, int intrinsics, float* residuals, float* grad, int* touched,
                                   float* exp_avg, float* exp_avg_sq, int* steps, const float* lrs,
                                   double beta1, double beta2, float eps, unsigned int* nan_flag,
                                   const unsigned int* skip_flag, int debug, gh_stream_t stream_)
{
    const char* who = "gh_camera_adam_step";
    gh_clear_error();
    const void* ptrs[] = {residuals, grad, touched, exp_avg, exp_avg_sq, steps, lrs, nan_flag};
    const int rc = gh_camera_check(who, n, debug, ptrs, 8);
    if (rc != GH_OK) return rc;
    if (gh_misaligned(skip_flag)) return gh_set_error(GH_E_INVALID_ARG, "%s: pointers must be 4-byte aligned", who);
    gh_camera_adam_kernel<<<1, 256, 0, (cudaStream_t)stream_>>>(n, intrinsics ? GH_CAM_ROW : 6, residuals, grad, touched,
                                                                exp_avg, exp_avg_sq, steps, lrs, beta1, beta2, eps,
                                                                nan_flag, skip_flag);
    return gh_launch_status(who, 1);
}
