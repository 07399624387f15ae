// Internal launcher declarations (one per stage); the public C-ABI lives in include/gh_rasterizer.h.
#pragma once
#include "gh_common.cuh"

void gh_launch_preprocess(int P, const float* means3D, const float* scales, float scale_modifier,
                          const float* rotations, const float* opacities, const float* cov3D_precomp,
                          const float* conic_precomp, const float* viewmatrix, const float* projmatrix,
                          int W, int H, float tan_fovx, float tan_fovy, int* radii,
                          GhGeomWS geom, GhImgWS img, int gx, int gy, int prefiltered, cudaStream_t stream);

void gh_launch_mark_visible(int P, const float* means3D, const float* viewmatrix, bool* present,
                            cudaStream_t stream);

// exclusive scan of the tile histogram -> ranges, cursors, R, longest list
void gh_launch_tile_scan(int T, GhImgWS img, cudaStream_t stream);

// scatter (depth|idx) records into their tile buckets; writes nothing if R (img.ctrl) exceeds `capacity` records
void gh_launch_emit(int P, const int* radii, GhGeomWS geom, GhImgWS img, GhBinWS bin, unsigned int capacity,
                    int gx, int gy, cudaStream_t stream);

// sort every tile bucket by (depth bits, gaussian idx)
// returns the number of kernels launched
int gh_launch_tile_sort(int T, unsigned int max_tile_len, long long R, GhImgWS img, GhBinWS bin, cudaStream_t stream);

// The capturable forward (R only on the device, a binning buffer of `capacity` records):
//  - capacity guard, right behind the tile scan: when R > capacity it ORs GH_STATUS_BINNING_OVERFLOW into *status and
//    turns the frame into an empty one -- every tile range (0, 0) and every radius 0 -- so that no later kernel reads
//    or writes a record at or beyond `capacity`; *num_rendered_out (may be NULL) receives R either way;
//  - the long-list sort with grids bounded by T and `capacity` (its CTAs exit when their list is short); returns the
//    number of kernels launched.
void gh_launch_capacity_guard(int P, int* radii, int T, GhImgWS img, unsigned int capacity, unsigned int* status,
                              unsigned int* num_rendered_out, cudaStream_t stream);
int gh_launch_tile_sort_capturable(int T, unsigned int capacity, GhImgWS img, GhBinWS bin, cudaStream_t stream);

// zero_records: the kernel also clears geom.acc16 (P records) for the fast blend backward
void gh_launch_blend_forward(int W, int H, int gx, int gy, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                             const float* features, const float* bg, float* out_color,
                             int P, bool zero_records, cudaStream_t stream);

// accumulates into geom.acc16 (must be zero on entry)
void gh_launch_blend_backward(int W, int H, int gx, int gy, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                              const float* features, const float* bg, const float* dL_dpix,
                              cudaStream_t stream);

// Deterministic blend backward (no atomics), three stages: the row offsets of every Gaussian (returns the number of
// kernels launched; det.off[P] = R afterwards), the per-tile walk writing one partial row per instance, and the gather
// that ASSIGNS geom.acc16 (no zeroing needed) by summing each Gaussian's rows in order.
int gh_launch_det_offsets(int P, int gx, int gy, const int* radii, GhGeomWS geom, GhDetWS det, cudaStream_t stream);
void gh_launch_blend_backward_det(int W, int H, int gx, int gy, const int* radii, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                                  GhDetWS det, const float* features, const float* bg, const float* dL_dpix,
                                  cudaStream_t stream);
void gh_launch_det_gather(int P, GhGeomWS geom, GhDetWS det, cudaStream_t stream);

// geom.acc16 -> dL_dmean2D (P,3), dL_dconic (P,4), dL_dopacity (P), dL_dcolor (P,10); writes every row
// (also zero-fills the geometry gradients that are non-null: used when the conic was supplied)
void gh_launch_unpack_grads(int P, GhGeomWS geom, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                            float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot,
                            cudaStream_t stream);

void gh_launch_preprocess_backward(int P, const float* means3D, const int* radii,
                                   const float* scales, float scale_modifier, const float* rotations,
                                   const float* cov3D_precomp, const float* conic_precomp,
                                   const float* viewmatrix, const float* projmatrix,
                                   int W, int H, float tan_fovx, float tan_fovy,
                                   const float* acc16, float* dL_dmean2D, float* dL_dconic,
                                   float* dL_dopacity, float* dL_dcolor,
                                   float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot,
                                   cudaStream_t stream);

// The forward's first phase around its per-Gaussian kernel (gh_forward_preprocess, gh_project_forward_binned):
// tile grid and its bound, workspace carving, ctrl + histogram memset, `bin(geom, img, gx, gy)` (launches the kernel on
// `stream` and counts it), tile scan, read-back of R and the longest tile list.  `who` names the entry point in error
// messages.  With a binning buffer of `bin_capacity` records (`radii` then names the radii the kernel writes), emit is
// launched right behind the read-back, so it runs while the host waits for R; *emitted tells whether R fitted.
struct GhPhase1Bin {
    const int* radii;          // written by the per-Gaussian kernel
    char* buffer;              // NULL: no emit in this phase
    long long capacity;        // records
    int* emitted;              // out: 1 if emit ran into `buffer` (R <= capacity)
};
typedef void (*GhBinLaunch)(const void* bin, const GhGeomWS& geom, const GhImgWS& img, int gx, int gy);
int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, const GhPhase1Bin& emit, GhBinLaunch launch,
                      const void* bin);
template <class F>
int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, const GhPhase1Bin& emit, const F& bin) {
    return gh_forward_phase1(who, P, width, height, geom_buffer, img_buffer, num_rendered, max_tile_len, debug, stream, emit,
                             [](const void* f, const GhGeomWS& g, const GhImgWS& i, int gx, int gy) { (*static_cast<const F*>(f))(g, i, gx, gy); }, &bin);
}
// argument checks of the optional binning buffer of the first-phase entry points (before any launch)
int gh_check_phase1_bin(const char* who, const GhPhase1Bin& emit);

// The first phase of the capturable forward (gh_project_forward_binned_capturable): as gh_forward_phase1, but nothing is
// read back and emit always goes into the caller's buffer of `capacity` records, behind the capacity guard
// (gh_launch_capacity_guard).  No host synchronisation, no allocation.
int gh_forward_phase1_capturable(const char* who, int P, int width, int height, int* radii, char* geom_buffer,
                                 char* img_buffer, char* binning_buffer, long long capacity, unsigned int* status,
                                 unsigned int* num_rendered_out, cudaStream_t stream, GhBinLaunch launch, const void* bin);
template <class F>
int gh_forward_phase1_capturable(const char* who, int P, int width, int height, int* radii, char* geom_buffer,
                                 char* img_buffer, char* binning_buffer, long long capacity, unsigned int* status,
                                 unsigned int* num_rendered_out, cudaStream_t stream, const F& bin) {
    return gh_forward_phase1_capturable(who, P, width, height, radii, geom_buffer, img_buffer, binning_buffer, capacity,
                                        status, num_rendered_out, stream,
                                        [](const void* f, const GhGeomWS& g, const GhImgWS& i, int gx, int gy) { (*static_cast<const F*>(f))(g, i, gx, gy); }, &bin);
}
// the strand geometry kernels of gh_strands.cu (gh_strand_midpoints, gh_strand_backward) without their argument checks
void gh_launch_strand_midpoints(int S, int L, const float* origins, const float* dirs, float* xyz, cudaStream_t stream);
void gh_launch_strand_backward(int S, int L, const float* d_xyz, float* d_dirs, unsigned int* nan_flag, cudaStream_t stream);
// shared refusals of every capturable entry point (before any launch): debug != 0 and calls while the stage timer is on
// (both synchronise with the host)
int gh_check_capturable(const char* who, int debug);
// the binning capacity argument of the capturable entry points: [0, 2^32)
int gh_check_capacity(const char* who, long long capacity);

// per-thread error message behind gh_last_error(): every extern "C" entry point clears it on entry and
// sets it before returning a GH_E_* code (defined in gh_api.cu).  gh_set_error is its only writer (printf-style,
// returns `code`).
void gh_clear_error();
int gh_set_error(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
// after `n` kernel launches: counts them (gh_count_launches) and returns GH_OK, or GH_E_CUDA with
// "[CUDA ERROR] <who>: <cudaGetErrorString>" if a launch failed
int gh_launch_status(const char* who, int n);
// status of a CUDA runtime call (memset, attribute, event, host API): GH_OK, or GH_E_CUDA with
// "[CUDA ERROR] <who>: <what>: <cudaGetErrorString>"
int gh_cuda_status(const char* who, const char* what, cudaError_t e);

// kernels launched outside gh_api.cu (optimizer, image losses) report themselves to gh_kernel_launch_count()
void gh_count_launches(int n);
