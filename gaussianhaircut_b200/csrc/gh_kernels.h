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

// scatter (depth|idx) records into their tile buckets
void gh_launch_emit(int P, const int* radii, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                    int gx, int gy, cudaStream_t stream);

// sort every tile bucket by (depth bits, gaussian idx)
// returns the number of kernels launched
int gh_launch_tile_sort(int T, unsigned int max_tile_len, long long R, GhImgWS img, GhBinWS bin, cudaStream_t stream);

void gh_launch_blend_forward(int W, int H, int gx, int gy, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                             const float* features, const float* bg, float* out_color,
                             cudaStream_t stream);

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

// The forward's first phase around its per-Gaussian kernel (gh_forward_preprocess, gh_project_forward_binned): tile grid
// and its bound, workspace carving, ctrl + histogram memset, `bin(geom, img, gx, gy)` (launches the kernel on `stream` and
// counts it), tile scan, read-back of R and the longest tile list.  `who` names the entry point in error messages.
typedef void (*GhBinLaunch)(const void* bin, const GhGeomWS& geom, const GhImgWS& img, int gx, int gy);
int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, GhBinLaunch launch, const void* bin);
template <class F>
int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, const F& bin) {
    return gh_forward_phase1(who, P, width, height, geom_buffer, img_buffer, num_rendered, max_tile_len, debug, stream,
                             [](const void* f, const GhGeomWS& g, const GhImgWS& i, int gx, int gy) { (*static_cast<const F*>(f))(g, i, gx, gy); }, &bin);
}

// per-thread error message behind gh_last_error(): every extern "C" entry point clears it on entry and
// sets it before returning a GH_E_* code (defined in gh_api.cu)
void gh_clear_error();
int gh_set_error(int code, const char* msg);

// kernels launched outside gh_api.cu (optimizer, image losses) report themselves to gh_kernel_launch_count()
void gh_count_launches(int n);
