// extern "C" entry points of libgh_raster.so (see include/gh_rasterizer.h for the contract).
// Orchestration only: argument checks, workspace carving, kernel launches in stream order.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>

// per-thread error message shared by every entry point of the library (gh_kernels.h)
static thread_local char g_err[512] = "";
void gh_clear_error() { g_err[0] = 0; }
int gh_set_error(int code, const char* msg) {
    std::snprintf(g_err, sizeof(g_err), "%s", msg ? msg : "");
    return code;
}

namespace {

int gh_check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return GH_OK;
    std::snprintf(g_err, sizeof(g_err), "[CUDA ERROR] %s: %s", what, cudaGetErrorString(e));
    return GH_E_CUDA;
}

// debug mode mirrors the reference's CHECK_CUDA (auxiliary.h:166-173): sync + report after each stage
#define GH_STAGE(stream, debug, what)                                             \
    do {                                                                           \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ == cudaSuccess && (debug)) e__ = cudaStreamSynchronize(stream);    \
        if (e__ != cudaSuccess) return gh_check_cuda(e__, what);                   \
    } while (0)

// ---- optional per-stage device timing (bench / roofline only; off by default) -------------------
enum { GH_ST_PREPROCESS = 0, GH_ST_TILE_SCAN, GH_ST_EMIT, GH_ST_TILE_SORT, GH_ST_BLEND_FWD, GH_ST_BLEND_BWD,
       GH_ST_PREPROCESS_BWD, GH_ST_COUNT };
// The only process-wide state of the library: the launch counter (atomic) and the diagnostic stage
// timer (a mutex guards its sums; events are created per stage on the caller's current device, so the
// forward thread, autograd's backward thread and several devices can use it at once).
std::atomic<bool> g_timing{false};
std::mutex g_timing_mu;
double g_stage_ms[GH_ST_COUNT] = {0};
unsigned long long g_stage_calls[GH_ST_COUNT] = {0};
std::atomic<unsigned long long> g_launches{0};     // kernels launched by this library since load

struct GhStageTimer {
    int stage; cudaStream_t stream; unsigned long long l0; bool on;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    GhStageTimer(int st, cudaStream_t s) : stage(st), stream(s), l0(g_launches.load()), on(g_timing.load()) {
        if (on) {
            on = (cudaEventCreate(&ev0) == cudaSuccess) && (cudaEventCreate(&ev1) == cudaSuccess);
            if (on) cudaEventRecord(ev0, stream);
        }
    }
    ~GhStageTimer() {
        if (on && g_launches.load() != l0) {     // a stage that launched nothing (in-kernel tile sort) is not a stage
            cudaEventRecord(ev1, stream);
            cudaEventSynchronize(ev1);
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) {
                std::lock_guard<std::mutex> lk(g_timing_mu);
                g_stage_ms[stage] += ms; g_stage_calls[stage] += 1;
            }
        }
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
};

__global__ void gh_export_keys_kernel(const uint2* __restrict__ ranges, const uint64_t* __restrict__ inst,
                                      unsigned long long* __restrict__ keys, unsigned int* __restrict__ plist)
{
    const uint2 rg = ranges[blockIdx.x];
    for (uint32_t i = rg.x + threadIdx.x; i < rg.y; i += blockDim.x) {
        const uint64_t r = inst[i];
        if (keys) keys[i] = ((unsigned long long)blockIdx.x << 32) | (r >> 32);
        if (plist) plist[i] = (unsigned int)r;
    }
}

__global__ void gh_export_geom_kernel(int P, const GhGeo* __restrict__ geo, float* __restrict__ means2D,
                                      float* __restrict__ conic_opacity)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const GhGeo g = geo[i];
    if (means2D) { means2D[2 * i] = g.x; means2D[2 * i + 1] = g.y; }
    if (conic_opacity) {
        conic_opacity[4 * i + 0] = g.ca; conic_opacity[4 * i + 1] = g.cb;
        conic_opacity[4 * i + 2] = g.cc; conic_opacity[4 * i + 3] = g.op;
    }
}

}  // namespace

void gh_count_launches(int n) { g_launches.fetch_add((unsigned long long)n); }

int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, GhBinLaunch launch, const void* bin)
{
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    if ((unsigned long long)gx * gx * gy >= (1ull << 32)) {    // exactness bound of the tile enumeration (gh_warp_rects)
        std::snprintf(g_err, sizeof(g_err), "%s: image too large (tile grid gx * gx * gy must stay below 2^32)", who);
        return GH_E_INVALID_ARG;
    }
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    // ctrl + tile histogram are contiguous: one memset
    cudaError_t e = cudaMemsetAsync(img.ctrl, 0, 256 + gh_align_up((size_t)T * 4, 256), stream);
    if (e != cudaSuccess) return gh_check_cuda(e, "memset(tile histogram)");
    launch(bin, geom, img, gx, gy);
    GH_STAGE(stream, debug, "preprocess");
    {
        GhStageTimer t(GH_ST_TILE_SCAN, stream);
        gh_launch_tile_scan(T, img, stream);
        g_launches += 1;
    }
    GH_STAGE(stream, debug, "tile scan");
    GhCtrl h;
    e = cudaMemcpyAsync(&h, img.ctrl, sizeof(GhCtrl), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return gh_check_cuda(e, "read back num_rendered");
    *num_rendered = (int)h.num_rendered;
    if (max_tile_len) *max_tile_len = (int)h.max_tile_len;
    if (h.err_flags & GH_ERR_PREFILTERED)
        return gh_set_error(GH_E_PREFILTERED, "Point is filtered although prefiltered is set. This shouldn't happen!");
    return GH_OK;
}

extern "C" {

int gh_abi_version(void) { return 4; }

unsigned long long gh_kernel_launch_count(void) { return g_launches.load(); }

void gh_stage_timing_enable(int on) {
    std::lock_guard<std::mutex> lk(g_timing_mu);
    g_timing.store(on != 0);
    for (int i = 0; i < GH_ST_COUNT; i++) { g_stage_ms[i] = 0.0; g_stage_calls[i] = 0; }
}

int gh_stage_timing_read(double* ms_sum, unsigned long long* calls, int capacity) {
    std::lock_guard<std::mutex> lk(g_timing_mu);
    const int n = capacity < GH_ST_COUNT ? capacity : GH_ST_COUNT;
    for (int i = 0; i < n; i++) { if (ms_sum) ms_sum[i] = g_stage_ms[i]; if (calls) calls[i] = g_stage_calls[i]; }
    return GH_ST_COUNT;
}
int gh_num_channels(void) { return GH_NUM_CHANNELS; }
const char* gh_last_error(void) { return g_err; }

int gh_forward_workspace_sizes(int P, int width, int height, size_t* geom_bytes, size_t* img_bytes)
{
    if (P < 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_workspace_sizes: bad P/width/height");
    int gx, gy; gh_tile_grid(width, height, gx, gy);
    if (geom_bytes) *geom_bytes = GhGeomWS::bytes((size_t)P);
    if (img_bytes) *img_bytes = GhImgWS::bytes((size_t)width * height, (size_t)gx * gy);
    return GH_OK;
}

int gh_binning_workspace_size(long long R, size_t* binning_bytes)
{
    if (R < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_binning_workspace_size: negative R");
    if (binning_bytes) *binning_bytes = GhBinWS::bytes((size_t)R);
    return GH_OK;
}

int gh_backward_det_workspace_size(int P, long long R, size_t* bytes)
{
    if (P < 0 || R < 0 || R > 0xffffffffll) return gh_set_error(GH_E_INVALID_ARG, "gh_backward_det_workspace_size: bad P/R");
    if (bytes) *bytes = GhDetWS::bytes((size_t)P, (size_t)R);
    return GH_OK;
}

int gh_forward_preprocess(
    int P, int D, int M, int width, int height,
    const float* means3D, const float* means2D_precomp, const float* shs,
    const float* colors_precomp, const float* opacities,
    const float* scales, float scale_modifier, const float* rotations,
    const float* cov3D_precomp, const float* conic_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
    float tan_fovx, float tan_fovy, int prefiltered,
    int* radii, char* geom_buffer, char* img_buffer,
    int* num_rendered, int* max_tile_len, int debug, gh_stream_t stream_)
{
    (void)D; (void)M; (void)means2D_precomp; (void)shs; (void)cam_pos;
    cudaStream_t stream = (cudaStream_t)stream_;
    g_err[0] = 0;
    if (P <= 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_preprocess: P, width, height must be positive");
    if (colors_precomp == nullptr)
        return gh_set_error(GH_E_NO_COLORS, "For non-RGB, provide precomputed Gaussian colors!");
    if (!means3D || !opacities || !viewmatrix || !projmatrix || !radii || !geom_buffer || !img_buffer || !num_rendered)
        return gh_set_error(GH_E_INVALID_ARG, "gh_forward_preprocess: missing mandatory pointer");
    if (conic_precomp == nullptr && cov3D_precomp == nullptr && (scales == nullptr || rotations == nullptr))
        return gh_set_error(GH_E_INVALID_ARG, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (rotations && ((size_t)rotations & 15)) return gh_set_error(GH_E_INVALID_ARG, "rotations must be 16-byte aligned");
    if (((size_t)colors_precomp & 7)) return gh_set_error(GH_E_INVALID_ARG, "colors_precomp must be 8-byte aligned");
    return gh_forward_phase1("gh_forward_preprocess", P, width, height, geom_buffer, img_buffer, num_rendered, max_tile_len,
                             debug, stream, [&](const GhGeomWS& geom, const GhImgWS& img, int gx, int gy) {
        GhStageTimer t(GH_ST_PREPROCESS, stream);
        gh_launch_preprocess(P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp,
                             conic_precomp, viewmatrix, projmatrix, width, height, tan_fovx, tan_fovy,
                             radii, geom, img, gx, gy, prefiltered, stream);
        g_launches += 1;
    });
}

int gh_forward_render(
    int P, int width, int height,
    const float* background, const float* colors_precomp, const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    int num_rendered, int max_tile_len, float* out_color, int debug, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    g_err[0] = 0;
    if (P <= 0 || width <= 0 || height <= 0 || num_rendered < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_render: bad sizes");
    if (!background || !colors_precomp || !radii || !geom_buffer || !img_buffer || !out_color || (num_rendered > 0 && !binning_buffer))
        return gh_set_error(GH_E_INVALID_ARG, "gh_forward_render: missing mandatory pointer");
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    GhBinWS bin = GhBinWS::carve(binning_buffer, (size_t)num_rendered);

    if (num_rendered > 0) {
        {
            GhStageTimer t(GH_ST_EMIT, stream);
            gh_launch_emit(P, radii, geom, img, bin, gx, gy, stream);
            g_launches += 1;
        }
        GH_STAGE(stream, debug, "emit");
        {
            GhStageTimer t(GH_ST_TILE_SORT, stream);
            g_launches += gh_launch_tile_sort(T, (unsigned int)max_tile_len, (long long)num_rendered, img, bin, stream);
        }
        GH_STAGE(stream, debug, "tile sort");
    }
    {
        GhStageTimer t(GH_ST_BLEND_FWD, stream);
        gh_launch_blend_forward(width, height, gx, gy, geom, img, bin, colors_precomp, background, out_color, stream);
        g_launches += 1;
    }
    GH_STAGE(stream, debug, "blend forward");
    return GH_OK;
}

int gh_backward(
    int P, int D, int M, int R, int width, int height,
    const float* background,
    const float* means3D, const float* shs, const float* colors_precomp,
    const float* scales, float scale_modifier, const float* rotations,
    const float* cov3D_precomp, const float* conic_precomp,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    const float* dL_dpix,
    float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
    float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
    int debug, gh_stream_t stream_, char* det_buffer, size_t det_bytes)
{
    (void)D; (void)M; (void)shs; (void)campos; (void)dL_dsh;
    cudaStream_t stream = (cudaStream_t)stream_;
    g_err[0] = 0;
    if (P <= 0 || width <= 0 || height <= 0 || R < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_backward: bad sizes");
    if (det_buffer == nullptr && det_bytes != 0)
        return gh_set_error(GH_E_INVALID_ARG, "gh_backward: det_bytes given without a det_buffer");
    if (det_buffer != nullptr && det_bytes < GhDetWS::bytes((size_t)P, (size_t)R))
        return gh_set_error(GH_E_INVALID_ARG, "gh_backward: det_buffer smaller than gh_backward_det_workspace_size");
    // conic supplied + all four 2-D gradient outputs NULL: leave the accumulation records in the geometry workspace
    const bool keep_records = (conic_precomp != nullptr) && !dL_dmean2D && !dL_dconic && !dL_dopacity && !dL_dcolor;
    if (!background || !means3D || !colors_precomp || !viewmatrix || !projmatrix || !radii ||
        !geom_buffer || !img_buffer || !dL_dpix || (R > 0 && !binning_buffer) ||
        (!keep_records && (!dL_dmean2D || !dL_dconic || !dL_dopacity || !dL_dcolor)))
        return gh_set_error(GH_E_INVALID_ARG, "gh_backward: missing mandatory pointer");
    if (conic_precomp == nullptr) {
        if (!dL_dmean3D || !dL_dcov3D) return gh_set_error(GH_E_INVALID_ARG, "gh_backward: dL_dmean3D/dL_dcov3D required");
        if (cov3D_precomp == nullptr && (!scales || !rotations || !dL_dscale || !dL_drot))
            return gh_set_error(GH_E_INVALID_ARG, "gh_backward: scales/rotations and their gradient buffers required");
        if (rotations && ((size_t)rotations & 15)) return gh_set_error(GH_E_INVALID_ARG, "rotations must be 16-byte aligned");
        if (dL_drot && ((size_t)dL_drot & 15)) return gh_set_error(GH_E_INVALID_ARG, "dL_drot must be 16-byte aligned");
    }
    if (((size_t)colors_precomp & 7)) return gh_set_error(GH_E_INVALID_ARG, "colors_precomp must be 8-byte aligned");
    if (((size_t)dL_dconic & 15)) return gh_set_error(GH_E_INVALID_ARG, "dL_dconic must be 16-byte aligned");
    if (((size_t)dL_dcolor & 7)) return gh_set_error(GH_E_INVALID_ARG, "dL_dcolor must be 8-byte aligned");
    if (keep_records && (dL_dmean3D || dL_dcov3D || dL_dscale || dL_drot))
        return gh_set_error(GH_E_INVALID_ARG, "gh_backward: geometry gradients cannot be requested without the 2-D gradient outputs");
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    GhBinWS bin = GhBinWS::carve(binning_buffer, (size_t)R);

    if (R == 0 && keep_records) {
        cudaError_t e = cudaMemsetAsync(geom.acc16, 0, (size_t)P * 64, stream);
        if (e != cudaSuccess) return gh_check_cuda(e, "memset(accumulation records)");
    }
    if (R == 0) {
        // nothing was rendered: every gradient is zero (P * floats-per-row each)
        struct { float* p; size_t n; } z[] = {{dL_dmean2D, 3}, {dL_dconic, 4}, {dL_dopacity, 1}, {dL_dcolor, GH_NUM_CHANNELS},
                                              {dL_dmean3D, 3}, {dL_dcov3D, 6}, {dL_dscale, 3}, {dL_drot, 4}};
        for (auto& b : z)
            if (b.p) {
                cudaError_t e = cudaMemsetAsync(b.p, 0, (size_t)P * b.n * sizeof(float), stream);
                if (e != cudaSuccess) return gh_check_cuda(e, "memset(gradients)");
            }
    }
    if (R > 0 && det_buffer != nullptr) {
        // deterministic path: offsets of the Gaussian-major rows, per-tile rows, fixed-order gather into acc16
        GhStageTimer t(GH_ST_BLEND_BWD, stream);
        GhDetWS det = GhDetWS::carve(det_buffer, (size_t)P, (size_t)R);
        g_launches += gh_launch_det_offsets(P, gx, gy, radii, geom, det, stream);
        if (debug) {
            uint32_t total = 0;
            cudaError_t e = cudaMemcpyAsync(&total, det.off + P, sizeof(total), cudaMemcpyDeviceToHost, stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return gh_check_cuda(e, "read back the row count");
            if (total != (uint32_t)R)
                return gh_set_error(GH_E_INVALID_ARG, "gh_backward: the tile rectangles of radii do not add up to R");
        }
        gh_launch_blend_backward_det(width, height, gx, gy, radii, geom, img, bin, det, colors_precomp, background, dL_dpix, stream);
        gh_launch_det_gather(P, geom, det, stream);
        g_launches += 2;
        if (conic_precomp != nullptr && !keep_records) {
            gh_launch_unpack_grads(P, geom, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
                                   dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, stream);
            g_launches += 1;
        }
    } else if (R > 0) {
        GhStageTimer t(GH_ST_BLEND_BWD, stream);
        cudaError_t e = cudaMemsetAsync(geom.acc16, 0, (size_t)P * 64, stream);
        if (e != cudaSuccess) return gh_check_cuda(e, "memset(accumulation records)");
        gh_launch_blend_backward(width, height, gx, gy, geom, img, bin, colors_precomp, background, dL_dpix, stream);
        g_launches += 1;
        if (conic_precomp != nullptr && !keep_records) {   // otherwise the geometry backward unpacks the records itself
            gh_launch_unpack_grads(P, geom, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
                                   dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, stream);
            g_launches += 1;
        }
    }
    GH_STAGE(stream, debug, "blend backward");
    if (conic_precomp == nullptr && R > 0) {   // reference: geometry backward is a no-op when the conic was supplied
        GhStageTimer t(GH_ST_PREPROCESS_BWD, stream);
        gh_launch_preprocess_backward(P, means3D, radii, scales, scale_modifier, rotations, cov3D_precomp,
                                      conic_precomp, viewmatrix, projmatrix, width, height, tan_fovx, tan_fovy,
                                      geom.acc16, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
                                      dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, stream);
        g_launches += 1;
    }
    GH_STAGE(stream, debug, "preprocess backward");
    return GH_OK;
}

int gh_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    unsigned char* present, gh_stream_t stream_)
{
    (void)projmatrix;
    cudaStream_t stream = (cudaStream_t)stream_;
    g_err[0] = 0;
    if (P < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_mark_visible: negative P");
    if (P == 0) return GH_OK;
    if (!means3D || !viewmatrix || !present) return gh_set_error(GH_E_INVALID_ARG, "gh_mark_visible: missing pointer");
    gh_launch_mark_visible(P, means3D, viewmatrix, reinterpret_cast<bool*>(present), stream);
    GH_STAGE(stream, 0, "mark visible");
    return GH_OK;
}

int gh_debug_export(
    int P, int width, int height, long long R,
    const char* geom_buffer, const char* binning_buffer, const char* img_buffer,
    unsigned long long* keys_sorted, unsigned int* point_list, unsigned int* ranges,
    float* final_T, unsigned int* n_contrib,
    float* depths, float* means2D, float* conic_opacity, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    g_err[0] = 0;
    if (P <= 0 || width <= 0 || height <= 0 || R < 0 || !geom_buffer || !img_buffer)
        return gh_set_error(GH_E_INVALID_ARG, "gh_debug_export: bad arguments");
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    const size_t npix = (size_t)width * height;
    GhGeomWS geom = GhGeomWS::carve(const_cast<char*>(geom_buffer), (size_t)P);
    GhImgWS img = GhImgWS::carve(const_cast<char*>(img_buffer), npix, (size_t)T);
    cudaError_t e = cudaSuccess;
    if (R > 0 && binning_buffer && (keys_sorted || point_list)) {
        GhBinWS bin = GhBinWS::carve(const_cast<char*>(binning_buffer), (size_t)R);
        gh_export_keys_kernel<<<T, 128, 0, stream>>>(img.ranges, bin.inst, keys_sorted, point_list);
    }
    if (ranges && e == cudaSuccess) e = cudaMemcpyAsync(ranges, img.ranges, (size_t)T * 8, cudaMemcpyDeviceToDevice, stream);
    if (final_T && e == cudaSuccess) e = cudaMemcpyAsync(final_T, img.final_T, npix * 4, cudaMemcpyDeviceToDevice, stream);
    if (n_contrib && e == cudaSuccess) e = cudaMemcpyAsync(n_contrib, img.n_contrib, npix * 4, cudaMemcpyDeviceToDevice, stream);
    if (depths && e == cudaSuccess) e = cudaMemcpyAsync(depths, geom.depth, (size_t)P * 4, cudaMemcpyDeviceToDevice, stream);
    if ((means2D || conic_opacity) && e == cudaSuccess)
        gh_export_geom_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, geom.geo, means2D, conic_opacity);
    if (e != cudaSuccess) return gh_check_cuda(e, "debug export");
    GH_STAGE(stream, 0, "debug export");
    return GH_OK;
}

}  // extern "C"
