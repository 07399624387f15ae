// extern "C" entry points of libgh_raster.so (see include/gh_rasterizer.h for the contract).
// Orchestration only: argument checks, workspace carving, kernel launches in stream order.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

// per-thread error message shared by every entry point of the library (gh_kernels.h)
static thread_local char g_err[512] = "";
void gh_clear_error() { g_err[0] = 0; }
int gh_set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    std::vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
int gh_cuda_status(const char* who, const char* what, cudaError_t e) {
    return e == cudaSuccess ? GH_OK : gh_set_error(GH_E_CUDA, "[CUDA ERROR] %s: %s: %s", who, what, cudaGetErrorString(e));
}

namespace {

// debug mode mirrors the reference's CHECK_CUDA (auxiliary.h:166-173): sync + report after each stage
#define GH_STAGE(who, stream, debug, what)                                        \
    do {                                                                           \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ == cudaSuccess && (debug)) e__ = cudaStreamSynchronize(stream);    \
        if (e__ != cudaSuccess) return gh_cuda_status(who, what, e__);             \
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

// The read-back of R: one thread copies ctrl into the caller's pinned host slot (mapped into the device's address space
// under unified addressing).  A kernel rather than cudaMemcpyAsync: the copy engine's hand-offs from the tile scan and
// back to emit cost more than the copy itself.
__global__ void gh_ctrl_readback_kernel(const GhCtrl* __restrict__ ctrl, GhCtrl* host) {
    gh_pdl_wait();                                    // ctrl is the tile scan's
    gh_pdl_trigger();
    *host = *ctrl;
}

}  // namespace

void gh_count_launches(int n) { g_launches.fetch_add((unsigned long long)n); }

int gh_launch_status(const char* who, int n) {
    gh_count_launches(n);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GH_OK : gh_set_error(GH_E_CUDA, "[CUDA ERROR] %s: %s", who, cudaGetErrorString(e));
}

// The read-back target of gh_forward_phase1: one pinned slot per host thread (allocated on first use and kept for the
// thread's lifetime; pinned memory is mapped for every device under unified addressing), so that work enqueued behind
// the read-back runs while the host waits for it.
static cudaError_t gh_pinned_ctrl(GhCtrl** out) {
    static thread_local GhCtrl* slot = nullptr;
    const cudaError_t e = slot != nullptr ? cudaSuccess : cudaMallocHost((void**)&slot, sizeof(GhCtrl));
    if (e != cudaSuccess) slot = nullptr;
    *out = slot;
    return e;
}

int gh_check_phase1_bin(const char* who, const GhPhase1Bin& emit)
{
    if (emit.capacity < 0 || emit.capacity > 0xffffffffll)
        return gh_set_error(GH_E_INVALID_ARG, "%s: binning_capacity must lie in [0, 2^32)", who);
    if (emit.buffer == nullptr && emit.capacity != 0)
        return gh_set_error(GH_E_INVALID_ARG, "%s: binning_capacity given without a binning_buffer", who);
    if (emit.buffer != nullptr && emit.emitted == nullptr)
        return gh_set_error(GH_E_INVALID_ARG, "%s: a binning_buffer needs the `emitted` output", who);
    return GH_OK;
}

int gh_forward_phase1(const char* who, int P, int width, int height, char* geom_buffer, char* img_buffer, int* num_rendered,
                      int* max_tile_len, int debug, cudaStream_t stream, const GhPhase1Bin& emit, GhBinLaunch launch,
                      const void* bin)
{
    if (emit.emitted) *emit.emitted = 0;
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    if ((unsigned long long)gx * gx * gy >= (1ull << 32))      // exactness bound of the tile enumeration (gh_warp_rects)
        return gh_set_error(GH_E_INVALID_ARG, "%s: image too large (tile grid gx * gx * gy must stay below 2^32)", who);
    GhCtrl* h = nullptr;
    int rc = gh_cuda_status(who, "cudaMallocHost(read-back slot)", gh_pinned_ctrl(&h));
    if (rc != GH_OK) return rc;
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    // ctrl + tile histogram are contiguous: one memset
    rc = gh_cuda_status(who, "memset(tile histogram)", cudaMemsetAsync(img.ctrl, 0, 256 + gh_align_up((size_t)T * 4, 256), stream));
    if (rc != GH_OK) return rc;
    launch(bin, geom, img, gx, gy);
    GH_STAGE(who, stream, debug, "preprocess");
    {
        GhStageTimer t(GH_ST_TILE_SCAN, stream);
        gh_launch_tile_scan(T, img, stream);
        g_launches += 1;
    }
    GH_STAGE(who, stream, debug, "tile scan");
    cudaEvent_t ready = nullptr;
    rc = gh_cuda_status(who, "create the read-back event", cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    if (rc == GH_OK) {
        gh_launch_pdl(gh_ctrl_readback_kernel, 1, 1, 0, stream, img.ctrl, h);
        rc = gh_launch_status(who, 1);
    }
    if (rc == GH_OK) rc = gh_cuda_status(who, "record the read-back event", cudaEventRecord(ready, stream));
    if (rc == GH_OK && emit.buffer != nullptr) {
        // emit goes in behind the read-back: it runs while the host wakes up and prepares the second phase.  It reads R
        // from ctrl and writes nothing when the buffer is too small (the host then takes the exact-size path).
        GhStageTimer t(GH_ST_EMIT, stream);
        const unsigned int cap = (unsigned int)emit.capacity;
        gh_launch_emit(P, emit.radii, geom, img, GhBinWS::carve(emit.buffer, (size_t)cap), cap, gx, gy, stream);
        rc = gh_launch_status(who, 1);
    }
    if (rc == GH_OK) rc = gh_cuda_status(who, "read back num_rendered", cudaEventSynchronize(ready));
    if (ready) cudaEventDestroy(ready);
    if (rc != GH_OK) return rc;
    if (emit.buffer != nullptr) GH_STAGE(who, stream, debug, "emit");
    const GhCtrl hc = *h;
    *num_rendered = (int)hc.num_rendered;
    if (max_tile_len) *max_tile_len = (int)hc.max_tile_len;
    if (hc.err_flags & GH_ERR_PREFILTERED)
        return gh_set_error(GH_E_PREFILTERED, "Point is filtered although prefiltered is set. This shouldn't happen!");
    if (emit.buffer != nullptr) *emit.emitted = ((long long)hc.num_rendered <= emit.capacity) ? 1 : 0;
    return GH_OK;
}

int gh_check_capturable(const char* who, int debug)
{
    if (debug != 0) return gh_set_error(GH_E_INVALID_ARG, "%s: debug mode synchronises after every stage and cannot be captured", who);
    if (g_timing.load()) return gh_set_error(GH_E_INVALID_ARG, "%s: the stage timer synchronises after every stage; disable it (gh_stage_timing_enable(0))", who);
    return GH_OK;
}

int gh_check_capacity(const char* who, long long capacity)
{
    if (capacity < 0 || capacity > 0xffffffffll) return gh_set_error(GH_E_INVALID_ARG, "%s: capacity must lie in [0, 2^32)", who);
    return GH_OK;
}

int gh_forward_phase1_capturable(const char* who, int P, int width, int height, int* radii, char* geom_buffer,
                                 char* img_buffer, char* binning_buffer, long long capacity, unsigned int* status,
                                 unsigned int* num_rendered_out, cudaStream_t stream, GhBinLaunch launch, const void* bin)
{
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    if ((unsigned long long)gx * gx * gy >= (1ull << 32))      // exactness bound of the tile enumeration (gh_warp_rects)
        return gh_set_error(GH_E_INVALID_ARG, "%s: image too large (tile grid gx * gx * gy must stay below 2^32)", who);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    int rc = gh_cuda_status(who, "memset(tile histogram)", cudaMemsetAsync(img.ctrl, 0, 256 + gh_align_up((size_t)T * 4, 256), stream));
    if (rc != GH_OK) return rc;
    launch(bin, geom, img, gx, gy);
    gh_launch_tile_scan(T, img, stream);
    gh_launch_capacity_guard(P, radii, T, img, (unsigned int)capacity, status, num_rendered_out, stream);
    gh_launch_emit(P, radii, geom, img, GhBinWS::carve(binning_buffer, (size_t)capacity), (unsigned int)capacity, gx, gy, stream);
    return gh_launch_status(who, 3);
}

extern "C" {

int gh_abi_version(void) { return 6; }

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
    gh_clear_error();
    if (P < 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_workspace_sizes: bad P/width/height");
    int gx, gy; gh_tile_grid(width, height, gx, gy);
    if (geom_bytes) *geom_bytes = GhGeomWS::bytes((size_t)P);
    if (img_bytes) *img_bytes = GhImgWS::bytes((size_t)width * height, (size_t)gx * gy);
    return GH_OK;
}

int gh_binning_workspace_size(long long R, size_t* binning_bytes)
{
    gh_clear_error();
    if (R < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_binning_workspace_size: negative R");
    if (binning_bytes) *binning_bytes = GhBinWS::bytes((size_t)R);
    return GH_OK;
}

int gh_backward_det_workspace_size(int P, long long R, size_t* bytes)
{
    gh_clear_error();
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
    char* binning_buffer, long long binning_capacity,
    int* num_rendered, int* max_tile_len, int* emitted, int debug, gh_stream_t stream_)
{
    (void)D; (void)M; (void)means2D_precomp; (void)shs; (void)cam_pos;
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (P <= 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_preprocess: P, width, height must be positive");
    if (colors_precomp == nullptr)
        return gh_set_error(GH_E_NO_COLORS, "For non-RGB, provide precomputed Gaussian colors!");
    if (!means3D || !opacities || !viewmatrix || !projmatrix || !radii || !geom_buffer || !img_buffer || !num_rendered)
        return gh_set_error(GH_E_INVALID_ARG, "gh_forward_preprocess: missing mandatory pointer");
    if (conic_precomp == nullptr && cov3D_precomp == nullptr && (scales == nullptr || rotations == nullptr))
        return gh_set_error(GH_E_INVALID_ARG, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (rotations && ((size_t)rotations & 15)) return gh_set_error(GH_E_INVALID_ARG, "rotations must be 16-byte aligned");
    if (((size_t)colors_precomp & 7)) return gh_set_error(GH_E_INVALID_ARG, "colors_precomp must be 8-byte aligned");
    const GhPhase1Bin emit{radii, binning_buffer, binning_capacity, emitted};
    const int rc = gh_check_phase1_bin("gh_forward_preprocess", emit);
    if (rc != GH_OK) return rc;
    return gh_forward_phase1("gh_forward_preprocess", P, width, height, geom_buffer, img_buffer, num_rendered, max_tile_len,
                             debug, stream, emit, [&](const GhGeomWS& geom, const GhImgWS& img, int gx, int gy) {
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
    int num_rendered, int max_tile_len, int emitted, float* out_color, int flags, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    const int debug = flags & GH_FLAG_DEBUG;
    gh_clear_error();
    if (P <= 0 || width <= 0 || height <= 0 || num_rendered < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_forward_render: bad sizes");
    if (!background || !colors_precomp || !radii || !geom_buffer || !img_buffer || !out_color || (num_rendered > 0 && !binning_buffer))
        return gh_set_error(GH_E_INVALID_ARG, "gh_forward_render: missing mandatory pointer");
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    GhBinWS bin = GhBinWS::carve(binning_buffer, (size_t)num_rendered);

    if (num_rendered > 0) {
        if (!emitted) {
            GhStageTimer t(GH_ST_EMIT, stream);
            gh_launch_emit(P, radii, geom, img, bin, (unsigned int)num_rendered, gx, gy, stream);
            g_launches += 1;
        }
        GH_STAGE("gh_forward_render", stream, debug, "emit");
        {
            GhStageTimer t(GH_ST_TILE_SORT, stream);
            g_launches += gh_launch_tile_sort(T, (unsigned int)max_tile_len, (long long)num_rendered, img, bin, stream);
        }
        GH_STAGE("gh_forward_render", stream, debug, "tile sort");
    }
    {
        GhStageTimer t(GH_ST_BLEND_FWD, stream);
        gh_launch_blend_forward(width, height, gx, gy, geom, img, bin, colors_precomp, background, out_color,
                                P, (flags & GH_FLAG_ZERO_RECORDS) != 0, stream);
        g_launches += 1;
    }
    GH_STAGE("gh_forward_render", stream, debug, "blend forward");
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
    int flags, gh_stream_t stream_, char* det_buffer, size_t det_bytes)
{
    (void)D; (void)M; (void)shs; (void)campos; (void)dL_dsh;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int debug = flags & GH_FLAG_DEBUG;
    gh_clear_error();
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
        if (e != cudaSuccess) return gh_cuda_status("gh_backward", "memset(accumulation records)", e);
    }
    if (R == 0) {
        // nothing was rendered: every gradient is zero (P * floats-per-row each)
        struct { float* p; size_t n; } z[] = {{dL_dmean2D, 3}, {dL_dconic, 4}, {dL_dopacity, 1}, {dL_dcolor, GH_NUM_CHANNELS},
                                              {dL_dmean3D, 3}, {dL_dcov3D, 6}, {dL_dscale, 3}, {dL_drot, 4}};
        for (auto& b : z)
            if (b.p) {
                cudaError_t e = cudaMemsetAsync(b.p, 0, (size_t)P * b.n * sizeof(float), stream);
                if (e != cudaSuccess) return gh_cuda_status("gh_backward", "memset(gradients)", e);
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
            if (e != cudaSuccess) return gh_cuda_status("gh_backward", "read back the row count", e);
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
        if (!(flags & GH_FLAG_RECORDS_ZEROED)) {       // otherwise the forward's blend cleared them
            cudaError_t e = cudaMemsetAsync(geom.acc16, 0, (size_t)P * 64, stream);
            if (e != cudaSuccess) return gh_cuda_status("gh_backward", "memset(accumulation records)", e);
        }
        gh_launch_blend_backward(width, height, gx, gy, geom, img, bin, colors_precomp, background, dL_dpix, stream);
        g_launches += 1;
        if (conic_precomp != nullptr && !keep_records) {   // otherwise the geometry backward unpacks the records itself
            gh_launch_unpack_grads(P, geom, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
                                   dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, stream);
            g_launches += 1;
        }
    }
    GH_STAGE("gh_backward", stream, debug, "blend backward");
    if (conic_precomp == nullptr && R > 0) {   // reference: geometry backward is a no-op when the conic was supplied
        GhStageTimer t(GH_ST_PREPROCESS_BWD, stream);
        gh_launch_preprocess_backward(P, means3D, radii, scales, scale_modifier, rotations, cov3D_precomp,
                                      conic_precomp, viewmatrix, projmatrix, width, height, tan_fovx, tan_fovy,
                                      geom.acc16, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
                                      dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, stream);
        g_launches += 1;
    }
    GH_STAGE("gh_backward", stream, debug, "preprocess backward");
    return GH_OK;
}

int gh_forward_render_capturable(
    int P, int width, int height, long long capacity,
    const float* background, const float* colors_precomp,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    float* out_color, int flags, gh_stream_t stream_)
{
    const char* who = "gh_forward_render_capturable";
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_check_capturable(who, flags & GH_FLAG_DEBUG);
    if (rc == GH_OK) rc = gh_check_capacity(who, capacity);
    if (rc != GH_OK) return rc;
    if (P <= 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: bad sizes", who);
    if (!background || !colors_precomp || !geom_buffer || !binning_buffer || !img_buffer || !out_color)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    GhBinWS bin = GhBinWS::carve(binning_buffer, (size_t)capacity);
    const int n = gh_launch_tile_sort_capturable(T, (unsigned int)capacity, img, bin, stream);
    gh_launch_blend_forward(width, height, gx, gy, geom, img, bin, colors_precomp, background, out_color,
                            P, (flags & GH_FLAG_ZERO_RECORDS) != 0, stream);
    return gh_launch_status(who, n + 1);
}

int gh_backward_capturable(
    int P, int width, int height, long long capacity,
    const float* background, const float* colors_precomp, const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    const float* dL_dpix, int flags, gh_stream_t stream_, char* det_buffer, size_t det_bytes)
{
    const char* who = "gh_backward_capturable";
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_check_capturable(who, flags & GH_FLAG_DEBUG);
    if (rc == GH_OK) rc = gh_check_capacity(who, capacity);
    if (rc != GH_OK) return rc;
    if (P <= 0 || width <= 0 || height <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: bad sizes", who);
    if (det_buffer == nullptr && det_bytes != 0)
        return gh_set_error(GH_E_INVALID_ARG, "%s: det_bytes given without a det_buffer", who);
    if (det_buffer != nullptr && det_bytes < GhDetWS::bytes((size_t)P, (size_t)capacity))
        return gh_set_error(GH_E_INVALID_ARG, "%s: det_buffer smaller than gh_backward_det_workspace_size(P, capacity)", who);
    if (!background || !colors_precomp || !radii || !geom_buffer || !binning_buffer || !img_buffer || !dL_dpix)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
    if (((size_t)colors_precomp & 7)) return gh_set_error(GH_E_INVALID_ARG, "colors_precomp must be 8-byte aligned");
    int gx, gy; const int T = gh_tile_grid(width, height, gx, gy);
    GhGeomWS geom = GhGeomWS::carve(geom_buffer, (size_t)P);
    GhImgWS img = GhImgWS::carve(img_buffer, (size_t)width * height, (size_t)T);
    GhBinWS bin = GhBinWS::carve(binning_buffer, (size_t)capacity);
    // no R == 0 branch: an empty (or overflowed, see gh_launch_capacity_guard) frame has no instance in any tile, and
    // both variants then leave zero records
    if (det_buffer != nullptr) {
        // deterministic: the row offsets come from the radii, so off[P] = R <= capacity rows
        GhDetWS det = GhDetWS::carve(det_buffer, (size_t)P, (size_t)capacity);
        const int n = gh_launch_det_offsets(P, gx, gy, radii, geom, det, stream);
        gh_launch_blend_backward_det(width, height, gx, gy, radii, geom, img, bin, det, colors_precomp, background, dL_dpix, stream);
        gh_launch_det_gather(P, geom, det, stream);
        return gh_launch_status(who, n + 2);
    }
    if (!(flags & GH_FLAG_RECORDS_ZEROED)) {
        rc = gh_cuda_status(who, "memset(accumulation records)", cudaMemsetAsync(geom.acc16, 0, (size_t)P * 64, stream));
        if (rc != GH_OK) return rc;
    }
    gh_launch_blend_backward(width, height, gx, gy, geom, img, bin, colors_precomp, background, dL_dpix, stream);
    return gh_launch_status(who, 1);
}

int gh_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    unsigned char* present, gh_stream_t stream_)
{
    (void)projmatrix;
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (P < 0) return gh_set_error(GH_E_INVALID_ARG, "gh_mark_visible: negative P");
    if (P == 0) return GH_OK;
    if (!means3D || !viewmatrix || !present) return gh_set_error(GH_E_INVALID_ARG, "gh_mark_visible: missing pointer");
    gh_launch_mark_visible(P, means3D, viewmatrix, reinterpret_cast<bool*>(present), stream);
    GH_STAGE("gh_mark_visible", stream, 0, "mark visible");
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
    gh_clear_error();
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
    if (e != cudaSuccess) return gh_cuda_status("gh_debug_export", "copy", e);
    GH_STAGE("gh_debug_export", stream, 0, "debug export");
    return GH_OK;
}

}  // extern "C"
