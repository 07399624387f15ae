// The evaluation SSIM and PSNR of B image pairs (SRC/metrics.py, SRC/utils/loss_utils.py:72-121 with size_average,
// SRC/utils/image_utils.py:17-19), forward only:
//     ssim = mean over 3 H W of ssim_map(img1, img2)      (11x11 Gaussian window, sigma 1.5, zero padding 5)
//     psnr = 20 log10(1 / sqrt(mse)),  mse = mean over 3 H W of (img1 - img2)^2
// Each image is float32 or uint8 (x / 255 rounded as torchvision's to_tensor rounds it), optionally clamped to [0, 1],
// optionally multiplied by a per-pair (1,H,W) mask.  Two launches:
//     gh_ssim_tile_kernel    one 32x32 tile of one pair per CTA (grid: tiles x tiles x B): separable window over shared
//                            memory, the per-pixel SSIM expression of the training loss (gh_image_math.cuh; its
//                            every-operation-rounded form), the squared differences; per-CTA sums in double, added in CTA order by the pair's last CTA
//     gh_ssim_finish_kernel  one thread per pair: the means, the PSNR, the strided outputs
// Pair i reads only its own images and writes only its own workspace slots, so its result does not depend on B.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_image_math.cuh"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_ST 32                       // tile edge (pixels); 256 threads, 4 pixels each
#define GH_SR GH_SSIM_R                // window radius: 11 taps
#define GH_SH (GH_ST + 2 * GH_SR)      // halo tile edge: 42
#define GH_SXS (GH_SH + 1)             // row stride of the halo array (float2): conflict-free column walks
#define GH_SHS (GH_ST + 1)             // row stride of the horizontally filtered arrays
#define GH_SITEMS (GH_SH * (GH_ST / 8))   // horizontal work items: one halo row x 8 output columns = 168

// per pair, in the workspace: GH_SS_SLOTS doubles of sums (ssim, squared error, ticket), then 2 per-CTA slots per tile
enum { GH_SS_SSIM = 0, GH_SS_SE = 1, GH_SS_TICKET = 2, GH_SS_SLOTS = 4 };

struct GhSsimWindow { float g[11]; };

struct GhSsimArgs {
    int W, H;
    const void* img1; long long stride1;
    const void* img2; long long stride2;
    const float* mask; long long mask_stride;
    unsigned flags;
};

// u8: the CTA's table of torchvision's to_tensor, img.float().div(255) (one correctly rounded division per byte value)
__device__ __forceinline__ float gh_ssim_value(const float* p, int i, const float*) { return __ldg(p + i); }
__device__ __forceinline__ float gh_ssim_value(const unsigned char* p, int i, const float* u8) { return u8[__ldg(p + i)]; }
__device__ __forceinline__ float gh_clamp01f(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

template <typename T1, typename T2>
__global__ void __launch_bounds__(256, 3)      // 3 CTAs per SM: up to 80 registers, no spills
gh_ssim_tile_kernel(GhSsimArgs a, GhSsimWindow wnd, double* __restrict__ ws, int tiles)
{
    __shared__ float2 sXY[GH_SH][GH_SXS];            // (x, y) = (img1, img2) after conversion, clamp and mask
    __shared__ float2 sH01[GH_SH][GH_SHS], sH23[GH_SH][GH_SHS];   // row-filtered (x, y), (x^2, y^2)
    __shared__ float sH4[GH_SH][GH_SHS];             // row-filtered x y
    __shared__ float s_u8[256];                      // byte value -> x / 255
    const int W = a.W, H = a.H, plane = W * H;       // B 3 H W < 2^31: checked by the host entry point
    const int pair = blockIdx.z;
    const T1* img1 = static_cast<const T1*>(a.img1) + (long long)pair * a.stride1;
    const T2* img2 = static_cast<const T2*>(a.img2) + (long long)pair * a.stride2;
    const float* mask = a.mask ? a.mask + (long long)pair * a.mask_stride : nullptr;
    const bool c1 = a.flags & GH_SSIM_CLAMP_IMG1, c2 = a.flags & GH_SSIM_CLAMP_IMG2, cm = a.flags & GH_SSIM_CLAMP_MASK;
    const int tx0 = blockIdx.x * GH_ST, ty0 = blockIdx.y * GH_ST;
    const int tid = threadIdx.x;
    double a_ssim = 0.0, a_se = 0.0;
    s_u8[tid] = __fdiv_rn((float)tid, 255.f);        // (published by the first __syncthreads below)
    for (int c = 0; c < 3; c++) {
        __syncthreads();
        {   // halo load: warp w takes rows w, w+8, ...; zeros outside the image (F.conv2d padding=5)
            const int lane = tid & 31, warp = tid >> 5;
            const T1* p1 = img1 + c * plane;
            const T2* p2 = img2 + c * plane;
#pragma unroll
            for (int j = 0; j < 6; j++) {
                const int hy = warp + 8 * j, gy = ty0 + hy - GH_SR;
                const bool rowok = hy < GH_SH && gy >= 0 && gy < H;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int hx = lane + 32 * h, gx = tx0 + hx - GH_SR;
                    if (hy >= GH_SH || hx >= GH_SH) continue;
                    float x = 0.f, y = 0.f;
                    if (rowok && gx >= 0 && gx < W) {
                        const int q = gy * W + gx;
                        x = gh_ssim_value(p1, q, s_u8);
                        y = gh_ssim_value(p2, q, s_u8);
                        if (c1) x = gh_clamp01f(x);
                        if (c2) y = gh_clamp01f(y);
                        if (mask) {
                            float m = __ldg(mask + q);
                            if (cm) m = gh_clamp01f(m);
                            x = __fmul_rn(x, m);
                            y = __fmul_rn(y, m);
                        }
                    }
                    sXY[hy][hx] = make_float2(x, y);
                }
            }
        }
        __syncthreads();
        if (tid < GH_SITEMS) {                               // horizontal pass: row r, output columns 8 gq .. 8 gq + 7
            const int r = tid % GH_SH, gq = tid / GH_SH;
            float2 s01[8], s23[8];
            float s4[8];
#pragma unroll
            for (int o = 0; o < 8; o++) { s01[o] = make_float2(0.f, 0.f); s23[o] = make_float2(0.f, 0.f); s4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < 18; k++) {
                const float2 v = sXY[r][8 * gq + k];
                const float sx = __fmul_rn(v.x, v.x), sy = __fmul_rn(v.y, v.y), xy = __fmul_rn(v.x, v.y);
#pragma unroll
                for (int o = 0; o < 8; o++) {
                    if (k - o >= 0 && k - o <= 10) {         // taps in window order: one rounding per tap
                        const float gk = wnd.g[k - o];
                        s01[o].x = __fmaf_rn(gk, v.x, s01[o].x);
                        s01[o].y = __fmaf_rn(gk, v.y, s01[o].y);
                        s23[o].x = __fmaf_rn(gk, sx, s23[o].x);
                        s23[o].y = __fmaf_rn(gk, sy, s23[o].y);
                        s4[o] = __fmaf_rn(gk, xy, s4[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < 8; o++) { sH01[r][8 * gq + o] = s01[o]; sH23[r][8 * gq + o] = s23[o]; sH4[r][8 * gq + o] = s4[o]; }
        }
        __syncthreads();
        {                                                    // vertical pass: column lx, output rows 4 rg .. 4 rg + 3
            const int lx = tid & 31, rg = tid >> 5;
            float2 m4[4], e4[4];
            float e12_4[4];
#pragma unroll
            for (int o = 0; o < 4; o++) { m4[o] = make_float2(0.f, 0.f); e4[o] = make_float2(0.f, 0.f); e12_4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < 14; k++) {
                const float2 a01 = sH01[4 * rg + k][lx], a23 = sH23[4 * rg + k][lx];
                const float a4 = sH4[4 * rg + k][lx];
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    if (k - o >= 0 && k - o <= 10) {
                        const float gk = wnd.g[k - o];
                        m4[o].x = __fmaf_rn(gk, a01.x, m4[o].x);
                        m4[o].y = __fmaf_rn(gk, a01.y, m4[o].y);
                        e4[o].x = __fmaf_rn(gk, a23.x, e4[o].x);
                        e4[o].y = __fmaf_rn(gk, a23.y, e4[o].y);
                        e12_4[o] = __fmaf_rn(gk, a4, e12_4[o]);
                    }
                }
            }
            const int px = tx0 + lx;
#pragma unroll
            for (int o = 0; o < 4; o++) {
                const int py = ty0 + 4 * rg + o;
                if (px < W && py < H) {
                    a_ssim += (double)gh_ssim_pixel<true>(m4[o].x, m4[o].y, e4[o].x, e4[o].y, e12_4[o]).S;
                    const float2 v = sXY[4 * rg + o + GH_SR][lx + GH_SR];
                    const double d = (double)__fsub_rn(v.x, v.y);   // the float32 difference, squared exactly
                    a_se += d * d;
                }
            }
        }
    }
    double v[2] = {a_ssim, a_se};
    double* sums = ws + (size_t)pair * GH_SS_SLOTS;
    double* part = ws + (size_t)gridDim.z * GH_SS_SLOTS + (size_t)pair * 2 * tiles;
    gh_block_sum_fixed<2>(v, part, sums, {GH_SS_SSIM, GH_SS_SE}, GH_SS_TICKET);
}

// one thread per pair: ssim = sum / (3 H W); psnr = 20 log10(1 / sqrt(mse)) in double (mse 0 -> inf, as the reference)
__global__ void __launch_bounds__(128)
gh_ssim_finish_kernel(int B, int plane, const double* __restrict__ ws, float* __restrict__ ssim, long long ssim_stride,
                      float* __restrict__ psnr, long long psnr_stride)
{
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= B) return;
    const double n = 3.0 * (double)plane;
    const double* s = ws + (size_t)i * GH_SS_SLOTS;
    ssim[(long long)i * ssim_stride] = (float)(s[GH_SS_SSIM] / n);
    if (psnr) psnr[(long long)i * psnr_stride] = (float)(20.0 * log10(1.0 / sqrt(s[GH_SS_SE] / n)));
}

size_t gh_ssim_tiles(int W, int H) { return (size_t)((W + GH_ST - 1) / GH_ST) * (size_t)((H + GH_ST - 1) / GH_ST); }

size_t gh_ssim_ws_bytes(int B, int W, int H) { return (size_t)B * (GH_SS_SLOTS + 2 * gh_ssim_tiles(W, H)) * sizeof(double); }

int gh_ssim_check_size(const char* who, int B, int W, int H)
{
    if (B <= 0 || W <= 0 || H <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: bad B/width/height (%d, %d, %d)", who, B, W, H);
    if (B > 65535) return gh_set_error(GH_E_INVALID_ARG, "%s: B = %d pairs, at most 65535 per call", who, B);
    if ((long long)B * 3 * W * H > 0x7fffffffll)     // 32-bit element offsets inside the kernel
        return gh_set_error(GH_E_INVALID_ARG, "%s: B * 3 * H * W = %lld exceeds 2^31 - 1", who, (long long)B * 3 * W * H);
    return GH_OK;
}

template <typename T1, typename T2>
void gh_ssim_launch(const GhSsimArgs& a, const GhSsimWindow& w, double* ws, int B, cudaStream_t stream)
{
    const dim3 grid((a.W + GH_ST - 1) / GH_ST, (a.H + GH_ST - 1) / GH_ST, B);
    gh_ssim_tile_kernel<T1, T2><<<grid, 256, 0, stream>>>(a, w, ws, (int)gh_ssim_tiles(a.W, a.H));
}

}  // namespace

extern "C" int gh_eval_ssim_workspace_size(int B, int width, int height, size_t* bytes)
{
    gh_clear_error();
    const int rc = gh_ssim_check_size("gh_eval_ssim_workspace_size", B, width, height);
    if (rc != GH_OK) return rc;
    if (!bytes) return gh_set_error(GH_E_INVALID_ARG, "gh_eval_ssim_workspace_size: bytes is NULL");
    *bytes = gh_ssim_ws_bytes(B, width, height);
    return GH_OK;
}

extern "C" int gh_eval_ssim(int B, int width, int height, const void* img1, int dtype1, long long stride1,
                            const void* img2, int dtype2, long long stride2, const float* mask, long long mask_stride,
                            unsigned flags, float* ssim, long long ssim_stride, float* psnr, long long psnr_stride,
                            void* workspace, size_t workspace_bytes, int debug, gh_stream_t stream_)
{
    static const char* who = "gh_eval_ssim";
    gh_clear_error();
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = gh_ssim_check_size(who, B, width, height);
    if (rc != GH_OK) return rc;
    for (int d : {dtype1, dtype2})
        if (d != GH_DTYPE_FLOAT32 && d != GH_DTYPE_UINT8) return gh_set_error(GH_E_INVALID_ARG, "%s: unknown dtype code %d", who, d);
    if (!img1 || !img2 || !ssim || !workspace)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing image, ssim or workspace pointer", who);
    if (flags & ~(GH_SSIM_CLAMP_IMG1 | GH_SSIM_CLAMP_IMG2 | GH_SSIM_CLAMP_MASK))
        return gh_set_error(GH_E_INVALID_ARG, "%s: unknown flag bits 0x%x", who, flags);
    const long long n3 = 3ll * width * height;
    if (B > 1 && (stride1 < n3 || stride2 < n3 || (mask && mask_stride < (long long)width * height)))
        return gh_set_error(GH_E_INVALID_ARG, "%s: pair strides must not overlap the pairs (>= 3 H W, mask >= H W)", who);
    if ((B - 1) * (stride1 > stride2 ? stride1 : stride2) + n3 > 0x7fffffffll ||
        (mask && (B - 1) * mask_stride + n3 / 3 > 0x7fffffffll))
        return gh_set_error(GH_E_INVALID_ARG, "%s: strided pairs reach beyond 2^31 - 1 elements", who);
    if (B > 1 && (ssim_stride <= 0 || (psnr && psnr_stride <= 0)))
        return gh_set_error(GH_E_INVALID_ARG, "%s: output strides must be positive", who);
    if (((size_t)img1 & 3 && dtype1 == GH_DTYPE_FLOAT32) || ((size_t)img2 & 3 && dtype2 == GH_DTYPE_FLOAT32) ||
        ((size_t)mask & 3) || ((size_t)ssim & 3) || ((size_t)psnr & 3))
        return gh_set_error(GH_E_INVALID_ARG, "%s: float arrays must be 4-byte aligned", who);
    if ((size_t)workspace & 7) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace must be 8-byte aligned", who);
    const size_t need = gh_ssim_ws_bytes(B, width, height);
    if (workspace_bytes < need)
        return gh_set_error(GH_E_INVALID_ARG, "%s: workspace of %zu bytes, %zu needed", who, workspace_bytes, need);
    if (debug && (rc = gh_check_capturable(who, 0)) != GH_OK) return rc;      // debug synchronises: not with the timer on

    GhSsimWindow w;
    gh_ssim_window(w.g);
    const GhSsimArgs a = {width, height, img1, stride1, img2, stride2, mask, mask_stride, flags};
    double* ws = static_cast<double*>(workspace);
    rc = gh_cuda_status(who, "memset(sums)", cudaMemsetAsync(ws, 0, (size_t)B * GH_SS_SLOTS * sizeof(double), stream));
    if (rc != GH_OK) return rc;
    const bool u1 = dtype1 == GH_DTYPE_UINT8, u2 = dtype2 == GH_DTYPE_UINT8;
    if (!u1 && !u2) gh_ssim_launch<float, float>(a, w, ws, B, stream);
    else if (!u1 && u2) gh_ssim_launch<float, unsigned char>(a, w, ws, B, stream);
    else if (u1 && !u2) gh_ssim_launch<unsigned char, float>(a, w, ws, B, stream);
    else gh_ssim_launch<unsigned char, unsigned char>(a, w, ws, B, stream);
    gh_ssim_finish_kernel<<<(B + 127) / 128, 128, 0, stream>>>(B, width * height, ws, ssim, ssim_stride, psnr, psnr_stride);
    rc = gh_launch_status(who, 2);
    if (rc == GH_OK && debug) rc = gh_cuda_status(who, "synchronise (debug)", cudaStreamSynchronize(stream));
    return rc;
}
