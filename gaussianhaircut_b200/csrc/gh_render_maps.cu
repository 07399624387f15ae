// The inference side of the raw (10,H,W) image of gh_forward_render: what the reference's render scripts and trainers'
// training_report compute from it with a few dozen full-frame PyTorch kernels, in one pass each.
//   gh_render_maps    the maps SRC/render_gaussians.py:50-68 and SRC/render_strands.py:51-69 write per view: the
//                     orientation angle (SRC/gaussian_renderer/__init__.py:100-105), the masked confidence, and the
//                     bytes torchvision.utils.save_image makes of render, masks, orientation and the two vis_orient
//                     colourings (SRC/utils/image_utils.py:22-37)
//   gh_eval_metrics   one view's numbers of training_report (SRC/train_gaussians.py:254-277, SRC/train_strands.py,
//                     SRC/train_latent_strands.py:235-258): L1, mask L1 or cross entropy, orientation loss, PSNR
// Output channel layout: image 0..2, mask 3..4 (hair, head), dir 5..7, orientation confidence 8, depth 9.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_image_math.cuh"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_MT 256                      // pixels (= threads) per CTA

// save_image's quantisation, x.mul(255).add_(0.5).clamp_(0, 255).to(uint8): a rounded multiply, a rounded add, then
// truncation.  The intrinsics keep the compiler from contracting the pair into an FMA, which rounds once and lands on
// the other side of a byte boundary at ties.  NaN -> 0.
__device__ __forceinline__ unsigned gh_quant_u8(float x)
{
    const float v = __fadd_rn(__fmul_rn(x, 255.f), 0.5f);
    return (unsigned)fminf(fmaxf(v, 0.f), 255.f);
}

// one triangle of vis_orient: clamp(1 - |deg - c| / 45, 0, 1), every operation rounded on its own like the tensor code
__device__ __forceinline__ float gh_vis_tri(float deg, float c)
{
    const float v = __fsub_rn(1.f, __fdiv_rn(fabsf(__fsub_rn(deg, c)), 45.f));
    return fminf(fmaxf(v, 0.f), 1.f);
}

// vis_orient(angle, mask): red (vertical) + green (horizontal) + magenta / teal (diagonals) in BGR, swapped to RGB.
// The integer colour vectors make every product exact, so a channel is the sum of the triangles it contains, in the
// order the reference adds them.
__device__ __forceinline__ void gh_vis_orient(float ang, float mask, float (&rgb)[3])
{
    const float deg = __fmul_rn(ang, 180.f);
    const float red = __fadd_rn(gh_vis_tri(deg, 0.f), gh_vis_tri(deg, 180.f));
    const float green = gh_vis_tri(deg, 90.f), magenta = gh_vis_tri(deg, 45.f), teal = gh_vis_tri(deg, 135.f);
    rgb[0] = __fmul_rn(__fadd_rn(red, magenta), mask);
    rgb[1] = __fmul_rn(__fadd_rn(green, teal), mask);
    rgb[2] = __fmul_rn(__fadd_rn(magenta, teal), mask);
}

// the CTA's `n` staged bytes to dst (4-byte aligned) as 32-bit words; only the last CTA of a map whose size is not a
// multiple of 4 has single bytes left over
__device__ __forceinline__ void gh_store_staged(unsigned char* __restrict__ dst, const unsigned char* s, int n)
{
    const int tid = threadIdx.x, words = n >> 2;
    if (tid < words) reinterpret_cast<unsigned*>(dst)[tid] = reinterpret_cast<const unsigned*>(s)[tid];
    if (tid < (n & 3)) dst[4 * words + tid] = s[4 * words + tid];
}

struct GhMapOutputs {
    float* orient_angle;
    float* orient_conf_masked;
    unsigned char* render_u8;
    unsigned char* hair_mask_u8;
    unsigned char* head_mask_u8;
    unsigned char* orient_u8;
    unsigned char* orient_vis_u8;
    unsigned char* orient_conf_vis_u8;
};

// One pixel per thread; 32 B read (channels 0..6 and 8), up to 20 B written.  The byte maps are staged in shared memory
// so that the 1- and 3-byte pixels leave as coalesced 32-bit words.
__global__ void __launch_bounds__(GH_MT)
gh_render_maps_kernel(int plane, const float* __restrict__ out, GhMapOutputs o)
{
    __shared__ __align__(16) unsigned char s_grey[3][GH_MT];
    __shared__ __align__(16) unsigned char s_rgb[3][3 * GH_MT];
    const int tid = threadIdx.x, base = blockIdx.x * GH_MT, pi = base + tid;
    if (pi < plane) {
        const float hair = out[3 * plane + pi], head = out[4 * plane + pi];
        const float ang = gh_orient_angle(out[5 * plane + pi], out[6 * plane + pi]).ang;
        const float conf_m = __fmul_rn(out[8 * plane + pi], hair);
        if (o.orient_angle) o.orient_angle[pi] = ang;
        if (o.orient_conf_masked) o.orient_conf_masked[pi] = conf_m;
        s_grey[0][tid] = (unsigned char)gh_quant_u8(hair);
        s_grey[1][tid] = (unsigned char)gh_quant_u8(head);
        s_grey[2][tid] = (unsigned char)gh_quant_u8(__fmul_rn(ang, hair));
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; c++) s_rgb[0][3 * tid + c] = (unsigned char)gh_quant_u8(out[c * plane + pi]);
        gh_vis_orient(ang, hair, v);
#pragma unroll
        for (int c = 0; c < 3; c++) s_rgb[1][3 * tid + c] = (unsigned char)gh_quant_u8(v[c]);
        // the confidence colouring: 1 - 1 / (conf * hair + 1) in place of the mask
        gh_vis_orient(ang, __fsub_rn(1.f, __fdiv_rn(1.f, __fadd_rn(conf_m, 1.f))), v);
#pragma unroll
        for (int c = 0; c < 3; c++) s_rgb[2][3 * tid + c] = (unsigned char)gh_quant_u8(v[c]);
    }
    __syncthreads();
    const int n = min(GH_MT, plane - base);
    if (o.hair_mask_u8) gh_store_staged(o.hair_mask_u8 + base, s_grey[0], n);
    if (o.head_mask_u8) gh_store_staged(o.head_mask_u8 + base, s_grey[1], n);
    if (o.orient_u8) gh_store_staged(o.orient_u8 + base, s_grey[2], n);
    if (o.render_u8) gh_store_staged(o.render_u8 + 3 * (size_t)base, s_rgb[0], 3 * n);
    if (o.orient_vis_u8) gh_store_staged(o.orient_vis_u8 + 3 * (size_t)base, s_rgb[1], 3 * n);
    if (o.orient_conf_vis_u8) gh_store_staged(o.orient_conf_vis_u8 + 3 * (size_t)base, s_rgb[2], 3 * n);
}

// ------------------------------------------------------------------------------------------------ evaluation metrics
// sums[] (doubles): the seven sums, then the completion ticket (uint32, zeroed with the sums)
enum { GH_ES_L1 = 0, GH_ES_MASK = 1, GH_ES_OR = 2, GH_ES_W = 3, GH_ES_SE = 4 /* 4..6: r g b */, GH_ES_TICKET = 8,
       GH_ES_COUNT = 16, GH_ES_K = 7 };

int gh_eval_ctas(int W, int H)
{
    const size_t plane = (size_t)W * H, want = (plane + GH_MT - 1) / GH_MT;
    return (int)(want < 132u * 16u ? want : 132u * 16u);
}

__device__ __forceinline__ float gh_clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

// LATENT == false (train_gaussians.py:254-277, train_strands.py): render, mask, angle and their ground truths clamped
// to [0, 1]; |image - gt|, |mask - gt_mask| over both mask channels, or_loss without confidences, squared error.
// LATENT == true (train_latent_strands.py:235-258): image and gt multiplied by gt_mask[0] first, and the binary cross
// entropy of the hair mask (prediction clamped to [1e-3, 1 - 1e-3], logs clamped at -100 like F.binary_cross_entropy)
// in place of the mask L1.
template <bool LATENT>
__global__ void __launch_bounds__(GH_MT)
gh_eval_metrics_kernel(int plane, const float* __restrict__ out, const float* __restrict__ gt_image,
                       const float* __restrict__ gt_mask, const float* __restrict__ gt_angle,
                       const float* __restrict__ gt_conf, double* __restrict__ sums, double* __restrict__ part)
{
    double v[GH_ES_K] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int pi = blockIdx.x * GH_MT + threadIdx.x; pi < plane; pi += gridDim.x * GH_MT) {
        const float gm0 = gh_clamp01(gt_mask[pi]);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float a = gh_clamp01(out[c * plane + pi]), g = gh_clamp01(gt_image[c * plane + pi]);
            if (LATENT) { a = __fmul_rn(a, gm0); g = __fmul_rn(g, gm0); }
            const float d = a - g;
            v[GH_ES_L1] += (double)fabsf(d);
            v[GH_ES_SE + c] += (double)__fmul_rn(d, d);
        }
        const float m0 = gh_clamp01(out[3 * plane + pi]);
        if (LATENT) {
            const float p = fminf(fmaxf(m0, 1e-3f), 1.f - 1e-3f);
            v[GH_ES_MASK] += (double)((gm0 - 1.f) * fmaxf(logf(1.f - p), -100.f) - gm0 * fmaxf(logf(p), -100.f));
        } else {
            const float m1 = gh_clamp01(out[4 * plane + pi]), gm1 = gh_clamp01(gt_mask[plane + pi]);
            v[GH_ES_MASK] += (double)fabsf(m0 - gm0) + (double)fabsf(m1 - gm1);
        }
        const float ang = gh_clamp01(gh_orient_angle(out[5 * plane + pi], out[6 * plane + pi]).ang);
        const float d0 = ang - gh_clamp01(gt_angle[pi]);
        const float l = fminf(fabsf(d0), fminf(fabsf(d0 - 1.f), fabsf(d0 + 1.f))) * GH_PI_F * gm0;
        const float w = gt_conf[pi];
        v[GH_ES_OR] += (double)(l * w);
        v[GH_ES_W] += (double)w;
    }
    gh_block_sum_fixed<GH_ES_K>(v, part, sums, {0, 1, 2, 3, 4, 5, 6}, GH_ES_TICKET);
}

// row: l1, mask L1 or cross entropy, orientation loss, psnr, ssim (not computed: NaN), mse r g b
template <bool LATENT>
__global__ void gh_eval_finish_kernel(int plane, const double* __restrict__ sums, float* __restrict__ row)
{
    if (threadIdx.x != 0) return;
    const double n = (double)plane;
    double psnr = 0.0;
    for (int c = 0; c < 3; c++) {
        const double mse = sums[GH_ES_SE + c] / n;
        row[5 + c] = (float)mse;
        psnr += 20.0 * log10(1.0 / sqrt(mse));              // mse 0 -> inf, as the reference
    }
    row[0] = (float)(sums[GH_ES_L1] / (3.0 * n));
    row[1] = (float)(sums[GH_ES_MASK] / (LATENT ? n : 2.0 * n));
    row[2] = (float)(sums[GH_ES_OR] / sums[GH_ES_W]);       // weight sum 0 -> NaN (or inf), as the reference
    row[3] = (float)(psnr / 3.0);
    row[4] = __int_as_float(0x7fc00000);
}

}  // namespace

extern "C" int gh_render_maps(int width, int height, const float* out_color, float* orient_angle,
                              float* orient_conf_masked, unsigned char* render_u8, unsigned char* hair_mask_u8,
                              unsigned char* head_mask_u8, unsigned char* orient_u8, unsigned char* orient_vis_u8,
                              unsigned char* orient_conf_vis_u8, gh_stream_t stream_)
{
    gh_clear_error();
    if (width <= 0 || height <= 0 || !out_color)
        return gh_set_error(GH_E_INVALID_ARG, "gh_render_maps: bad size or missing raw image");
    if ((long long)width * height > (1ll << 27))      // 32-bit offsets inside the kernel (10 planes, 3-byte pixels)
        return gh_set_error(GH_E_INVALID_ARG, "gh_render_maps: image larger than 2^27 pixels");
    const unsigned char* bytes[6] = {render_u8, hair_mask_u8, head_mask_u8, orient_u8, orient_vis_u8, orient_conf_vis_u8};
    for (int i = 0; i < 6; i++)
        if ((size_t)bytes[i] & 3) return gh_set_error(GH_E_INVALID_ARG, "gh_render_maps: byte maps must be 4-byte aligned");
    const int plane = width * height;
    const GhMapOutputs o = {orient_angle, orient_conf_masked, render_u8, hair_mask_u8, head_mask_u8, orient_u8,
                            orient_vis_u8, orient_conf_vis_u8};
    gh_render_maps_kernel<<<(plane + GH_MT - 1) / GH_MT, GH_MT, 0, (cudaStream_t)stream_>>>(plane, out_color, o);
    return gh_launch_status("gh_render_maps", 1);
}

extern "C" int gh_eval_metrics_workspace_size(int width, int height, size_t* bytes)
{
    gh_clear_error();
    if (width <= 0 || height <= 0 || !bytes || (long long)width * height > (1ll << 27))
        return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics_workspace_size: bad width/height");
    *bytes = (GH_ES_COUNT + (size_t)GH_ES_K * gh_eval_ctas(width, height)) * sizeof(double);
    return GH_OK;
}

extern "C" int gh_eval_metrics(int width, int height, int stage, const float* out_color, const float* gt_image,
                               const float* gt_mask, const float* gt_orient_angle, const float* gt_orient_conf,
                               void* workspace, size_t workspace_bytes, float* row, gh_stream_t stream_)
{
    gh_clear_error();
    cudaStream_t stream = (cudaStream_t)stream_;
    if (width <= 0 || height <= 0 || !out_color || !gt_image || !gt_mask || !gt_orient_angle || !gt_orient_conf ||
        !workspace || !row)
        return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics: bad size or missing pointer");
    if (stage < GH_LOSS_STAGE_APPEARANCE || stage > GH_LOSS_STAGE_LATENT_STRANDS)
        return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics: unknown stage %d", stage);
    if ((long long)width * height > (1ll << 27))
        return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics: image larger than 2^27 pixels");
    if ((size_t)workspace & 7) return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics: workspace must be 8-byte aligned");
    const int ctas = gh_eval_ctas(width, height);
    const size_t need = (GH_ES_COUNT + (size_t)GH_ES_K * ctas) * sizeof(double);
    if (workspace_bytes < need)
        return gh_set_error(GH_E_INVALID_ARG, "gh_eval_metrics: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    double* sums = reinterpret_cast<double*>(workspace);
    double* part = sums + GH_ES_COUNT;
    const cudaError_t e = cudaMemsetAsync(sums, 0, GH_ES_COUNT * sizeof(double), stream);      // sums + ticket
    if (e != cudaSuccess) return gh_cuda_status("gh_eval_metrics", "memset(sums)", e);
    const int plane = width * height;
    if (stage == GH_LOSS_STAGE_LATENT_STRANDS) {
        gh_eval_metrics_kernel<true><<<ctas, GH_MT, 0, stream>>>(plane, out_color, gt_image, gt_mask, gt_orient_angle,
                                                                  gt_orient_conf, sums, part);
        gh_eval_finish_kernel<true><<<1, 32, 0, stream>>>(plane, sums, row);
    } else {
        gh_eval_metrics_kernel<false><<<ctas, GH_MT, 0, stream>>>(plane, out_color, gt_image, gt_mask, gt_orient_angle,
                                                                   gt_orient_conf, sums, part);
        gh_eval_finish_kernel<false><<<1, 32, 0, stream>>>(plane, sums, row);
    }
    return gh_launch_status("gh_eval_metrics", 2);
}
