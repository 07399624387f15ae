// "Next" row 4 (SURVEY.md 8f): the image-space losses of the appearance stage, fused forward + backward.
// They consume the rasterizer's (10,H,W) output on every training iteration and hand dL/dout(10,H,W)
// straight back to the blend backward:
//     Ll1     = l1_loss(image, gt_image, mask = gt_mask[1:])                 SRC/train_gaussians.py:126
//     Lssim   = 1 - ssim(image * gt_mask[1:], gt_image * gt_mask[1:])         :127, SRC/utils/loss_utils.py:83-121
//     Lmask   = l1_loss(mask, gt_mask)                                       :128
//     Lorient = or_loss(orient_angle, gt_orient_angle, orient_conf,
//                       weight = gt_orient_conf, mask = gt_mask[:1])         :130-131, loss_utils.py:31-48
//               with orient_angle = acos(clamp(normalize(out[5:7]).y) * mirror) / pi
//                                                                            SRC/gaussian_renderer/__init__.py:100-105
//               and "NaN -> 0"                                               :133
//     loss    = l_dl1 Ll1 + l_dssim Lssim + l_dmask Lmask + l_dorient Lorient :135-140
// The reference runs this as ~60 elementwise / reduction kernels plus five 11x11 depthwise convolutions
// and their autograd mirror; here it is 5 launches:
//     gh_loss_presum_kernel    sum of the orientation weights (the gradient needs 1 / sum)
//     gh_loss_pointwise_kernel masked L1 value, mask L1, orientation loss -> loss sums, dL/dout channels 3..9
//     gh_loss_main_kernel      SSIM statistics (separable 11-tap window, register
//                              blocked over shared memory, float2 pairs) -> SSIM sum, three derivative maps
//     gh_loss_ssim_bwd_kernel  second separable pass over the derivative maps -> dL/dout channels 0..2
//     gh_loss_finalize_kernel  scalars; zeroes the orientation gradients if Lorient was NaN
// Output channel layout (SRC/gaussian_renderer/__init__.py:98): image 0..2, mask 3..4, dir 5..7,
// orientation confidence 8, depth 9.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_LT 32                       // loss tile edge (pixels); 256 threads, 4 pixels each
#define GH_LR 5                        // window radius: 11 taps
#define GH_LH (GH_LT + 2 * GH_LR)      // halo tile edge: 42
#define GH_XS (GH_LH + 1)              // row stride of the halo arrays (float2): conflict-free column walks
#define GH_HS (GH_LT + 1)              // row stride of the horizontally filtered arrays
#define GH_HITEMS (GH_LH * (GH_LT / 8))   // horizontal work items: one halo row x 8 output columns = 168

struct GhLossParams {
    int W, H;
    float l_dl1, l_dssim, l_dmask, l_dorient;
    float g[11];                       // normalised 1-D Gaussian window, sigma 1.5 (loss_utils.py:74-76)
};

enum { GH_LS_W = 0, GH_LS_L1 = 1, GH_LS_SSIM = 2, GH_LS_MASK = 3, GH_LS_ORIENT = 4, GH_LS_COUNT = 16 };

__device__ __forceinline__ float gh_sign(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }
__device__ __forceinline__ float2 gh_l2(float a) { return make_float2(a, a); }
// (x, y) pairs filtered together; each half is one IEEE-rounded FMUL / FFMA
__device__ __forceinline__ float2 gh_mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 gh_fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

__device__ __forceinline__ void gh_block_add(double v, double* dst, double* s_part) {
    // 256-thread CTA: warp shuffle tree, then one atomic per CTA
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int tid = threadIdx.x;
    __syncthreads();
    if ((tid & 31) == 0) s_part[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += s_part[w];
        atomicAdd(dst, t);
    }
}

// sums[] (doubles): 0 sum w, 1 sum |I-G| m, 2 sum ssim_map, 3 sum |M-GM|, 4 sum orient loss * w; slots 8.. hold the
// completion tickets of the three summing kernels (uint32, zeroed with the sums)
enum { GH_TK_PRESUM = 8, GH_TK_POINTWISE = 9, GH_TK_MAIN = 10 };

// Deterministic variant of gh_block_add for K sums (gh_image_loss with deterministic != 0): warp shuffle tree, the 8
// warps in warp order, then the CTA's total goes to its own slot part[k * gridDim + CTA] -- no floating-point atomics.
// The last CTA to finish (ticket) adds the slots in CTA order into sums[idx[k]], staging 256 slots at a time in shared
// memory; that is one of the orders the per-CTA atomicAdd could produce, now the only one, so the loss values and the
// 1 / sum(w) that scales the orientation gradient are reproducible.
template <int K>
__device__ __forceinline__ void gh_block_sum_fixed(double (&v)[K], double* __restrict__ part, double* sums,
                                                   const int (&idx)[K], int ticket_slot) {
    __shared__ double s_part[K][8];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
#pragma unroll
    for (int k = 0; k < K; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    __syncthreads();
    if ((tid & 31) == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) s_part[k][tid >> 5] = v[k];
    }
    __syncthreads();
    const unsigned G = gridDim.x * gridDim.y, b = blockIdx.y * gridDim.x + blockIdx.x;
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) {
            double t = 0.0;
            for (int w = 0; w < 8; w++) t += s_part[k][w];
            part[(size_t)k * G + b] = t;
        }
        __threadfence();
        s_last = atomicAdd(reinterpret_cast<unsigned*>(sums + ticket_slot), 1u) == G - 1u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ double s_stage[K][256];
    double t = 0.0;                     // thread k: sum k
    for (unsigned c0 = 0; c0 < G; c0 += 256) {
        const unsigned m = min(256u, G - c0);
#pragma unroll
        for (int k = 0; k < K; k++)
            if ((unsigned)tid < m) s_stage[k][tid] = __ldcg(part + (size_t)k * G + c0 + tid);
        __syncthreads();
        if (tid < K)
            for (unsigned i = 0; i < m; i++) t += s_stage[tid][i];
        __syncthreads();
    }
    if (tid < K) {
        int d = idx[0];
#pragma unroll
        for (int k = 1; k < K; k++) d = (tid == k) ? idx[k] : d;
        sums[d] = t;
    }
}

// per-CTA slots of the three summing kernels, after the sums: presum, pointwise (3 sums), SSIM
struct GhLossParts {
    int rb, pb, mb;                    // CTAs of presum / finalize, pointwise, main
    static GhLossParts of(int W, int H) {
        const size_t plane = (size_t)W * H;
        GhLossParts p;
        p.rb = (int)((plane + 255) / 256 < 132u * 8u ? (plane + 255) / 256 : 132u * 8u);
        p.pb = (int)((plane + 255) / 256 < 132u * 16u ? (plane + 255) / 256 : 132u * 16u);
        p.mb = ((W + GH_LT - 1) / GH_LT) * ((H + GH_LT - 1) / GH_LT);
        return p;
    }
    size_t doubles() const { return (size_t)rb + 3 * (size_t)pb + (size_t)mb; }
};

template <bool DET>
__global__ void __launch_bounds__(256)
gh_loss_presum_kernel(const float* __restrict__ gt_orient_conf, size_t n, double* __restrict__ sums, double* __restrict__ part)
{
    double acc = 0.0;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) acc += (double)gt_orient_conf[i];
    if constexpr (DET) {
        double v[1] = {acc};
        gh_block_sum_fixed<1>(v, part, sums, {GH_LS_W}, GH_TK_PRESUM);
    } else {
        __shared__ double s_part[8];
        gh_block_add(acc, sums + GH_LS_W, s_part);
    }
}

// Pointwise terms of one pixel: loss contributions (returned through the accumulators) and dL/dout for
// channels 3..9 (and 0..2 in the latent-strand stage, which has no SSIM pass).
//   STAGE 0 (appearance):     L1 masked by gt_mask[1]; mask L1 over both channels
//   STAGE 1 (strands):        L1 unmasked (m1 = 1, exact); mask L1 over both channels
//   STAGE 2 (latent strands): L1 unmasked, its gradient written here; mask L1 over channel 3 only, channel 4 zero
//   OPTS: GH_LOSS_ORIENT_UNIT_WEIGHT (w = 1, sum of weights = W H), GH_LOSS_ORIENT_NO_CONF (no confidence factor and
//   no log term: channel 8 is zero)
template <int STAGE, unsigned OPTS>
__device__ __forceinline__ void gh_loss_pointwise(const GhLossParams& prm, size_t plane, size_t pi, float inv_sum_w,
                                                  const float* __restrict__ out, const float* __restrict__ gt_image,
                                                  const float* __restrict__ gt_mask, const float* __restrict__ gt_angle,
                                                  const float* __restrict__ gt_conf, float* __restrict__ dL,
                                                  double& a_l1, double& a_mask, double& a_orient)
{
    constexpr bool unit_w = (OPTS & GH_LOSS_ORIENT_UNIT_WEIGHT) != 0, no_conf = (OPTS & GH_LOSS_ORIENT_NO_CONF) != 0;
    const float m0 = gt_mask[pi], m1 = (STAGE == 0) ? gt_mask[plane + pi] : 1.f;
    // masked L1 on the image (value only; its gradient is written with the SSIM gradient, or here in stage 2)
    const float s_l1 = prm.l_dl1 / (float)(3.0 * (double)plane);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        a_l1 += (double)(fabsf(out[c * plane + pi] - gt_image[c * plane + pi]) * m1);
        if constexpr (STAGE == 2) dL[c * plane + pi] = s_l1 * gh_sign(out[c * plane + pi] - gt_image[c * plane + pi]);
    }
    // L1 on the two mask channels (stage 2: on channel 3 only)
    constexpr int NMASK = (STAGE == 2) ? 1 : 2;
    const float dm_scale = prm.l_dmask / (float)((STAGE == 2 ? 1.0 : 2.0) * (double)plane);
#pragma unroll
    for (int k = 0; k < NMASK; k++) {
        const float d = out[(3 + k) * plane + pi] - gt_mask[k * plane + pi];
        a_mask += (double)fabsf(d);
        dL[(3 + k) * plane + pi] = dm_scale * gh_sign(d);
    }
    if constexpr (STAGE == 2) dL[4 * plane + pi] = 0.f;
    // orientation: dir = normalize(out[5:7]), mirrored so that dir.x >= 0, angle = acos(dir.y)/pi
    const float c5 = out[5 * plane + pi], c6 = out[6 * plane + pi], conf = no_conf ? 1.f : out[8 * plane + pi];
    const float nrm = sqrtf(c5 * c5 + c6 * c6);
    const float den = fmaxf(nrm, 1e-12f);                  // F.normalize eps
    const float dirx = c5 / den, diry = c6 / den;
    const float mirror = (dirx < 0.f) ? -1.f : 1.f;
    const float lo = -1.f + 1e-3f, hi = 1.f - 1e-3f;
    const float tcl = fminf(fmaxf(diry, lo), hi);
    const float t = tcl * mirror;
    const float PI = 3.14159265358979323846f;
    const float ang = acosf(t) / PI;
    const float g = gt_angle[pi];
    const float d0 = ang - g, d1 = d0 - 1.f, d2 = d0 + 1.f;
    const float l0 = fabsf(d0), l1 = fabsf(d1), l2 = fabsf(d2);
    const float inner = fminf(l1, l2);
    const float Lmin = fminf(l0, inner) * PI;
    const float w = unit_w ? 1.f : gt_conf[pi];
    const float lp = no_conf ? Lmin * m0 : (Lmin * conf - logf(conf + 1e-7f)) * m0;
    a_orient += (double)(lp * w);
    // gradients; 1 / sum(w) is known from the presum launch (W H with unit weights)
    const float up = m0 * w * (prm.l_dorient * inv_sum_w);   // d loss / d (per-pixel loss before mask)
    // torch.minimum splits the gradient evenly on ties
    const float w_outer0 = (l0 < inner) ? 1.f : ((l0 == inner) ? 0.5f : 0.f);
    const float w_in = 1.f - w_outer0;
    const float w1 = (l1 < l2) ? 1.f : ((l1 == l2) ? 0.5f : 0.f);
    const float upc = no_conf ? up : up * conf;
    const float dL_dang = upc * PI * (w_outer0 * gh_sign(d0) + w_in * (w1 * gh_sign(d1) + (1.f - w1) * gh_sign(d2)));
    const float dang_dt = -1.f / (PI * sqrtf(fmaxf(1.f - t * t, 0.f)));
    const float dt_ddiry = (diry >= lo && diry <= hi) ? mirror : 0.f;       // clamp passes the gradient inside [lo, hi]
    const float gdy = dL_dang * dang_dt * dt_ddiry;
    float ddy_dc5, ddy_dc6;
    if (nrm > 1e-12f) {
        const float inv = 1.f / nrm, inv3 = inv * inv * inv;
        ddy_dc5 = -c5 * c6 * inv3;
        ddy_dc6 = c5 * c5 * inv3;
    } else {                                                 // norm clamped to eps: constant denominator
        ddy_dc5 = 0.f; ddy_dc6 = 1.f / 1e-12f;
    }
    dL[5 * plane + pi] = gdy * ddy_dc5;
    dL[6 * plane + pi] = gdy * ddy_dc6;
    dL[7 * plane + pi] = 0.f;
    dL[8 * plane + pi] = no_conf ? 0.f : up * (Lmin - 1.f / (conf + 1e-7f));
    dL[9 * plane + pi] = 0.f;
}

// All pointwise terms (masked L1 value, mask L1, orientation) of every pixel: loss sums and dL/dout
// channels 3..9 (0..9 in stage 2).  Plain elementwise kernel, one pixel per thread per grid-stride step.
template <bool DET, int STAGE, unsigned OPTS>
__global__ void __launch_bounds__(256)
gh_loss_pointwise_kernel(GhLossParams prm, const float* __restrict__ out, const float* __restrict__ gt_image,
                         const float* __restrict__ gt_mask, const float* __restrict__ gt_angle,
                         const float* __restrict__ gt_conf, double* __restrict__ sums, float* __restrict__ dL,
                         double* __restrict__ part)
{
    const size_t plane = (size_t)prm.W * prm.H;
    double a_l1 = 0.0, a_mask = 0.0, a_orient = 0.0;
    const float inv_sum_w = 1.0f / (float)((OPTS & GH_LOSS_ORIENT_UNIT_WEIGHT) ? (double)plane : sums[GH_LS_W]);
    for (size_t pi = (size_t)blockIdx.x * 256 + threadIdx.x; pi < plane; pi += (size_t)gridDim.x * 256)
        gh_loss_pointwise<STAGE, OPTS>(prm, plane, pi, inv_sum_w, out, gt_image, gt_mask, gt_angle, gt_conf, dL,
                                       a_l1, a_mask, a_orient);
    if constexpr (DET) {
        double v[3] = {a_l1, a_mask, a_orient};
        gh_block_sum_fixed<3>(v, part, sums, {GH_LS_L1, GH_LS_MASK, GH_LS_ORIENT}, GH_TK_POINTWISE);
    } else {
        __shared__ double s_part[8];
        gh_block_add(a_l1, sums + GH_LS_L1, s_part);
        gh_block_add(a_mask, sums + GH_LS_MASK, s_part);
        gh_block_add(a_orient, sums + GH_LS_ORIENT, s_part);
    }
}

// SSIM statistics of a 32x32 tile: separable 11-tap window, register blocked (a thread filters 8
// adjacent columns of a halo row, then 4 adjacent rows of a column, so a shared-memory value is reused
// by up to 8 taps) and paired: (x, y) and (x^2, y^2) travel as float2.  STAGE 1 takes the image unmasked (the mask is
// 1: x * 1 is exact, so this is the STAGE 0 arithmetic without the mask loads).
template <int MINB, bool DET, int STAGE>
__global__ void __launch_bounds__(256, MINB)
gh_loss_main_kernel(GhLossParams prm, const float* __restrict__ out, const float* __restrict__ gt_image,
                    const float* __restrict__ gt_mask, double* __restrict__ sums,
                    float* __restrict__ dmaps,      // [3 channels][3 maps][H*W]
                    double* __restrict__ part)
{
    __shared__ float2 sXY[GH_LH][GH_XS];             // (x, y) = (render, target) * mask
    __shared__ float2 sH01[GH_LH][GH_HS], sH23[GH_LH][GH_HS];   // row-filtered (x, y), (x^2, y^2)
    __shared__ float sH4[GH_LH][GH_HS];              // row-filtered x y
    const int W = prm.W, H = prm.H;
    const int plane = W * H;            // 10 * plane < 2^31 is checked by the host entry point
    const int tx0 = blockIdx.x * GH_LT, ty0 = blockIdx.y * GH_LT;
    const int tid = threadIdx.x;

    // ------------------------------------------------------------------ SSIM statistics, channel by channel
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    double a_ssim = 0.0;
    for (int c = 0; c < 3; c++) {
        __syncthreads();
        {   // halo load: warp w takes rows w, w+8, ...; all loads of a thread are issued before the first use
            const int lane = tid & 31, warp = tid >> 5;
            const float* oc = out + c * plane;
            const float* gc = gt_image + c * plane;
            const float* mc = gt_mask + plane;
#pragma unroll
            for (int jb = 0; jb < 6; jb += 3) {
            float xo[6], xg[6], xm[6];
#pragma unroll
            for (int jj = 0; jj < 3; jj++) {
                const int j = jb + jj;
                const int hy = warp + 8 * j, gy = ty0 + hy - GH_LR;
                const bool rowok = hy < GH_LH && gy >= 0 && gy < H;
                const int rowbase = (rowok ? gy : 0) * W;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int hx = lane + 32 * h, gx = tx0 + hx - GH_LR;
                    const bool ok = rowok && hx < GH_LH && gx >= 0 && gx < W;
                    const int q = rowbase + (ok ? gx : 0);
                    xo[2 * jj + h] = ok ? oc[q] : 0.f;
                    xg[2 * jj + h] = ok ? gc[q] : 0.f;
                    xm[2 * jj + h] = ok ? (STAGE == 0 ? mc[q] : 1.f) : 0.f;   // zero padding (F.conv2d padding=5)
                }
            }
#pragma unroll
            for (int jj = 0; jj < 3; jj++) {
                const int hy = warp + 8 * (jb + jj);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int hx = lane + 32 * h;
                    if (hy < GH_LH && hx < GH_LH) sXY[hy][hx] = make_float2(xo[2 * jj + h] * xm[2 * jj + h], xg[2 * jj + h] * xm[2 * jj + h]);
                }
            }
            }
        }
        __syncthreads();
        if (tid < GH_HITEMS) {                               // horizontal pass: row r, output columns 8 gq .. 8 gq + 7
            const int r = tid % GH_LH, gq = tid / GH_LH;
            // input-stationary: each loaded value feeds the (up to 8) outputs whose window contains it
            float2 s01[8], s23[8];
            float s4[8];
#pragma unroll
            for (int o = 0; o < 8; o++) { s01[o] = make_float2(0.f, 0.f); s23[o] = make_float2(0.f, 0.f); s4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < 18; k++) {
                const float2 v = sXY[r][8 * gq + k];
                const float2 sq = gh_mul2(v, v);
                const float xy = v.x * v.y;
#pragma unroll
                for (int o = 0; o < 8; o++) {
                    if (k - o >= 0 && k - o <= 10) {
                        const float gk = prm.g[k - o];
                        s01[o] = gh_fma2(gh_l2(gk), v, s01[o]);
                        s23[o] = gh_fma2(gh_l2(gk), sq, s23[o]);
                        s4[o] = fmaf(gk, xy, s4[o]);
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
                        const float gk = prm.g[k - o];
                        m4[o] = gh_fma2(gh_l2(gk), a01, m4[o]);
                        e4[o] = gh_fma2(gh_l2(gk), a23, e4[o]);
                        e12_4[o] = fmaf(gk, a4, e12_4[o]);
                    }
                }
            }
            const int px = tx0 + lx;
#pragma unroll
            for (int o = 0; o < 4; o++) {
                const float2 m = m4[o], e = e4[o];
                const float e12 = e12_4[o];
                const int py = ty0 + 4 * rg + o;
                if (px < W && py < H) {
                    const int pi = py * W + px;
                    const float mu1 = m.x, mu2 = m.y;
                    const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
                    const float sg1 = e.x - mu1_sq, sg2 = e.y - mu2_sq, sg12 = e12 - mu12;
                    const float a1 = 2.f * mu12 + C1, a2 = 2.f * sg12 + C2;
                    const float b1 = mu1_sq + mu2_sq + C1, b2 = sg1 + sg2 + C2;
                    const float ib = __frcp_rn(b1 * b2);
                    const float S = a1 * a2 * ib;
                    a_ssim += (double)S;
                    // derivatives of the map w.r.t. conv(x), conv(x^2), conv(x y) at this pixel
                    float* dm = dmaps + (size_t)c * 3 * (size_t)plane;
                    dm[pi] = 2.f * mu2 * (a2 - a1) * ib - 2.f * mu1 * S * (b2 - b1) * ib;
                    dm[plane + pi] = -S * __frcp_rn(b2);
                    dm[2 * plane + pi] = 2.f * a1 * ib;
                }
            }
        }
    }
    if constexpr (DET) {
        double v[1] = {a_ssim};
        gh_block_sum_fixed<1>(v, part, sums, {GH_LS_SSIM}, GH_TK_MAIN);
    } else {
        __shared__ double s_part[8];
        gh_block_add(a_ssim, sums + GH_LS_SSIM, s_part);
    }
}

template <int MINB, int STAGE>
__global__ void __launch_bounds__(256, MINB)
gh_loss_ssim_bwd_kernel(GhLossParams prm, const float* __restrict__ out, const float* __restrict__ gt_image,
                        const float* __restrict__ gt_mask, const float* __restrict__ dmaps, float* __restrict__ dL)
{
    __shared__ float2 sD01[GH_LH][GH_XS];
    __shared__ float sD2[GH_LH][GH_XS];
    __shared__ float2 sH01[GH_LH][GH_HS];
    __shared__ float sH2[GH_LH][GH_HS];
    const int W = prm.W, H = prm.H;
    const int plane = W * H;            // 10 * plane < 2^31 is checked by the host entry point
    const int tx0 = blockIdx.x * GH_LT, ty0 = blockIdx.y * GH_LT;
    const int tid = threadIdx.x;
    const float n3 = (float)(3.0 * (double)plane);
    const float s_ssim = -prm.l_dssim / n3;       // d loss / d ssim_map(p): Lssim = 1 - mean(map)
    const float s_l1 = prm.l_dl1 / n3;
    for (int c = 0; c < 3; c++) {
        const float* dm = dmaps + (size_t)c * 3 * (size_t)plane;
        __syncthreads();
        {   // halo load (map pixels outside the image do not exist: zeros)
            const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
            for (int jb = 0; jb < 6; jb += 3) {
            float x0[6], x1[6], x2[6];
#pragma unroll
            for (int jj = 0; jj < 3; jj++) {
                const int j = jb + jj;
                const int hy = warp + 8 * j, gy = ty0 + hy - GH_LR;
                const bool rowok = hy < GH_LH && gy >= 0 && gy < H;
                const int rowbase = (rowok ? gy : 0) * W;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int hx = lane + 32 * h, gx = tx0 + hx - GH_LR;
                    const bool ok = rowok && hx < GH_LH && gx >= 0 && gx < W;
                    const int q = rowbase + (ok ? gx : 0);
                    x0[2 * jj + h] = ok ? dm[q] : 0.f;
                    x1[2 * jj + h] = ok ? dm[plane + q] : 0.f;
                    x2[2 * jj + h] = ok ? dm[2 * plane + q] : 0.f;
                }
            }
#pragma unroll
            for (int jj = 0; jj < 3; jj++) {
                const int hy = warp + 8 * (jb + jj);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int hx = lane + 32 * h;
                    if (hy < GH_LH && hx < GH_LH) { sD01[hy][hx] = make_float2(x0[2 * jj + h], x1[2 * jj + h]); sD2[hy][hx] = x2[2 * jj + h]; }
                }
            }
            }
        }
        __syncthreads();
        if (tid < GH_HITEMS) {
            const int r = tid % GH_LH, gq = tid / GH_LH;
            float2 s01[8];
            float s2[8];
#pragma unroll
            for (int o = 0; o < 8; o++) { s01[o] = make_float2(0.f, 0.f); s2[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < 18; k++) {
                const float2 v = sD01[r][8 * gq + k];
                const float u = sD2[r][8 * gq + k];
#pragma unroll
                for (int o = 0; o < 8; o++) {
                    if (k - o >= 0 && k - o <= 10) {
                        s01[o] = gh_fma2(gh_l2(prm.g[k - o]), v, s01[o]);
                        s2[o] = fmaf(prm.g[k - o], u, s2[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < 8; o++) { sH01[r][8 * gq + o] = s01[o]; sH2[r][8 * gq + o] = s2[o]; }
        }
        __syncthreads();
        {
            const int lx = tid & 31, rg = tid >> 5;
            float2 D01_4[4];
            float D2_4[4];
#pragma unroll
            for (int o = 0; o < 4; o++) { D01_4[o] = make_float2(0.f, 0.f); D2_4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < 14; k++) {
                const float2 a01 = sH01[4 * rg + k][lx];
                const float a2 = sH2[4 * rg + k][lx];
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    if (k - o >= 0 && k - o <= 10) {
                        D01_4[o] = gh_fma2(gh_l2(prm.g[k - o]), a01, D01_4[o]);
                        D2_4[o] = fmaf(prm.g[k - o], a2, D2_4[o]);
                    }
                }
            }
            const int px = tx0 + lx;
#pragma unroll
            for (int o = 0; o < 4; o++) {
                const float2 D01 = D01_4[o];
                const float D2 = D2_4[o];
                const int py = ty0 + 4 * rg + o;
                if (px < W && py < H) {
                    const int pi = py * W + px;
                    const float m1 = (STAGE == 0) ? gt_mask[plane + pi] : 1.f;
                    const float I = out[c * plane + pi], G = gt_image[c * plane + pi];
                    const float x = I * m1, y = G * m1;
                    // the window is symmetric: the adjoint of the convolution is the same convolution
                    const float dS_dx = D01.x + 2.f * x * D01.y + y * D2;
                    dL[c * plane + pi] = s_ssim * dS_dx * m1 + s_l1 * gh_sign(I - G) * m1;
                }
            }
        }
    }
}

// losses[8]: total, Ll1, Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN flag, slot 7.
// Stage 2 (SRC/train_latent_strands.py:142-152): slot 2 is 0, slot 3 holds LCE, and Ll1, LCE and LOR are each replaced
// by 0 when NaN, zeroing their gradient channels; slot 7 holds the replaced terms as a bitmask (1 Ll1, 2 LCE).
template <int STAGE, unsigned OPTS>
__global__ void __launch_bounds__(256)
gh_loss_finalize_kernel(GhLossParams prm, const double* __restrict__ sums, float* __restrict__ losses, float* __restrict__ dL)
{
    constexpr bool unit_w = (OPTS & GH_LOSS_ORIENT_UNIT_WEIGHT) != 0;
    const size_t plane = (size_t)prm.W * prm.H;
    const double n = (double)plane;
    const float Lorient_raw = (float)(sums[GH_LS_ORIENT] / (unit_w ? n : sums[GH_LS_W]));
    const bool bad = (Lorient_raw != Lorient_raw);                    // torch.isnan(Lorient).any() -> zeros_like
    if constexpr (STAGE == 2) {
        const float Ll1_raw = (float)(sums[GH_LS_L1] / (3.0 * n));
        const float LCE_raw = (float)(sums[GH_LS_MASK] / n);
        const bool bad_l1 = (Ll1_raw != Ll1_raw), bad_ce = (LCE_raw != LCE_raw);
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            const float Ll1 = bad_l1 ? 0.f : Ll1_raw, LCE = bad_ce ? 0.f : LCE_raw, LOR = bad ? 0.f : Lorient_raw;
            losses[0] = Ll1 * prm.l_dl1 + LCE * prm.l_dmask + LOR * prm.l_dorient;
            losses[1] = Ll1; losses[2] = 0.f; losses[3] = LCE; losses[4] = LOR;
            losses[5] = (float)(unit_w ? n : sums[GH_LS_W]); losses[6] = bad ? 1.f : 0.f;
            losses[7] = (bad_l1 ? 1.f : 0.f) + (bad_ce ? 2.f : 0.f);
        }
        if (!(bad || bad_l1 || bad_ce)) return;
        // a replaced term is a constant: nothing flows into its channels
        for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < plane; i += (size_t)gridDim.x * 256) {
            if (bad_l1) { dL[i] = 0.f; dL[plane + i] = 0.f; dL[2 * plane + i] = 0.f; }
            if (bad_ce) dL[3 * plane + i] = 0.f;
            if (bad) { dL[5 * plane + i] = 0.f; dL[6 * plane + i] = 0.f; dL[8 * plane + i] = 0.f; }
        }
    } else {
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            const float Ll1 = (float)(sums[GH_LS_L1] / (3.0 * n));
            const float Lssim = 1.0f - (float)(sums[GH_LS_SSIM] / (3.0 * n));
            const float Lmask = (float)(sums[GH_LS_MASK] / (2.0 * n));
            const float Lorient = bad ? 0.f : Lorient_raw;
            losses[0] = Ll1 * prm.l_dl1 + Lssim * prm.l_dssim + Lmask * prm.l_dmask + Lorient * prm.l_dorient;
            losses[1] = Ll1; losses[2] = Lssim; losses[3] = Lmask; losses[4] = Lorient;
            losses[5] = (float)(unit_w ? n : sums[GH_LS_W]); losses[6] = bad ? 1.f : 0.f; losses[7] = 0.f;
        }
        if (!bad) return;
        // the orientation term was replaced by a constant: nothing flows into channels 5, 6, 8
        for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < plane; i += (size_t)gridDim.x * 256) {
            dL[5 * plane + i] = 0.f; dL[6 * plane + i] = 0.f; dL[8 * plane + i] = 0.f;
        }
    }
}

// The launches of one (stage, options) pair: presum (unless the weights are unit), pointwise, the two SSIM passes
// (stages 0 and 1), finalize.  Returns the number of kernels launched.
template <int STAGE, unsigned OPTS>
int gh_loss_launch(const GhLossParams& prm, const float* out_color, const float* gt_image, const float* gt_mask,
                   const float* gt_orient_angle, const float* gt_orient_conf, double* sums, float* losses,
                   float* dL_dout, cudaStream_t stream, bool deterministic)
{
    constexpr bool unit_w = (OPTS & GH_LOSS_ORIENT_UNIT_WEIGHT) != 0, ssim = STAGE != 2;
    const int width = prm.W, height = prm.H;
    const GhLossParts np = GhLossParts::of(width, height);
    double* part_presum = sums + GH_LS_COUNT;
    double* part_pointwise = part_presum + np.rb;
    double* part_main = part_pointwise + 3 * (size_t)np.pb;
    float* dmaps = reinterpret_cast<float*>(part_main + np.mb);
    const size_t plane = (size_t)width * height;
    const int rb = np.rb, pb = np.pb;
    const dim3 grid((width + GH_LT - 1) / GH_LT, (height + GH_LT - 1) / GH_LT), block(256);
    if (deterministic) {
        if (!unit_w) gh_loss_presum_kernel<true><<<rb, 256, 0, stream>>>(gt_orient_conf, plane, sums, part_presum);
        gh_loss_pointwise_kernel<true, STAGE, OPTS><<<pb, 256, 0, stream>>>(prm, out_color, gt_image, gt_mask,
            gt_orient_angle, gt_orient_conf, sums, dL_dout, part_pointwise);
        if constexpr (ssim)
            gh_loss_main_kernel<4, true, STAGE><<<grid, block, 0, stream>>>(prm, out_color, gt_image, gt_mask, sums, dmaps, part_main);
    } else {
        if (!unit_w) gh_loss_presum_kernel<false><<<rb, 256, 0, stream>>>(gt_orient_conf, plane, sums, nullptr);
        gh_loss_pointwise_kernel<false, STAGE, OPTS><<<pb, 256, 0, stream>>>(prm, out_color, gt_image, gt_mask,
            gt_orient_angle, gt_orient_conf, sums, dL_dout, nullptr);
        // 4 CTAs per SM (64 registers)
        if constexpr (ssim)
            gh_loss_main_kernel<4, false, STAGE><<<grid, block, 0, stream>>>(prm, out_color, gt_image, gt_mask, sums, dmaps, nullptr);
    }
    if constexpr (ssim)
        gh_loss_ssim_bwd_kernel<4, STAGE><<<grid, block, 0, stream>>>(prm, out_color, gt_image, gt_mask, dmaps, dL_dout);
    gh_loss_finalize_kernel<STAGE, OPTS><<<rb, 256, 0, stream>>>(prm, sums, losses, dL_dout);
    return (unit_w ? 0 : 1) + 1 + (ssim ? 2 : 0) + 1;
}

// Argument checks and launches shared by gh_image_loss and gh_image_loss_stage; `who` names the entry point in the
// messages.  The stage and option checks are the caller's.
int gh_image_loss_run(const char* who, int width, int height, int stage, unsigned options, const float* out_color,
                      const float* gt_image, const float* gt_mask, const float* gt_orient_angle,
                      const float* gt_orient_conf, float lambda_dl1, float lambda_dssim, float lambda_dmask,
                      float lambda_dorient, void* workspace, float* losses, float* dL_dout, gh_stream_t stream_,
                      int deterministic)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    const bool conf_needed = !(options & GH_LOSS_ORIENT_UNIT_WEIGHT);
    if (width <= 0 || height <= 0 || !out_color || !gt_image || !gt_mask || !gt_orient_angle ||
        (conf_needed && !gt_orient_conf) || !workspace || !losses || !dL_dout)
        return gh_set_error(GH_E_INVALID_ARG, "%s: bad size or missing pointer", who);
    if ((size_t)workspace & 7) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace must be 8-byte aligned", who);
    if ((long long)width * height > (1ll << 27))      // 32-bit pixel offsets inside the kernels
        return gh_set_error(GH_E_INVALID_ARG, "%s: image larger than 2^27 pixels", who);
    GhLossParams prm;
    prm.W = width; prm.H = height;
    prm.l_dl1 = lambda_dl1; prm.l_dssim = lambda_dssim; prm.l_dmask = lambda_dmask; prm.l_dorient = lambda_dorient;
    {   // gaussian(11, 1.5) as the reference builds it: float32 taps, float32 normalisation
        float g[11], sum = 0.f;
        for (int k = 0; k < 11; k++) { g[k] = (float)exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)); sum += g[k]; }
        for (int k = 0; k < 11; k++) prm.g[k] = g[k] / sum;
    }
    double* sums = reinterpret_cast<double*>(workspace);
    const cudaError_t e = cudaMemsetAsync(sums, 0, GH_LS_COUNT * sizeof(double), stream);     // sums + tickets
    if (e != cudaSuccess) return gh_cuda_status(who, "memset(partial sums)", e);
    const bool det = deterministic != 0;
#define GH_LOSS_ARGS prm, out_color, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, sums, losses, dL_dout, stream, det
    int n = 0;
    switch (stage * 4 + (int)options) {
    case 0: n = gh_loss_launch<0, 0u>(GH_LOSS_ARGS); break;
    case 4: n = gh_loss_launch<1, 0u>(GH_LOSS_ARGS); break;
    case 5: n = gh_loss_launch<1, 1u>(GH_LOSS_ARGS); break;
    case 6: n = gh_loss_launch<1, 2u>(GH_LOSS_ARGS); break;
    case 7: n = gh_loss_launch<1, 3u>(GH_LOSS_ARGS); break;
    case 8: n = gh_loss_launch<2, 0u>(GH_LOSS_ARGS); break;
    case 9: n = gh_loss_launch<2, 1u>(GH_LOSS_ARGS); break;
    case 10: n = gh_loss_launch<2, 2u>(GH_LOSS_ARGS); break;
    case 11: n = gh_loss_launch<2, 3u>(GH_LOSS_ARGS); break;
    default: return gh_set_error(GH_E_INVALID_ARG, "%s: unsupported stage %d with options %u", who, stage, options);
    }
#undef GH_LOSS_ARGS
    return gh_launch_status(who, n);
}

}  // namespace

extern "C" int gh_image_loss_workspace_size(int width, int height, size_t* bytes)
{
    gh_clear_error();
    if (width <= 0 || height <= 0 || !bytes) return gh_set_error(GH_E_INVALID_ARG, "gh_image_loss_workspace_size: bad width/height");
    *bytes = (GH_LS_COUNT + GhLossParts::of(width, height).doubles()) * sizeof(double) + (size_t)9 * width * height * sizeof(float);
    return GH_OK;
}

extern "C" int gh_image_loss(int width, int height, const float* out_color, const float* gt_image,
                             const float* gt_mask, const float* gt_orient_angle, const float* gt_orient_conf,
                             float lambda_dl1, float lambda_dssim, float lambda_dmask, float lambda_dorient,
                             void* workspace, float* losses, float* dL_dout, gh_stream_t stream_, int deterministic)
{
    gh_clear_error();
    return gh_image_loss_run("gh_image_loss", width, height, GH_LOSS_STAGE_APPEARANCE, 0u, out_color, gt_image, gt_mask,
                             gt_orient_angle, gt_orient_conf, lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient,
                             workspace, losses, dL_dout, stream_, deterministic);
}

extern "C" int gh_image_loss_stage(int width, int height, int stage, unsigned options, const float* out_color,
                                   const float* gt_image, const float* gt_mask, const float* gt_orient_angle,
                                   const float* gt_orient_conf, float lambda_dl1, float lambda_dssim,
                                   float lambda_dmask, float lambda_dorient, void* workspace, float* losses,
                                   float* dL_dout, gh_stream_t stream_, int deterministic)
{
    gh_clear_error();
    const unsigned known = GH_LOSS_ORIENT_UNIT_WEIGHT | GH_LOSS_ORIENT_NO_CONF;
    if (stage < GH_LOSS_STAGE_APPEARANCE || stage > GH_LOSS_STAGE_LATENT_STRANDS)
        return gh_set_error(GH_E_INVALID_ARG, "gh_image_loss_stage: unknown stage %d", stage);
    if (options & ~known)
        return gh_set_error(GH_E_INVALID_ARG, "gh_image_loss_stage: unknown option bits 0x%x", options & ~known);
    if (stage == GH_LOSS_STAGE_APPEARANCE && options)
        return gh_set_error(GH_E_INVALID_ARG, "gh_image_loss_stage: the appearance stage takes no options");
    if (stage == GH_LOSS_STAGE_LATENT_STRANDS && lambda_dssim != 0.f)
        return gh_set_error(GH_E_INVALID_ARG, "gh_image_loss_stage: the latent-strand stage has no SSIM term "
                                              "(lambda_dssim must be 0)");
    return gh_image_loss_run("gh_image_loss_stage", width, height, stage, options, out_color, gt_image, gt_mask,
                             gt_orient_angle, gt_orient_conf, lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient,
                             workspace, losses, dL_dout, stream_, deterministic);
}
