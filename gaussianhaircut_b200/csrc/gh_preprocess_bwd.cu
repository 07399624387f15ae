// Stage 5: backward of the per-Gaussian preprocess, one fused kernel.
//
// Also unpacks the blend backward's 64-byte accumulation records into the API gradient tensors.
// Covers the reference's computeCov2DCUDA (backward.cu:144-274), the projection part of
// preprocessCUDA (backward.cu:346-400) and the backward of computeCov3D (backward.cu:278-341).
// When the caller supplied the conic (`conic_precomp`, the mode both reference trainers use) the
// reference propagates nothing through the geometry and neither do we (the launcher skips the kernel).
// Gradients are w.r.t. the RAW quaternion (no normalisation Jacobian, backward.cu:340).
// The 3-D covariance is recomputed from scale/rotation instead of being stored by the forward.
#include "gh_common.cuh"
#include "gh_kernels.h"

namespace {

// One CTA of GH_PBWD_THREADS threads handles as many consecutive Gaussians, one per thread.  The array-of-structs rows
// move as whole CTA spans through shared memory (gh_span_load_async / gh_span_store in gh_common.cuh): every input span
// (acc16, means3D, scales or cov3D_precomp) is requested up front with cp.async, so a thread has all of its loads in
// flight at once, and every output with 3, 6 or 10 floats per row leaves as one contiguous span of 16-byte stores.
// Rows of 4 floats (dL_dconic, dL_drot) and of 1 float are stored directly: they already coalesce.
#define GH_PBWD_THREADS 128
// staging buffer in floats: the inputs 16 + 3 + 6 per row, then (after a barrier) the outputs 10 + 3 + 3 + 6 + 3 per
// row; + 4 floats of alignment slack per span
#define GH_PBWD_SMEM_FLOATS (25 * GH_PBWD_THREADS + 5 * 4)

__global__ void __launch_bounds__(GH_PBWD_THREADS, 7)
gh_preprocess_backward_kernel(int P, const float* __restrict__ means3D, const int* __restrict__ radii,
                              const float* __restrict__ scales, float mod,
                              const float* __restrict__ rotations,
                              const float* __restrict__ cov3D_precomp,
                              const float* __restrict__ view, const float* __restrict__ proj,
                              float h_x, float h_y, float tan_fovx, float tan_fovy,
                              const float* __restrict__ acc16,        // (P,16) accumulation records of the blend backward
                              float* __restrict__ dL_dmean2D,         // (P,3), NDC units, z unused      } written here
                              float* __restrict__ dL_dconic,          // (P,4): .x .y .w used            } from acc16
                              float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor,         // }
                              float* __restrict__ dL_dmean3D, float* __restrict__ dL_dcov3D,
                              float* __restrict__ dL_dscale, float* __restrict__ dL_drot)
{
    constexpr int N = GH_PBWD_THREADS;
    __shared__ __align__(16) float s_buf[GH_PBWD_SMEM_FLOATS];
    const int row0 = blockIdx.x * N, t = threadIdx.x;
    const int n = min(N, P - row0);              // rows of this CTA
    const int idx = row0 + t;
    const bool valid = t < n;
    const bool from_scale_rot = (cov3D_precomp == nullptr);

    // ---- inputs: the CTA's spans of acc16, means3D and scales (or cov3D_precomp), all requested at once
    float* s_acc = s_buf;                        // 16 N + 4
    float* s_mean = s_acc + 16 * N + 4;          //  3 N + 4
    float* s_c3 = s_mean + 3 * N + 4;            //  3 N + 4 (scales) or 6 N + 4 (cov3D_precomp)
    const float* g_acc = acc16 + (size_t)row0 * 16;
    const float* g_mean = means3D + (size_t)row0 * 3;
    const float* g_c3 = from_scale_rot ? scales + (size_t)row0 * 3 : cov3D_precomp + (size_t)row0 * 6;
    // the caller's inputs are requested before the wait: the blend backward (or the unpack) that runs before this
    // kernel writes none of them, and the kernels before it have completed
    gh_span_load_async(s_mean, g_mean, 3 * n);
    gh_span_load_async(s_c3, g_c3, (from_scale_rot ? 3 : 6) * n);
    const bool rendered = valid && radii[idx] > 0;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rendered && from_scale_rot) q = reinterpret_cast<const float4*>(rotations)[idx];
    gh_pdl_wait();                               // acc16 is the blend backward's output
    gh_pdl_trigger();
    gh_span_load_async(s_acc, g_acc, 16 * n);
    gh_span_wait();
    __syncthreads();
    // acc16 rows are 64-byte aligned (GhGeomWS), so this thread's record is four aligned float4 in shared memory
    const float4* rec = reinterpret_cast<const float4*>(s_acc + gh_span_shift(g_acc) + 16 * t);
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
    float mx = 0.f, my = 0.f, mz = 0.f;
    float c3[6];
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    if (valid) {
        a0 = rec[0]; a1 = rec[1]; a2 = rec[2]; a3 = rec[3];
        const float* m = s_mean + gh_span_shift(g_mean) + 3 * t;
        mx = m[0]; my = m[1]; mz = m[2];
        if (!from_scale_rot) {
            const float* c = s_c3 + gh_span_shift(g_c3) + 6 * t;
#pragma unroll
            for (int k = 0; k < 6; k++) c3[k] = c[k];
        } else {
            const float* sc = s_c3 + gh_span_shift(g_c3) + 3 * t;
            s0 = sc[0]; s1 = sc[1]; s2 = sc[2];
        }
    }
    __syncthreads();                             // the input spans are consumed: the buffer now stages the outputs

    // ---- outputs: this CTA's rows of the 3-, 6- and 10-float gradients, staged at their spans' alignment
    float* const s_color = s_buf;                // 10 N + 4
    float* const s_m2 = s_color + 10 * N + 4;    //  3 N + 4
    float* const s_m3 = s_m2 + 3 * N + 4;        //  3 N + 4
    float* const s_cov = s_m3 + 3 * N + 4;       //  6 N + 4
    float* const s_scale = s_cov + 6 * N + 4;    //  3 N + 4
    float* const g_color = dL_dcolor + (size_t)row0 * GH_NUM_CHANNELS;
    float* const g_m2 = dL_dmean2D + (size_t)row0 * 3;
    float* const g_m3 = dL_dmean3D + (size_t)row0 * 3;
    float* const g_cov = dL_dcov3D + (size_t)row0 * 6;
    float* const g_scale = dL_dscale ? dL_dscale + (size_t)row0 * 3 : nullptr;
    float* const o_color = s_color + gh_span_shift(g_color) + GH_NUM_CHANNELS * t;   // this thread's staged rows
    float* const o_m2 = s_m2 + gh_span_shift(g_m2) + 3 * t;
    float* const o_m3 = s_m3 + gh_span_shift(g_m3) + 3 * t;
    float* const o_cov = s_cov + gh_span_shift(g_cov) + 6 * t;
    float* const o_scale = s_scale + (g_scale ? gh_span_shift(g_scale) : 0) + 3 * t;
    do {                                         // one row; `break` = row done (every thread reaches the barrier below)
        if (!valid) break;
        // unpack the 64-byte accumulation record into the reference binding's gradient layouts
        // (rasterize_points.cu:160-168) -- every row is written, also for Gaussians that were not rendered
        {
            o_color[0] = a0.x; o_color[1] = a0.y; o_color[2] = a0.z; o_color[3] = a0.w;
            o_color[4] = a1.x; o_color[5] = a1.y; o_color[6] = a1.z; o_color[7] = a1.w;
            o_color[8] = a2.x; o_color[9] = a2.y;
            o_m2[0] = a2.z; o_m2[1] = a2.w; o_m2[2] = 0.f;
            reinterpret_cast<float4*>(dL_dconic)[idx] = make_float4(a3.x, a3.y, 0.f, a3.z);
            dL_dopacity[idx] = a3.w;
        }
        if (!rendered) {
            // not rendered: all geometry gradients are zero (every output row is written, so the caller
            // does not have to zero-fill the buffers)
            o_m3[0] = 0.f; o_m3[1] = 0.f; o_m3[2] = 0.f;
#pragma unroll
            for (int k = 0; k < 6; k++) o_cov[k] = 0.f;
            if (dL_dscale) { o_scale[0] = 0.f; o_scale[1] = 0.f; o_scale[2] = 0.f; }
            if (dL_drot) reinterpret_cast<float4*>(dL_drot)[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
            break;
        }

        if (from_scale_rot) gh_cov3d(s0, s1, s2, mod, q.x, q.y, q.z, q.w, c3);

        // ---- computeCov2DCUDA -------------------------------------------------------------------
        const float dLdcon_x = a3.x, dLdcon_y = a3.y, dLdcon_z = a3.z;
        float tx = view[0] * mx + view[4] * my + view[8] * mz + view[12];
        float ty = view[1] * mx + view[5] * my + view[9] * mz + view[13];
        const float tz = view[2] * mx + view[6] * my + view[10] * mz + view[14];
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float txtz = tx / tz, tytz = ty / tz;
        tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
        ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;

        // glm column-major: J[c][r]; non-zero entries J[0][0], J[0][2], J[1][1], J[1][2]
        const float J00 = h_x / tz, J02 = -(h_x * tx) / (tz * tz);
        const float J11 = h_y / tz, J12 = -(h_y * ty) / (tz * tz);
        // W[c][r] = view[4*r + c]  (W = mat3(v0,v4,v8, v1,v5,v9, v2,v6,v10))
        const float W00 = view[0], W01 = view[4], W02 = view[8];
        const float W10 = view[1], W11 = view[5], W12 = view[9];
        const float W20 = view[2], W21 = view[6], W22 = view[10];
        // T = W * J : T[j][i] = W[0][i] J[j][0] + W[1][i] J[j][1] + W[2][i] J[j][2]
        const float T00 = W00 * J00 + W20 * J02, T01 = W01 * J00 + W21 * J02, T02 = W02 * J00 + W22 * J02;
        const float T10 = W10 * J11 + W20 * J12, T11 = W11 * J11 + W21 * J12, T12 = W12 * J11 + W22 * J12;
        // Vrk symmetric
        const float V00 = c3[0], V01 = c3[1], V02 = c3[2], V11 = c3[3], V12 = c3[4], V22 = c3[5];
        // cov2D = T^T Vrk^T T  (upper-left 2x2)
        const float TV00 = T00 * V00 + T01 * V01 + T02 * V02;   // (T[0] . Vrk[0])
        const float TV01 = T00 * V01 + T01 * V11 + T02 * V12;
        const float TV02 = T00 * V02 + T01 * V12 + T02 * V22;
        const float TV10 = T10 * V00 + T11 * V01 + T12 * V02;
        const float TV11 = T10 * V01 + T11 * V11 + T12 * V12;
        const float TV12 = T10 * V02 + T11 * V12 + T12 * V22;
        const float a = TV00 * T00 + TV01 * T01 + TV02 * T02 + 0.3f;
        const float b = TV00 * T10 + TV01 * T11 + TV02 * T12;
        const float c = TV10 * T10 + TV11 * T11 + TV12 * T12 + 0.3f;

        const float denom = a * c - b * b;
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (denom2inv != 0.f) {
            dL_da = denom2inv * (-c * c * dLdcon_x + 2 * b * c * dLdcon_y + (denom - a * c) * dLdcon_z);
            dL_dc = denom2inv * (-a * a * dLdcon_z + 2 * a * b * dLdcon_y + (denom - a * c) * dLdcon_x);
            dL_db = denom2inv * 2 * (b * c * dLdcon_x - (denom + 2 * b * b) * dLdcon_y + a * b * dLdcon_z);
            dcov[0] = (T00 * T00 * dL_da + T00 * T10 * dL_db + T10 * T10 * dL_dc);
            dcov[3] = (T01 * T01 * dL_da + T01 * T11 * dL_db + T11 * T11 * dL_dc);
            dcov[5] = (T02 * T02 * dL_da + T02 * T12 * dL_db + T12 * T12 * dL_dc);
            dcov[1] = 2 * T00 * T01 * dL_da + (T00 * T11 + T01 * T10) * dL_db + 2 * T10 * T11 * dL_dc;
            dcov[2] = 2 * T00 * T02 * dL_da + (T00 * T12 + T02 * T10) * dL_db + 2 * T10 * T12 * dL_dc;
            dcov[4] = 2 * T02 * T01 * dL_da + (T01 * T12 + T02 * T11) * dL_db + 2 * T11 * T12 * dL_dc;
        }
#pragma unroll
        for (int k = 0; k < 6; k++) o_cov[k] = dcov[k];

        // dL/dT (upper 2x3): Vrk[k][l] symmetric
        const float dL_dT00 = 2 * TV00 * dL_da + TV10 * dL_db;
        const float dL_dT01 = 2 * TV01 * dL_da + TV11 * dL_db;
        const float dL_dT02 = 2 * TV02 * dL_da + TV12 * dL_db;
        const float dL_dT10 = 2 * TV10 * dL_dc + TV00 * dL_db;
        const float dL_dT11 = 2 * TV11 * dL_dc + TV01 * dL_db;
        const float dL_dT12 = 2 * TV12 * dL_dc + TV02 * dL_db;
        // dL/dJ (non-zero entries), T = W * J
        const float dL_dJ00 = W00 * dL_dT00 + W01 * dL_dT01 + W02 * dL_dT02;
        const float dL_dJ02 = W20 * dL_dT00 + W21 * dL_dT01 + W22 * dL_dT02;
        const float dL_dJ11 = W10 * dL_dT10 + W11 * dL_dT11 + W12 * dL_dT12;
        const float dL_dJ12 = W20 * dL_dT10 + W21 * dL_dT11 + W22 * dL_dT12;
        const float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float dL_dtx = x_grad_mul * -h_x * itz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -h_y * itz2 * dL_dJ12;
        const float dL_dtz = -h_x * itz2 * dL_dJ00 - h_y * itz2 * dL_dJ11 + (2 * h_x * tx) * itz3 * dL_dJ02 + (2 * h_y * ty) * itz3 * dL_dJ12;
        // back through t = view * mean (transformVec4x3Transpose, auxiliary.h:88-97)
        float dmx = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
        float dmy = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
        float dmz = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;

        // ---- projection part of preprocessCUDA (backward.cu:371-391) -----------------------------
        {
            const float m_hom_w = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
            const float m_w = 1.0f / (m_hom_w + 0.0000001f);
            const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
            const float gx2 = a2.z, gy2 = a2.w;
            dmx += (proj[0] * m_w - proj[3] * mul1) * gx2 + (proj[1] * m_w - proj[3] * mul2) * gy2;
            dmy += (proj[4] * m_w - proj[7] * mul1) * gx2 + (proj[5] * m_w - proj[7] * mul2) * gy2;
            dmz += (proj[8] * m_w - proj[11] * mul1) * gx2 + (proj[9] * m_w - proj[11] * mul2) * gy2;
        }
        o_m3[0] = dmx;
        o_m3[1] = dmy;
        o_m3[2] = dmz;

        // ---- backward of computeCov3D (backward.cu:278-341) --------------------------------------
        if (!(from_scale_rot && scales != nullptr)) {
            if (dL_dscale) { o_scale[0] = 0.f; o_scale[1] = 0.f; o_scale[2] = 0.f; }
            if (dL_drot) reinterpret_cast<float4*>(dL_drot)[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            // R[c][r] as the glm ctor fills it (columns)
            const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - r * z), R02 = 2.f * (x * z + r * y);
            const float R10 = 2.f * (x * y + r * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - r * x);
            const float R20 = 2.f * (x * z - r * y), R21 = 2.f * (y * z + r * x), R22 = 1.f - 2.f * (x * x + y * y);
            const float sx = mod * s0, sy = mod * s1, sz = mod * s2;
            // M = S * R : M[c][r] = s_r R[c][r]
            const float M00 = sx * R00, M01 = sy * R01, M02 = sz * R02;
            const float M10 = sx * R10, M11 = sy * R11, M12 = sz * R12;
            const float M20 = sx * R20, M21 = sy * R21, M22 = sz * R22;
            // dL_dSigma (symmetric, off-diagonals halved)
            const float D00 = dcov[0], D01 = 0.5f * dcov[1], D02 = 0.5f * dcov[2];
            const float D11 = dcov[3], D12 = 0.5f * dcov[4], D22 = dcov[5];
            // dL_dM = 2 * M * dL_dSigma :  X[j][i] = sum_k (2M)[k][i] * D[j][k]
            const float X00 = 2.f * (M00 * D00 + M10 * D01 + M20 * D02);
            const float X01 = 2.f * (M01 * D00 + M11 * D01 + M21 * D02);
            const float X02 = 2.f * (M02 * D00 + M12 * D01 + M22 * D02);
            const float X10 = 2.f * (M00 * D01 + M10 * D11 + M20 * D12);
            const float X11 = 2.f * (M01 * D01 + M11 * D11 + M21 * D12);
            const float X12 = 2.f * (M02 * D01 + M12 * D11 + M22 * D12);
            const float X20 = 2.f * (M00 * D02 + M10 * D12 + M20 * D22);
            const float X21 = 2.f * (M01 * D02 + M11 * D12 + M21 * D22);
            const float X22 = 2.f * (M02 * D02 + M12 * D12 + M22 * D22);
            // Rt = transpose(R): Rt[c][r] = R[r][c];  dL_dMt = transpose(dL_dM): Y[c][r] = X[r][c]
            // dL_dscale.k = dot(Rt[k], Y[k]) = sum_r R[r][k] * X[r][k]
            o_scale[0] = R00 * X00 + R10 * X10 + R20 * X20;
            o_scale[1] = R01 * X01 + R11 * X11 + R21 * X21;
            o_scale[2] = R02 * X02 + R12 * X12 + R22 * X22;
            // Y[k] *= s_k   -> Y[c][r] = s_c * X[r][c]
            const float Y00 = sx * X00, Y01 = sx * X10, Y02 = sx * X20;
            const float Y10 = sy * X01, Y11 = sy * X11, Y12 = sy * X21;
            const float Y20 = sz * X02, Y21 = sz * X12, Y22 = sz * X22;
            float4 dq;
            dq.x = 2 * z * (Y01 - Y10) + 2 * y * (Y20 - Y02) + 2 * x * (Y12 - Y21);
            dq.y = 2 * y * (Y10 + Y01) + 2 * z * (Y20 + Y02) + 2 * r * (Y12 - Y21) - 4 * x * (Y22 + Y11);
            dq.z = 2 * x * (Y10 + Y01) + 2 * r * (Y20 - Y02) + 2 * z * (Y12 + Y21) - 4 * y * (Y22 + Y00);
            dq.w = 2 * r * (Y01 - Y10) + 2 * x * (Y20 + Y02) + 2 * y * (Y12 + Y21) - 4 * z * (Y11 + Y00);
            reinterpret_cast<float4*>(dL_drot)[idx] = dq;
        }
    } while (false);

    __syncthreads();
    gh_span_store(g_color, s_color, GH_NUM_CHANNELS * n);
    gh_span_store(g_m2, s_m2, 3 * n);
    gh_span_store(g_m3, s_m3, 3 * n);
    gh_span_store(g_cov, s_cov, 6 * n);
    if (g_scale) gh_span_store(g_scale, s_scale, 3 * n);
}

}  // namespace

void gh_launch_preprocess_backward(int P, const float* means3D, const int* radii,
                                   const float* scales, float scale_modifier, const float* rotations,
                                   const float* cov3D_precomp, const float* conic_precomp,
                                   const float* viewmatrix, const float* projmatrix,
                                   int W, int H, float tan_fovx, float tan_fovy,
                                   const float* acc16, float* dL_dmean2D, float* dL_dconic,
                                   float* dL_dopacity, float* dL_dcolor,
                                   float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot,
                                   cudaStream_t stream)
{
    if (conic_precomp != nullptr) return;   // reference: geometry backward is a no-op in this mode (caller unpacks)
    const float focal_y = H / (2.0f * tan_fovy);
    const float focal_x = W / (2.0f * tan_fovx);
    gh_launch_pdl(gh_preprocess_backward_kernel, (P + GH_PBWD_THREADS - 1) / GH_PBWD_THREADS, GH_PBWD_THREADS, 0, stream,
        P, means3D, radii, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix,
        focal_x, focal_y, tan_fovx, tan_fovy, acc16, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor,
        dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot);
}
