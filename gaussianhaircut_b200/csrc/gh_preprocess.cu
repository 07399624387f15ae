// Stage 1: per-Gaussian preprocess (near cull, projection, 3-D covariance from scale/quaternion,
// EWA 2-D covariance or caller-supplied conic, splat radius, tile rectangle) fused with the per-tile
// instance histogram that drives the bucketed binning of stage 2.
//
// Semantics follow the reference kernel preprocessCUDA (cuda_rasterizer/forward.cu:155-282) and
// its helpers in_frustum / computeCov3D / computeCov2D / ndc2Pix / getRect
// (auxiliary.h:139-164, forward.cu:118-152, :74-113, auxiliary.h:41-56); rounding order is the
// reference's (see gh_common.cuh).  Layout, fusion and the histogram are new.
#include "gh_common.cuh"
#include "gh_kernels.h"

namespace {

__global__ void __launch_bounds__(128, 12)
gh_preprocess_kernel(int P,
                     const float* __restrict__ means3D,
                     const float* __restrict__ scales, float scale_modifier,
                     const float* __restrict__ rotations,
                     const float* __restrict__ opacities,
                     const float* __restrict__ cov3D_precomp,
                     const float* __restrict__ conic_precomp,
                     const float* __restrict__ viewmatrix,
                     const float* __restrict__ projmatrix,
                     int W, int H, float tan_fovx, float tan_fovy, float focal_x, float focal_y,
                     int* __restrict__ radii,
                     GhGeo* __restrict__ geo, float* __restrict__ depth,
                     uint32_t* __restrict__ tile_count, GhCtrl* __restrict__ ctrl,
                     int gx, int gy, int prefiltered)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = idx < P;
    // the inputs may come from the kernel just before (the optimizer, the projection), and the tile histogram from the
    // memset before this launch: nothing is read before the wait
    gh_pdl_wait();
    gh_pdl_trigger();

    // radius 0 <=> "not rendered" (forward.cu:190-191)
    int out_radius = 0;
    int rect_minx = 0, rect_miny = 0, rect_maxx = 0, rect_maxy = 0;
    GhGeo g = gh_geo_not_rendered();
    float zview = 0.f;

    float px = 0.f, py = 0.f, pz = 0.f;
    if (valid) { px = means3D[3 * idx + 0]; py = means3D[3 * idx + 1]; pz = means3D[3 * idx + 2]; }
    const float* vm = viewmatrix;
    const float* pm = projmatrix;

    do {
        if (!valid) break;
        // near cull only (auxiliary.h:154); NDC projection, always recomputed (forward.cu:201-206: the means2D
        // argument is never read)
        float projx, projy;
        if (!gh_pre_project(px, py, pz, vm, pm, zview, projx, projy)) {
            if (prefiltered) atomicOr(&ctrl->err_flags, GH_ERR_PREFILTERED);
            break;
        }

        float covx, covz, det, conx, cony, conz;
        if (conic_precomp == nullptr) {
            float c3[6];
            if (cov3D_precomp != nullptr) {
#pragma unroll
                for (int k = 0; k < 6; k++) c3[k] = cov3D_precomp[6 * idx + k];
            } else {
                const float4 q = reinterpret_cast<const float4*>(rotations)[idx];
                gh_cov3d(scales[3 * idx + 0], scales[3 * idx + 1], scales[3 * idx + 2], scale_modifier,
                         q.x, q.y, q.z, q.w, c3);
            }
            // computeCov2D (forward.cu:74-113)
            const float v0 = __ldg(vm + 0), v1 = __ldg(vm + 1), v2 = __ldg(vm + 2);
            const float v4 = __ldg(vm + 4), v5 = __ldg(vm + 5), v6 = __ldg(vm + 6);
            const float v8 = __ldg(vm + 8), v9 = __ldg(vm + 9), v10 = __ldg(vm + 10);
            const float tx0 = GH_ADD(__ldg(vm + 12), GH_FMA(pz, v8, GH_FMA(px, v0, GH_MUL(py, v4))));
            const float ty0 = GH_ADD(__ldg(vm + 13), GH_FMA(pz, v9, GH_FMA(px, v1, GH_MUL(py, v5))));
            const float tz = zview;
            const float limx = GH_MUL(tan_fovx, 1.3f), limy = GH_MUL(tan_fovy, 1.3f);
            const float txtz = GH_DIV(tx0, tz), tytz = GH_DIV(ty0, tz);
            const float tx = GH_MUL(fminf(limx, fmaxf(-limx, txtz)), tz);
            const float ty = GH_MUL(fminf(limy, fmaxf(-limy, tytz)), tz);
            const float tz2 = GH_MUL(tz, tz);
            const float J00 = GH_DIV(focal_x, tz);
            const float J02 = -GH_DIV(GH_MUL(focal_x, tx), tz2);
            const float J11 = GH_DIV(focal_y, tz);
            const float J12 = -GH_DIV(GH_MUL(focal_y, ty), tz2);
            // T = W * J (glm), W columns = rows of the upper 3x3 of the (transposed) view matrix
            const float T00 = GH_FMA(v2, J02, GH_MUL(v0, J00));
            const float T01 = GH_FMA(v6, J02, GH_MUL(v4, J00));
            const float T02 = GH_FMA(v10, J02, GH_MUL(v8, J00));
            const float T10 = GH_FMA(v2, J12, GH_MUL(v1, J11));
            const float T11 = GH_FMA(v6, J12, GH_MUL(v5, J11));
            const float T12 = GH_FMA(v10, J12, GH_MUL(v9, J11));
            // A = transpose(T) * transpose(Vrk)
            const float A00 = GH_FMA(T02, c3[2], GH_FMA(T00, c3[0], GH_MUL(T01, c3[1])));
            const float A01 = GH_FMA(T12, c3[2], GH_FMA(T10, c3[0], GH_MUL(T11, c3[1])));
            const float A10 = GH_FMA(T02, c3[4], GH_FMA(T00, c3[1], GH_MUL(T01, c3[3])));
            const float A11 = GH_FMA(T12, c3[4], GH_FMA(T10, c3[1], GH_MUL(T11, c3[3])));
            const float A20 = GH_FMA(T02, c3[5], GH_FMA(T00, c3[2], GH_MUL(T01, c3[4])));
            const float A21 = GH_FMA(T12, c3[5], GH_FMA(T10, c3[2], GH_MUL(T11, c3[4])));
            // cov = A * T, +0.3 low-pass on the diagonal
            const float c00 = GH_FMA(T02, A20, GH_FMA(T00, A00, GH_MUL(T01, A10)));
            const float c01 = GH_FMA(T02, A21, GH_FMA(T00, A01, GH_MUL(T01, A11)));
            const float c11 = GH_FMA(T12, A21, GH_FMA(T10, A01, GH_MUL(T11, A11)));
            covx = GH_ADD(c00, 0.3f);
            covz = GH_ADD(c11, 0.3f);
            det = GH_FMA(covx, covz, -GH_MUL(c01, c01));
            if (det == 0.0f) break;
            const float det_inv = GH_RCP(det);
            conx = GH_MUL(covz, det_inv);
            cony = GH_MUL(det_inv, -c01);
            conz = GH_MUL(covx, det_inv);
        } else {
            // caller-supplied conic: invert it to size the splat (forward.cu:238-248)
            conx = conic_precomp[3 * idx + 0];
            cony = conic_precomp[3 * idx + 1];
            conz = conic_precomp[3 * idx + 2];
            if (!gh_pre_from_conic(conx, cony, conz, covx, covz, det)) break;
        }
        out_radius = gh_pre_finish(covx, covz, det, conx, cony, conz, projx, projy, opacities[idx], W, H, gx, gy,
                                   rect_minx, rect_miny, rect_maxx, rect_maxy, g);
    } while (false);

    if (valid) {
        radii[idx] = out_radius;
        depth[idx] = zview;
        float4* gp = reinterpret_cast<float4*>(geo + idx);
        gp[0] = make_float4(g.x, g.y, g.ca, g.cb);
        gp[1] = make_float4(g.cc, g.op, g.thr, g.pd);
    }

    gh_warp_tile_histogram(rect_minx, rect_miny, rect_maxx, rect_maxy, gx, tile_count);
}

// markVisible (rasterizer_impl.cu:54-66): near-plane test only.
__global__ void gh_check_frustum_kernel(int P, const float* __restrict__ means3D,
                                        const float* __restrict__ vm, bool* __restrict__ present)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float px = means3D[3 * idx + 0], py = means3D[3 * idx + 1], pz = means3D[3 * idx + 2];
    const float zview = GH_ADD(__ldg(vm + 14), GH_FMA(pz, __ldg(vm + 10), GH_FMA(px, __ldg(vm + 2), GH_MUL(py, __ldg(vm + 6)))));
    present[idx] = !(zview <= 0.2f);
}

}  // namespace

void gh_launch_preprocess(int P, const float* means3D, const float* scales, float scale_modifier,
                          const float* rotations, const float* opacities, const float* cov3D_precomp,
                          const float* conic_precomp, const float* viewmatrix, const float* projmatrix,
                          int W, int H, float tan_fovx, float tan_fovy, int* radii,
                          GhGeomWS geom, GhImgWS img, int gx, int gy, int prefiltered, cudaStream_t stream)
{
    const float focal_y = H / (2.0f * tan_fovy);   // rasterizer_impl.cu:224-225
    const float focal_x = W / (2.0f * tan_fovx);
    gh_launch_pdl(gh_preprocess_kernel, (P + 127) / 128, 128, 0, stream,
        P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp, conic_precomp,
        viewmatrix, projmatrix, W, H, tan_fovx, tan_fovy, focal_x, focal_y, radii,
        geom.geo, geom.depth, img.tile_count, img.ctrl, gx, gy, prefiltered);
}

void gh_launch_mark_visible(int P, const float* means3D, const float* viewmatrix, bool* present,
                            cudaStream_t stream)
{
    gh_check_frustum_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
}
