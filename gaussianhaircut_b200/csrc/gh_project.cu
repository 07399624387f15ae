// "Next" row 1 (SURVEY.md 8f-1): the caller-side projection preamble as ONE forward and ONE backward kernel.
//
// Every training iteration the reference's `render()` / `render_hair()` restate stage 1 of the rasterizer in
// PyTorch before calling it (~100 elementwise / bmm kernels with (P,3,3) temporaries and six boolean-mask
// gathers): src/gaussian_renderer/__init__.py:29-83,122-186 calling
//   GaussianModel.get_conic / get_covariance_2d / get_covariance   src/scene/gaussian_model.py:230-315
//   get_mean_2d :317-337, get_depths :339-342, get_direction_2d :344-393, filter_points :143-228
//   eval_sh                                                         src/utils/sh_utils.py:57-112
//   build_rotation (normalises the quaternion)                      src/utils/general_utils.py:79-109
// (the strand models restate the same functions: src/scene/gaussian_model_latent_strands.py:150-440).
// Here one thread owns one Gaussian from the RAW model parameters to everything the rasterizer consumes
// (conic, NDC mean, opacity, the 10-channel feature row) and back -- including the gradients w.r.t. the
// camera (world-view matrix, full projection matrix, camera centre, tan(fov/2)), which the reference
// obtains through autograd because cameras are trainable (src/scene/cameras.py:124-150).
//
// Row-vector convention of the Python code: t = x . V[:3,:3] + V[3,:3],  h = x . Pm[:3,:] + Pm[3,:].
//   s = exp(log s) * mod (or the activated scale),  R = build_rotation(q / |q|),  Sigma = sum_i s_i^2 R[i]^T R[i]
//   u0 = T[:,0], u1 = T[:,1] with T = V[:3,:3] @ J  (J from the clamped view-space position)
//   a = sum_i s_i^2 (R[i].u0)^2 + 0.3,  b = sum_i s_i^2 (R[i].u0)(R[i].u1),  c = sum_i s_i^2 (R[i].u1)^2 + 0.3
//   conic = (c, -b, a) / (ac - b^2 + eps)        eps = 1e-12 (GaussianModel :312) or 1e-7 (strand models :355)
//   dir2D = d3 . T,  d3 = s_max R[argmax s] (GaussianModel :385-391) or normalize(dir) (strand models :437-438)
//   feature row = [max(SH(v)+0.5, 0), label, 1, dir2D (3), orientation confidence, view depth]
// Gaussians failing the caller's prefilter (filter_points: near plane, det != 0, empty tile rectangle) are
// not compacted away: they get conic = 0, which the rasterizer drops (zero determinant, forward.cu:243-245),
// so indices stay the model's own (radii / visibility need no scatter) and every gradient row is written.
//
// f_rest rows are 180 bytes (45 floats): a CTA stages its 128 rows through shared memory with coalesced
// 128-bit loads / stores; the odd row stride (45 words) makes the per-thread accesses conflict free.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"
#include "gh_project_math.h"

namespace {

#define GH_PJ_THREADS 128

// stage the CTA's f_rest rows (or their gradients) through shared memory with coalesced 128-bit accesses
__device__ __forceinline__ void gh_rest_load(float* s_rest, const float* __restrict__ f_rest, int P, int row0) {
    const size_t base = (size_t)row0 * GH_PJ_REST;
    const size_t total = (size_t)P * GH_PJ_REST;
    const int n = (int)min((size_t)GH_PJ_THREADS * GH_PJ_REST, total - base);
    if ((reinterpret_cast<size_t>(f_rest + base) & 15) == 0) {
        const float4* src = reinterpret_cast<const float4*>(f_rest + base);
        for (int v = threadIdx.x; v < n / 4; v += GH_PJ_THREADS) reinterpret_cast<float4*>(s_rest)[v] = src[v];
        for (int e = (n & ~3) + threadIdx.x; e < n; e += GH_PJ_THREADS) s_rest[e] = f_rest[base + e];
    } else {
        for (int e = threadIdx.x; e < n; e += GH_PJ_THREADS) s_rest[e] = f_rest[base + e];
    }
}
__device__ __forceinline__ void gh_rest_store(const float* s_rest, float* __restrict__ out, int P, int row0) {
    const size_t base = (size_t)row0 * GH_PJ_REST;
    const size_t total = (size_t)P * GH_PJ_REST;
    const int n = (int)min((size_t)GH_PJ_THREADS * GH_PJ_REST, total - base);
    if ((reinterpret_cast<size_t>(out + base) & 15) == 0) {
        float4* dst = reinterpret_cast<float4*>(out + base);
        for (int v = threadIdx.x; v < n / 4; v += GH_PJ_THREADS) dst[v] = reinterpret_cast<const float4*>(s_rest)[v];
        for (int e = (n & ~3) + threadIdx.x; e < n; e += GH_PJ_THREADS) out[base + e] = s_rest[e];
    } else {
        for (int e = threadIdx.x; e < n; e += GH_PJ_THREADS) out[base + e] = s_rest[e];
    }
}

// ------------------------------------------------------------------------------------------------ forward
// BIN: also run stage 1 of the rasterizer for the Gaussian just projected (what gh_preprocess_kernel does when it is
// handed the conic): splat radius, tile rectangle, the 32-byte state record of the blend kernels, depth, and the
// per-tile instance histogram -- the conic, mean and opacity are still in registers, so the rasterizer's own
// preprocess launch (and its re-read of 28 bytes per Gaussian) disappears from a fused render.  Same device functions
// as gh_preprocess_kernel (gh_common.cuh), hence bit-identical radii / records / keys.
// STRAND: Gaussian i is a polyline segment whose scales and rotation come from dirs[i] (gh_proj_geometry).
template <bool BIN, bool STRAND>
__device__ __forceinline__ void
gh_project_forward_body(const GhProjArgs& A, float* __restrict__ means2D, float* __restrict__ colors,
                        float* __restrict__ opac_out, float* __restrict__ conic_out, float* __restrict__ cov3D_out,
                        unsigned char* __restrict__ mask_out,
                        int* __restrict__ radii, GhGeo* __restrict__ geo, float* __restrict__ depth,
                        uint32_t* __restrict__ tile_count, int gx, int gy)
{
    __shared__ __align__(16) float s_rest[GH_PJ_THREADS * GH_PJ_REST];
    const int row0 = blockIdx.x * GH_PJ_THREADS;
    const int i = row0 + threadIdx.x;
    if (A.sh_degree > 0) gh_rest_load(s_rest, A.f_rest, A.P, row0);
    __syncthreads();
    int rect_minx = 0, rect_miny = 0, rect_maxx = 0, rect_maxy = 0;
    if (i < A.P) {
        GhProjOut o;
        gh_project_forward_one<STRAND>(A, i, s_rest + threadIdx.x * GH_PJ_REST, cov3D_out != nullptr, o);
        means2D[3 * (size_t)i] = o.m2[0]; means2D[3 * (size_t)i + 1] = o.m2[1]; means2D[3 * (size_t)i + 2] = o.m2[2];
        conic_out[3 * (size_t)i] = o.conic[0]; conic_out[3 * (size_t)i + 1] = o.conic[1]; conic_out[3 * (size_t)i + 2] = o.conic[2];
        mask_out[i] = o.visible ? 1 : 0;
        opac_out[i] = o.opacity;
        if (cov3D_out) {
#pragma unroll
            for (int k = 0; k < 6; k++) cov3D_out[6 * (size_t)i + k] = o.cov3D[k];
        }
        float2* crow = reinterpret_cast<float2*>(colors + (size_t)i * GH_NUM_CHANNELS);
#pragma unroll
        for (int k = 0; k < GH_NUM_CHANNELS / 2; k++) crow[k] = make_float2(o.color[2 * k], o.color[2 * k + 1]);
        if (BIN) {
            int out_radius = 0;
            GhGeo g = gh_geo_not_rendered();
            float zview = 0.f, projx, projy, covx, covz, det;
            const float px = A.xyz[3 * (size_t)i], py = A.xyz[3 * (size_t)i + 1], pz = A.xyz[3 * (size_t)i + 2];
            // (culled Gaussians carry conic = 0 -> singular -> radius 0, exactly as in the two-kernel path)
            if (gh_pre_project(px, py, pz, A.V, A.Pm, zview, projx, projy) &&
                gh_pre_from_conic(o.conic[0], o.conic[1], o.conic[2], covx, covz, det))
                out_radius = gh_pre_finish(covx, covz, det, o.conic[0], o.conic[1], o.conic[2], projx, projy, o.opacity,
                                           A.W, A.H, gx, gy, rect_minx, rect_miny, rect_maxx, rect_maxy, g);
            radii[i] = out_radius;
            depth[i] = zview;
            float4* gp = reinterpret_cast<float4*>(geo + i);
            gp[0] = make_float4(g.x, g.y, g.ca, g.cb);
            gp[1] = make_float4(g.cc, g.op, g.thr, g.pd);
        }
    }
    if (BIN) gh_warp_tile_histogram(rect_minx, rect_miny, rect_maxx, rect_maxy, gx, tile_count);
}

template <bool BIN, bool STRAND>
__global__ void __launch_bounds__(GH_PJ_THREADS)
gh_project_forward_kernel(GhProjArgs A, float* __restrict__ means2D, float* __restrict__ colors,
                          float* __restrict__ opac_out, float* __restrict__ conic_out, float* __restrict__ cov3D_out,
                          unsigned char* __restrict__ mask_out,
                          int* __restrict__ radii, GhGeo* __restrict__ geo, float* __restrict__ depth,
                          uint32_t* __restrict__ tile_count, int gx, int gy)
{
    gh_project_forward_body<BIN, STRAND>(A, means2D, colors, opac_out, conic_out, cov3D_out, mask_out, radii, geo, depth,
                                         tile_count, gx, gy);
}

// The capturable first phase (gh_project_forward_binned_capturable): tan(fov / 2) is read from device memory, so that a
// captured launch serves every camera.  GaussianModel rows only.
__global__ void __launch_bounds__(GH_PJ_THREADS)
gh_project_forward_tan_kernel(GhProjArgs A, const float* __restrict__ tan_fov, float* __restrict__ means2D,
                              float* __restrict__ colors, float* __restrict__ opac_out, float* __restrict__ conic_out,
                              unsigned char* __restrict__ mask_out, int* __restrict__ radii, GhGeo* __restrict__ geo,
                              float* __restrict__ depth, uint32_t* __restrict__ tile_count, int gx, int gy)
{
    A.tanx = __ldg(tan_fov); A.tany = __ldg(tan_fov + 1);
    gh_project_forward_body<true, false>(A, means2D, colors, opac_out, conic_out, nullptr, mask_out, radii, geo, depth,
                                         tile_count, gx, gy);
}

// The strand rows of gh_hair_strands_forward_binned_capturable: gh_project_forward_tan_kernel for polyline segments.
// The caller offsets every output and workspace pointer by the head block's rows.
__global__ void __launch_bounds__(GH_PJ_THREADS)
gh_project_forward_strand_tan_kernel(GhProjArgs A, const float* __restrict__ tan_fov, float* __restrict__ means2D,
                                     float* __restrict__ colors, float* __restrict__ opac_out, float* __restrict__ conic_out,
                                     unsigned char* __restrict__ mask_out, int* __restrict__ radii, GhGeo* __restrict__ geo,
                                     float* __restrict__ depth, uint32_t* __restrict__ tile_count, int gx, int gy)
{
    A.tanx = __ldg(tan_fov); A.tany = __ldg(tan_fov + 1);
    gh_project_forward_body<true, true>(A, means2D, colors, opac_out, conic_out, nullptr, mask_out, radii, geo, depth,
                                        tile_count, gx, gy);
}

// ------------------------------------------------------------------------------------------------ backward
// Incoming gradients: either the four API-shaped tensors of gh_backward (dL_dmean2D (P,3) NDC units,
// dL_dconic (P,4) = (d/da, HALF d/db, unused, d/dc), dL_dcolor (P,10), dL_dopacity (P)), or -- when acc16 is
// given -- the blend backward's 64-byte accumulation records themselves (colors 0..9, mean2D x y, conic x y w,
// opacity), which skips the unpack kernel and its round trip through HBM.
// STRAND: the scale and rotation gradients are folded into d_dirs in registers; d_scaling / d_rotation are not written.
template <bool STRAND>
__device__ __forceinline__ void
gh_project_backward_body(const GhProjArgs& A, const unsigned char* __restrict__ mask,
                           const float* __restrict__ acc16,
                           const float* __restrict__ g_mean2D, const float* __restrict__ g_conic4,
                           const float* __restrict__ g_color, const float* __restrict__ g_opacity,
                           float* __restrict__ d_xyz, float* __restrict__ d_scaling, float* __restrict__ d_rotation,
                           float* __restrict__ d_dirs, float* __restrict__ d_fdc, float* __restrict__ d_frest,
                           float* __restrict__ d_opacity, float* __restrict__ d_label, float* __restrict__ d_conf,
                           float* __restrict__ d_mean2D_out,
                           float* __restrict__ cam_partial, unsigned int* __restrict__ cam_ticket,
                           float* __restrict__ d_cam,     // 16 V + 16 Pm + 3 campos + 2 tan, or NULL
                           unsigned int* __restrict__ nan_flag)   // set to 1 if any parameter gradient is NaN, or NULL
{
    __shared__ __align__(16) float s_rest[GH_PJ_THREADS * GH_PJ_REST];
    __shared__ float s_cam[GH_PJ_THREADS / 32][GH_PJ_NCAM];
    const int row0 = blockIdx.x * GH_PJ_THREADS;
    const int i = row0 + threadIdx.x;
    const bool want_cam = (d_cam != nullptr);
    if (A.sh_degree > 0) gh_rest_load(s_rest, A.f_rest, A.P, row0);
    __syncthreads();

    float cam[GH_PJ_NCAM];
#pragma unroll
    for (int k = 0; k < GH_PJ_NCAM; k++) cam[k] = 0.f;
    GhProjGradOut go;
#pragma unroll
    for (int k = 0; k < 3; k++) { go.xyz[k] = 0.f; go.scaling[k] = 0.f; go.dirs[k] = 0.f; go.f_dc[k] = 0.f; }
#pragma unroll
    for (int k = 0; k < 4; k++) go.rotation[k] = 0.f;
    go.opacity = 0.f; go.label = 0.f; go.conf = 0.f;
#pragma unroll
    for (int k = 0; k < GH_PJ_REST; k++) go.rest[k] = 0.f;

    if (i < A.P) {
        const bool live = (mask[i] != 0);
        GhProjGradIn gi;
        gi.m2x = 0.f; gi.m2y = 0.f; gi.con[0] = 0.f; gi.con[1] = 0.f; gi.con[2] = 0.f; gi.opacity = 0.f;
#pragma unroll
        for (int k = 0; k < GH_NUM_CHANNELS; k++) gi.color[k] = 0.f;
        if (live) {
            if (acc16) {
                const float4* rec = reinterpret_cast<const float4*>(acc16 + (size_t)i * 16);
                const float4 a0 = rec[0], a1 = rec[1], a2 = rec[2], a3 = rec[3];
                gi.color[0] = a0.x; gi.color[1] = a0.y; gi.color[2] = a0.z; gi.color[3] = a0.w; gi.color[4] = a1.x; gi.color[5] = a1.y;
                gi.color[6] = a1.z; gi.color[7] = a1.w; gi.color[8] = a2.x; gi.color[9] = a2.y;
                gi.m2x = a2.z; gi.m2y = a2.w; gi.con[0] = a3.x; gi.con[1] = 2.f * a3.y; gi.con[2] = a3.z; gi.opacity = a3.w;
            } else {
                gi.m2x = g_mean2D[3 * (size_t)i]; gi.m2y = g_mean2D[3 * (size_t)i + 1];
                const float4 c4 = reinterpret_cast<const float4*>(g_conic4)[i];
                gi.con[0] = c4.x; gi.con[1] = 2.f * c4.y; gi.con[2] = c4.w;     // python restack [g00, 2 g01, g11] (__init__.py:149-153)
                gi.opacity = g_opacity[i];
                const float2* cr = reinterpret_cast<const float2*>(g_color + (size_t)i * GH_NUM_CHANNELS);
#pragma unroll
                for (int k = 0; k < GH_NUM_CHANNELS / 2; k++) { const float2 v = cr[k]; gi.color[2 * k] = v.x; gi.color[2 * k + 1] = v.y; }
            }
            gh_project_backward_one<STRAND>(A, i, s_rest + threadIdx.x * GH_PJ_REST, gi, go, cam);
        }
        // every row of every per-Gaussian gradient is written (zeros for culled Gaussians)
        if (d_mean2D_out) { d_mean2D_out[3 * (size_t)i] = gi.m2x; d_mean2D_out[3 * (size_t)i + 1] = gi.m2y; d_mean2D_out[3 * (size_t)i + 2] = 0.f; }
        d_xyz[3 * (size_t)i] = go.xyz[0]; d_xyz[3 * (size_t)i + 1] = go.xyz[1]; d_xyz[3 * (size_t)i + 2] = go.xyz[2];
        if (!STRAND) {
            d_scaling[3 * (size_t)i] = go.scaling[0]; d_scaling[3 * (size_t)i + 1] = go.scaling[1]; d_scaling[3 * (size_t)i + 2] = go.scaling[2];
            reinterpret_cast<float4*>(d_rotation)[i] = make_float4(go.rotation[0], go.rotation[1], go.rotation[2], go.rotation[3]);
        }
        if (d_dirs) { d_dirs[3 * (size_t)i] = go.dirs[0]; d_dirs[3 * (size_t)i + 1] = go.dirs[1]; d_dirs[3 * (size_t)i + 2] = go.dirs[2]; }
        d_fdc[3 * (size_t)i] = go.f_dc[0]; d_fdc[3 * (size_t)i + 1] = go.f_dc[1]; d_fdc[3 * (size_t)i + 2] = go.f_dc[2];
        if (d_opacity) d_opacity[i] = go.opacity;
        if (d_label) d_label[i] = go.label;
        if (d_conf) d_conf[i] = go.conf;
    }
    if (nan_flag != nullptr) {
        // the optimizer's NaN guard (train_gaussians.py:174-181) rides on the kernel that produces the gradients
        float acc = go.opacity + go.label + go.conf;
#pragma unroll
        for (int k = 0; k < 3; k++) acc += go.xyz[k] + go.scaling[k] + go.dirs[k] + go.f_dc[k];
#pragma unroll
        for (int k = 0; k < 4; k++) acc += go.rotation[k];
#pragma unroll
        for (int k = 0; k < GH_PJ_REST; k++) acc += go.rest[k];
        // a sum is NaN iff a term is NaN or +inf and -inf meet: both must stop the step
        if (__any_sync(0xffffffffu, acc != acc) && (threadIdx.x & 31) == 0) atomicOr(nan_flag, 1u);
    }
    // f_rest gradients leave through shared memory (coalesced 128-bit stores)
    __syncthreads();                                   // every thread is done reading its coefficients
    if (i < A.P) {
        float* row = s_rest + threadIdx.x * GH_PJ_REST;
#pragma unroll
        for (int e = 0; e < GH_PJ_REST; e++) row[e] = go.rest[e];
    }
    __syncthreads();
    gh_rest_store(s_rest, d_frest, A.P, row0);

    if (!want_cam) return;
    // ---- camera gradients: warp shuffle -> CTA partial -> the last CTA sums all partials in double, in order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < GH_PJ_NCAM; k++) {
        float v = cam[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_cam[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < GH_PJ_NCAM) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < GH_PJ_THREADS / 32; w++) v += s_cam[w][threadIdx.x];
        cam_partial[(size_t)blockIdx.x * GH_PJ_NCAM + threadIdx.x] = v;
    }
    __threadfence();
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(cam_ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ double s_sum[GH_PJ_THREADS / 32][GH_PJ_NCAM];
    // warp w sums blocks w, w+4, ...; lane k < 29 owns accumulator k: a fixed order, hence deterministic
    if (lane < GH_PJ_NCAM) {
        double acc = 0.0;
        for (unsigned int b = warp; b < gridDim.x; b += GH_PJ_THREADS / 32) acc += (double)__ldcg(cam_partial + (size_t)b * GH_PJ_NCAM + lane);
        s_sum[warp][lane] = acc;
    }
    __syncthreads();
    if (threadIdx.x < GH_PJ_NCAM) {
        double acc = 0.0;
        for (int w = 0; w < GH_PJ_THREADS / 32; w++) acc += s_sum[w][threadIdx.x];
        const int k = threadIdx.x;
        const float v = (float)acc;
        if (k < 12) d_cam[4 * (k / 3) + (k % 3)] = v;                                  // V[i][j], j < 3
        else if (k < 24) { const int q = k - 12; const int col = q % 3; d_cam[16 + 4 * (q / 3) + (col == 2 ? 3 : col)] = v; }   // Pm[i][0,1,3]
        else if (k < 27) d_cam[32 + (k - 24)] = v;
        else d_cam[35 + (k - 27)] = v;
    }
    if (threadIdx.x == 0) {
        // entries that never receive a gradient
        d_cam[3] = 0.f; d_cam[7] = 0.f; d_cam[11] = 0.f; d_cam[15] = 0.f;
        d_cam[16 + 2] = 0.f; d_cam[16 + 6] = 0.f; d_cam[16 + 10] = 0.f; d_cam[16 + 14] = 0.f;
        *cam_ticket = 0u;
    }
}

template <bool STRAND>
__global__ void __launch_bounds__(GH_PJ_THREADS)
gh_project_backward_kernel(GhProjArgs A, const unsigned char* __restrict__ mask,
                           const float* __restrict__ acc16,
                           const float* __restrict__ g_mean2D, const float* __restrict__ g_conic4,
                           const float* __restrict__ g_color, const float* __restrict__ g_opacity,
                           float* __restrict__ d_xyz, float* __restrict__ d_scaling, float* __restrict__ d_rotation,
                           float* __restrict__ d_dirs, float* __restrict__ d_fdc, float* __restrict__ d_frest,
                           float* __restrict__ d_opacity, float* __restrict__ d_label, float* __restrict__ d_conf,
                           float* __restrict__ d_mean2D_out,
                           float* __restrict__ cam_partial, unsigned int* __restrict__ cam_ticket,
                           float* __restrict__ d_cam, unsigned int* __restrict__ nan_flag)
{
    gh_project_backward_body<STRAND>(A, mask, acc16, g_mean2D, g_conic4, g_color, g_opacity, d_xyz, d_scaling, d_rotation,
                                     d_dirs, d_fdc, d_frest, d_opacity, d_label, d_conf, d_mean2D_out, cam_partial,
                                     cam_ticket, d_cam, nan_flag);
}

// gh_project_backward_capturable: tan(fov / 2) from device memory, as in gh_project_forward_tan_kernel
template <bool STRAND>
__global__ void __launch_bounds__(GH_PJ_THREADS)
gh_project_backward_tan_kernel(GhProjArgs A, const float* __restrict__ tan_fov, const unsigned char* __restrict__ mask,
                               const float* __restrict__ acc16,
                               const float* __restrict__ g_mean2D, const float* __restrict__ g_conic4,
                               const float* __restrict__ g_color, const float* __restrict__ g_opacity,
                               float* __restrict__ d_xyz, float* __restrict__ d_scaling, float* __restrict__ d_rotation,
                               float* __restrict__ d_dirs, float* __restrict__ d_fdc, float* __restrict__ d_frest,
                               float* __restrict__ d_opacity, float* __restrict__ d_label, float* __restrict__ d_conf,
                               float* __restrict__ d_mean2D_out,
                               float* __restrict__ cam_partial, unsigned int* __restrict__ cam_ticket,
                               float* __restrict__ d_cam, unsigned int* __restrict__ nan_flag)
{
    A.tanx = __ldg(tan_fov); A.tany = __ldg(tan_fov + 1);
    gh_project_backward_body<STRAND>(A, mask, acc16, g_mean2D, g_conic4, g_color, g_opacity, d_xyz, d_scaling, d_rotation,
                                     d_dirs, d_fdc, d_frest, d_opacity, d_label, d_conf, d_mean2D_out, cam_partial,
                                     cam_ticket, d_cam, nan_flag);
}

int gh_proj_check(GhProjArgs& A, const char* who, bool strand)
{
    if (A.P <= 0 || A.W <= 0 || A.H <= 0) return gh_set_error(GH_E_INVALID_ARG, "%s: P, width, height must be positive", who);
    if (strand) {
        if (A.rotation) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode derives the rotation from dirs, rotation must be NULL", who);
        if (!A.dirs) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode needs dirs (the segment vectors)", who);
        if (!A.scaling) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode needs scaling = the strand thickness (one device float)", who);
        if (A.scale_act != 0 || A.dir_mode != 1) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode needs scale activation 0 and direction mode 1", who);
    }
    if (!A.xyz || !A.scaling || (!strand && !A.rotation) || !A.f_dc || !A.V || !A.Pm || !A.campos)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
    if (A.sh_degree < 0 || A.sh_degree > 3) return gh_set_error(GH_E_INVALID_ARG, "%s: sh_degree must be 0..3", who);
    if (A.sh_degree > 0 && !A.f_rest) return gh_set_error(GH_E_INVALID_ARG, "%s: features_rest required for sh_degree > 0", who);
    if ((size_t)A.rotation & 15) return gh_set_error(GH_E_INVALID_ARG, "%s: rotation must be 16-byte aligned", who);
    if (A.dir_mode == 1 && !A.dirs) return gh_set_error(GH_E_INVALID_ARG, "%s: dirs required for dir_mode 1", who);
    if ((A.opacity_act < 2 && !A.opacity) || (A.label_act < 2 && !A.label) || (A.conf_act < 2 && !A.conf))
        return gh_set_error(GH_E_INVALID_ARG, "%s: opacity / label / orient_conf pointer missing for the chosen activation", who);
    if (!(A.tanx > 0.f) || !(A.tany > 0.f)) return gh_set_error(GH_E_INVALID_ARG, "%s: tan_fov must be positive", who);
    return GH_OK;
}

GhProjArgs gh_proj_args(int P, int width, int height, const float* xyz, const float* scaling, const float* rotation,
                        const float* dirs, const float* f_dc, const float* f_rest, const float* opacity,
                        const float* label, const float* conf, const float* V, const float* Pm, const float* campos,
                        float tanx, float tany, float mod, int sh_degree, unsigned int flags, float det_eps)
{
    GhProjArgs A;
    A.P = P; A.W = width; A.H = height; A.mod = mod; A.det_eps = det_eps; A.tanx = tanx; A.tany = tany; A.sh_degree = sh_degree;
    A.scale_act = (int)(flags & 3u); A.opacity_act = (int)((flags >> 2) & 3u); A.label_act = (int)((flags >> 4) & 3u);
    A.conf_act = (int)((flags >> 6) & 3u); A.dir_mode = (int)((flags >> 8) & 3u);
    A.xyz = xyz; A.scaling = scaling; A.rotation = rotation; A.dirs = dirs; A.f_dc = f_dc; A.f_rest = f_rest;
    A.opacity = opacity; A.label = label; A.conf = conf; A.V = V; A.Pm = Pm; A.campos = campos;
    return A;
}

// flag bit 10: the strand instantiation (Gaussian i = segment i of a polyline, geometry derived from dirs[i])
bool gh_proj_strand(unsigned int flags) { return (flags >> 10) & 1u; }

// the row counts of the capturable hair entry points: n_head head rows, then `seg` segment rows; `counts` / `prod` name
// the segment counts and their product in the messages ("S and L" / "S * L" for polylines, "N" / "N" for given rows)
int gh_hair_rows_check(const char* who, int n_head, bool negative, unsigned long long seg, bool need_segments,
                       const char* counts, const char* prod)
{
    if (n_head < 0) return gh_set_error(GH_E_INVALID_ARG, "%s: n_head must not be negative", who);
    if (negative || (need_segments && seg == 0))
        return gh_set_error(GH_E_INVALID_ARG, "%s: %s must be %s", who, counts, need_segments ? "positive" : "non-negative");
    if (3ull * seg > 0x7fffffffull) return gh_set_error(GH_E_INVALID_ARG, "%s: %s overflows int (3 * %s must stay below 2^31)", who, prod, prod);
    if ((unsigned long long)n_head + seg > 0x7fffffffull) return gh_set_error(GH_E_INVALID_ARG, "%s: n_head + %s overflows int", who, prod);
    if (n_head == 0 && seg == 0) return gh_set_error(GH_E_INVALID_ARG, "%s: nothing to render (n_head == 0 and %s == 0)", who, prod);
    return GH_OK;
}

int gh_strand_rows_check(const char* who, int n_head, int S, int L, bool need_strands)
{
    return gh_hair_rows_check(who, n_head, S < 0 || L < 0, S < 0 || L < 0 ? 0ull : (unsigned long long)S * (unsigned long long)L,
                              need_strands, "S and L", "S * L");
}

int gh_segment_rows_check(const char* who, int n_head, int N, bool need_segments)
{
    return gh_hair_rows_check(who, n_head, N < 0, N < 0 ? 0ull : (unsigned long long)N, need_segments, "N", "N");
}

}  // namespace

extern "C" int gh_project_workspace_size(int P, size_t* bytes)
{
    gh_clear_error();
    if (P < 0 || !bytes) return gh_set_error(GH_E_INVALID_ARG, "gh_project_workspace_size: bad arguments");
    const size_t blocks = ((size_t)P + GH_PJ_THREADS - 1) / GH_PJ_THREADS;
    *bytes = 256 + blocks * GH_PJ_NCAM * sizeof(float);
    return GH_OK;
}

extern "C" int gh_project_forward(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, float* cov3D, unsigned char* visible,
    gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    GhProjArgs A = gh_proj_args(P, width, height, xyz, scaling, rotation, dirs, features_dc, features_rest, opacity, label,
                                orient_conf, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, scale_modifier, sh_degree, flags, det_eps);
    const bool strand = gh_proj_strand(flags);
    const int rc = gh_proj_check(A, "gh_project_forward", strand);
    if (rc != GH_OK) return rc;
    if (!means2D || !colors || !opacities || !conic || !visible) return gh_set_error(GH_E_INVALID_ARG, "gh_project_forward: missing output pointer");
    if ((size_t)colors & 7) return gh_set_error(GH_E_INVALID_ARG, "gh_project_forward: colors must be 8-byte aligned");
    auto kernel = strand ? gh_project_forward_kernel<false, true> : gh_project_forward_kernel<false, false>;
    kernel<<<(P + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
        A, means2D, colors, opacities, conic, cov3D, visible, nullptr, nullptr, nullptr, nullptr, 0, 0);
    return gh_launch_status("gh_project_forward", 1);
}

// gh_project_forward + the rasterizer's first phase (gh_forward_phase1, as in gh_forward_preprocess) in one pass over
// the Gaussians; continue with gh_forward_render.
extern "C" int gh_project_forward_binned(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, float* cov3D, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long binning_capacity,
    int* num_rendered, int* max_tile_len, int* emitted, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    GhProjArgs A = gh_proj_args(P, width, height, xyz, scaling, rotation, dirs, features_dc, features_rest, opacity, label,
                                orient_conf, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, scale_modifier, sh_degree, flags, det_eps);
    const bool strand = gh_proj_strand(flags);
    const int rc = gh_proj_check(A, "gh_project_forward_binned", strand);
    if (rc != GH_OK) return rc;
    if (!means2D || !colors || !opacities || !conic || !visible || !radii || !geom_buffer || !img_buffer || !num_rendered)
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_forward_binned: missing output pointer");
    if ((size_t)colors & 7) return gh_set_error(GH_E_INVALID_ARG, "gh_project_forward_binned: colors must be 8-byte aligned");
    const GhPhase1Bin emit{radii, binning_buffer, binning_capacity, emitted};
    const int rc_bin = gh_check_phase1_bin("gh_project_forward_binned", emit);
    if (rc_bin != GH_OK) return rc_bin;
    auto kernel = strand ? gh_project_forward_kernel<true, true> : gh_project_forward_kernel<true, false>;
    return gh_forward_phase1("gh_project_forward_binned", P, width, height, geom_buffer, img_buffer, num_rendered, max_tile_len,
                             0, stream, emit, [&](const GhGeomWS& geom, const GhImgWS& img, int gx, int gy) {
        kernel<<<(P + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
            A, means2D, colors, opacities, conic, cov3D, visible, radii, geom.geo, geom.depth, img.tile_count, gx, gy);
        gh_count_launches(1);
    });
}

extern "C" int gh_project_backward(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    const unsigned char* visible,
    const char* geom_buffer,
    const float* dL_dmeans2D, const float* dL_dconic, const float* dL_dcolors, const float* dL_dopacity,
    float* d_xyz, float* d_scaling, float* d_rotation, float* d_dirs, float* d_features_dc, float* d_features_rest,
    float* d_opacity, float* d_label, float* d_orient_conf, float* d_means2D, float* d_camera,
    unsigned int* nan_flag, void* workspace, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    GhProjArgs A = gh_proj_args(P, width, height, xyz, scaling, rotation, dirs, features_dc, features_rest, opacity, label,
                                orient_conf, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, scale_modifier, sh_degree, flags, det_eps);
    const bool strand = gh_proj_strand(flags);
    const int rc = gh_proj_check(A, "gh_project_backward", strand);
    if (rc != GH_OK) return rc;
    if (strand && (d_scaling || d_rotation))
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: strand mode folds scale and rotation gradients into d_dirs, d_scaling / d_rotation must be NULL");
    if (strand && !d_dirs)
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: strand mode needs d_dirs");
    if (!visible || !d_xyz || (!strand && (!d_scaling || !d_rotation)) || !d_features_dc || !d_features_rest)
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: missing mandatory pointer");
    if (geom_buffer == nullptr && (!dL_dmeans2D || !dL_dconic || !dL_dcolors || !dL_dopacity))
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: pass the geometry workspace of gh_backward or the four incoming gradients");
    if (((size_t)d_rotation & 15) || (dL_dconic && ((size_t)dL_dconic & 15)) || (dL_dcolors && ((size_t)dL_dcolors & 7)))
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: d_rotation / dL_dconic must be 16-byte, dL_dcolors 8-byte aligned");
    if (d_camera != nullptr && (workspace == nullptr || ((size_t)workspace & 15)))
        return gh_set_error(GH_E_INVALID_ARG, "gh_project_backward: camera gradients need the 16-byte aligned workspace");
    const float* acc16 = nullptr;
    if (geom_buffer != nullptr) acc16 = GhGeomWS::carve(const_cast<char*>(geom_buffer), (size_t)P).acc16;
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partial = workspace ? reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256) : nullptr;
    if (d_camera != nullptr) {
        // the ticket word is reset by the kernel's last CTA; zero it here for the very first use of a workspace
        const cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), stream);
        if (e != cudaSuccess) return gh_cuda_status("gh_project_backward", "memset(ticket)", e);
    }
    auto kernel = strand ? gh_project_backward_kernel<true> : gh_project_backward_kernel<false>;
    kernel<<<(P + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
        A, visible, acc16, dL_dmeans2D, dL_dconic, dL_dcolors, dL_dopacity,
        d_xyz, d_scaling, d_rotation, d_dirs, d_features_dc, d_features_rest, d_opacity, d_label, d_orient_conf,
        d_means2D, partial, ticket, d_camera, nan_flag);
    return gh_launch_status("gh_project_backward", 1);
}

// ------------------------------------------------------------------------------------------------ capturable
// gh_project_forward_binned and gh_project_backward with tan(fov / 2) read from device memory and R kept on the device:
// every argument of a captured launch stays valid from one camera and one iteration to the next.
extern "C" int gh_project_forward_binned_capturable(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream_)
{
    const char* who = "gh_project_forward_binned_capturable";
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc == GH_OK) rc = gh_check_capacity(who, capacity);
    if (rc != GH_OK) return rc;
    if (!tan_fov) return gh_set_error(GH_E_INVALID_ARG, "%s: tan_fov (device float[2]) is required", who);
    if (!status) return gh_set_error(GH_E_INVALID_ARG, "%s: status (device uint32) is required", who);
    if (gh_proj_strand(flags)) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode is not supported", who);
    // (the kernel reads tan(fov / 2) from tan_fov; 1 stands in for it in the host-side checks)
    GhProjArgs A = gh_proj_args(P, width, height, xyz, scaling, rotation, dirs, features_dc, features_rest, opacity, label,
                                orient_conf, viewmatrix, projmatrix, campos, 1.f, 1.f, scale_modifier, sh_degree, flags, det_eps);
    rc = gh_proj_check(A, who, false);
    if (rc != GH_OK) return rc;
    if (!means2D || !colors || !opacities || !conic || !visible || !radii || !geom_buffer || !img_buffer || !binning_buffer)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing output pointer", who);
    if ((size_t)colors & 7) return gh_set_error(GH_E_INVALID_ARG, "%s: colors must be 8-byte aligned", who);
    return gh_forward_phase1_capturable(who, P, width, height, radii, geom_buffer, img_buffer, binning_buffer, capacity,
                                        status, num_rendered, stream, [&](const GhGeomWS& geom, const GhImgWS& img, int gx, int gy) {
        gh_project_forward_tan_kernel<<<(P + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
            A, tan_fov, means2D, colors, opacities, conic, visible, radii, geom.geo, geom.depth, img.tile_count, gx, gy);
        gh_count_launches(1);
    });
}

extern "C" int gh_project_backward_capturable(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    const unsigned char* visible,
    const char* geom_buffer,
    const float* dL_dmeans2D, const float* dL_dconic, const float* dL_dcolors, const float* dL_dopacity,
    float* d_xyz, float* d_scaling, float* d_rotation, float* d_dirs, float* d_features_dc, float* d_features_rest,
    float* d_opacity, float* d_label, float* d_orient_conf, float* d_means2D, float* d_camera,
    unsigned int* nan_flag, void* workspace, int debug, gh_stream_t stream_)
{
    const char* who = "gh_project_backward_capturable";
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc != GH_OK) return rc;
    if (!tan_fov) return gh_set_error(GH_E_INVALID_ARG, "%s: tan_fov (device float[2]) is required", who);
    GhProjArgs A = gh_proj_args(P, width, height, xyz, scaling, rotation, dirs, features_dc, features_rest, opacity, label,
                                orient_conf, viewmatrix, projmatrix, campos, 1.f, 1.f, scale_modifier, sh_degree, flags, det_eps);
    const bool strand = gh_proj_strand(flags);
    rc = gh_proj_check(A, who, strand);
    if (rc != GH_OK) return rc;
    if (strand && (d_scaling || d_rotation))
        return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode folds scale and rotation gradients into d_dirs, d_scaling / d_rotation must be NULL", who);
    if (strand && !d_dirs) return gh_set_error(GH_E_INVALID_ARG, "%s: strand mode needs d_dirs", who);
    if (!visible || !d_xyz || (!strand && (!d_scaling || !d_rotation)) || !d_features_dc || !d_features_rest)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
    if (geom_buffer == nullptr && (!dL_dmeans2D || !dL_dconic || !dL_dcolors || !dL_dopacity))
        return gh_set_error(GH_E_INVALID_ARG, "%s: pass the geometry workspace of the blend backward or the four incoming gradients", who);
    if (((size_t)d_rotation & 15) || (dL_dconic && ((size_t)dL_dconic & 15)) || (dL_dcolors && ((size_t)dL_dcolors & 7)))
        return gh_set_error(GH_E_INVALID_ARG, "%s: d_rotation / dL_dconic must be 16-byte, dL_dcolors 8-byte aligned", who);
    if (d_camera != nullptr && (workspace == nullptr || ((size_t)workspace & 15)))
        return gh_set_error(GH_E_INVALID_ARG, "%s: camera gradients need the 16-byte aligned workspace", who);
    const float* acc16 = nullptr;
    if (geom_buffer != nullptr) acc16 = GhGeomWS::carve(const_cast<char*>(geom_buffer), (size_t)P).acc16;
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partial = workspace ? reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256) : nullptr;
    if (d_camera != nullptr) {
        rc = gh_cuda_status(who, "memset(ticket)", cudaMemsetAsync(ticket, 0, sizeof(unsigned int), stream));
        if (rc != GH_OK) return rc;
    }
    auto kernel = strand ? gh_project_backward_tan_kernel<true> : gh_project_backward_tan_kernel<false>;
    kernel<<<(P + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
        A, tan_fov, visible, acc16, dL_dmeans2D, dL_dconic, dL_dcolors, dL_dopacity,
        d_xyz, d_scaling, d_rotation, d_dirs, d_features_dc, d_features_rest, d_opacity, d_label, d_orient_conf,
        d_means2D, partial, ticket, d_camera, nan_flag);
    return gh_launch_status(who, 1);
}

// ------------------------------------------------------------------------------------------------ capturable, strands
// A segment model behind its frozen head block in one capturable first phase over P = n_head + n_seg rows -- head rows
// first, then the segments, the row order of the eager path -- and the records-mode parameter backward of the segment
// rows.  The head block is frozen and the cameras are not trained: no head-row or camera gradients.  Two models share
// these bodies:
//  - strands (render_hair_strands): S polylines of L segments from `origins` and `dirs`; the forward computes the
//    midpoints into `midpoints` first, the backward completes d_dirs with the suffix scan of the cumulative sum;
//  - segments (render_hair_segments): the n_seg midpoints `xyz` and segment vectors `dirs` as given; no midpoints
//    kernel and no suffix scan, the two gradients leave as the projection backward writes them.
// The entry points check the row counts, the capacity and the capturable contract first.
namespace {

int gh_hair_rows_forward_capturable(
    const char* who, int n_head, int n_seg, int S, int L, int width, int height,
    const float* head_xyz, const float* head_scaling, const float* head_rotation,
    const float* head_features_dc, const float* head_features_rest, const float* head_opacity,
    unsigned int head_flags, float head_det_eps,
    const float* origins, float* midpoints, const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, cudaStream_t stream, bool strands)
{
    int rc;
    if (!tan_fov) return gh_set_error(GH_E_INVALID_ARG, "%s: tan_fov (device float[2]) is required", who);
    if (!status) return gh_set_error(GH_E_INVALID_ARG, "%s: status (device uint32) is required", who);
    if (gh_proj_strand(head_flags)) return gh_set_error(GH_E_INVALID_ARG, "%s: head_flags must not set the strand bit", who);
    if (!gh_proj_strand(flags)) return gh_set_error(GH_E_INVALID_ARG, "%s: flags must set the strand bit (10)", who);
    const int P = n_head + n_seg;
    // (the kernels read tan(fov / 2) from tan_fov; 1 stands in for it in the host-side checks)
    GhProjArgs Ah = gh_proj_args(n_head, width, height, head_xyz, head_scaling, head_rotation, nullptr, head_features_dc,
                                 head_features_rest, head_opacity, nullptr, nullptr, viewmatrix, projmatrix, campos,
                                 1.f, 1.f, scale_modifier, sh_degree, head_flags, head_det_eps);
    GhProjArgs As = gh_proj_args(n_seg, width, height, xyz, scale, nullptr, dirs, features_dc, features_rest, nullptr,
                                 nullptr, orient_conf, viewmatrix, projmatrix, campos, 1.f, 1.f, scale_modifier, sh_degree,
                                 flags, det_eps);
    if (n_head > 0 && (rc = gh_proj_check(Ah, who, false)) != GH_OK) return rc;
    if (n_seg > 0) {
        if (strands && (!origins || !midpoints)) return gh_set_error(GH_E_INVALID_ARG, "%s: origins and midpoints are required", who);
        if ((rc = gh_proj_check(As, who, true)) != GH_OK) return rc;
    }
    if (!means2D || !colors || !opacities || !conic || !visible || !radii || !geom_buffer || !img_buffer || !binning_buffer)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing output pointer", who);
    if ((size_t)colors & 7) return gh_set_error(GH_E_INVALID_ARG, "%s: colors must be 8-byte aligned", who);
    return gh_forward_phase1_capturable(who, P, width, height, radii, geom_buffer, img_buffer, binning_buffer, capacity,
                                        status, num_rendered, stream, [&](const GhGeomWS& geom, const GhImgWS& img, int gx, int gy) {
        if (n_head > 0) {
            gh_project_forward_tan_kernel<<<(n_head + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
                Ah, tan_fov, means2D, colors, opacities, conic, visible, radii, geom.geo, geom.depth, img.tile_count, gx, gy);
            gh_count_launches(1);
        }
        if (n_seg > 0) {
            // strands: the midpoints in segment order (bit-identical to the eager path's) into As.xyz = midpoints first;
            // then the segment rows behind the head's
            if (strands) {
                gh_launch_strand_midpoints(S, L, origins, dirs, midpoints, stream);
                gh_count_launches(1);
            }
            const size_t h = (size_t)n_head;
            gh_project_forward_strand_tan_kernel<<<(n_seg + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
                As, tan_fov, means2D + 3 * h, colors + GH_NUM_CHANNELS * h, opacities + h, conic + 3 * h, visible + h,
                radii + h, geom.geo + h, geom.depth + h, img.tile_count, gx, gy);
            gh_count_launches(1);
        }
    });
}

int gh_hair_rows_backward_capturable(
    const char* who, int n_head, int n_seg, int S, int L, int width, int height,
    const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    const unsigned char* visible, const char* geom_buffer,
    float* d_xyz, float* d_dirs, float* d_features_dc, float* d_features_rest, float* d_orient_conf,
    unsigned int* nan_flag, cudaStream_t stream, bool strands)
{
    if (!tan_fov) return gh_set_error(GH_E_INVALID_ARG, "%s: tan_fov (device float[2]) is required", who);
    if (!gh_proj_strand(flags)) return gh_set_error(GH_E_INVALID_ARG, "%s: flags must set the strand bit (10)", who);
    GhProjArgs A = gh_proj_args(n_seg, width, height, xyz, scale, nullptr, dirs, features_dc, features_rest, nullptr,
                                nullptr, orient_conf, viewmatrix, projmatrix, campos, 1.f, 1.f, scale_modifier, sh_degree,
                                flags, det_eps);
    const int rc = gh_proj_check(A, who, true);
    if (rc != GH_OK) return rc;
    if (!visible || !geom_buffer || !d_xyz || !d_dirs || !d_features_dc || !d_features_rest)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing mandatory pointer", who);
    // the blend backward's accumulation records of the segment rows, in the geometry workspace of all P rows
    const size_t h = (size_t)n_head;
    const float* acc16 = GhGeomWS::carve(const_cast<char*>(geom_buffer), h + (size_t)n_seg).acc16 + 16 * h;
    gh_project_backward_tan_kernel<true><<<(n_seg + GH_PJ_THREADS - 1) / GH_PJ_THREADS, GH_PJ_THREADS, 0, stream>>>(
        A, tan_fov, visible + h, acc16, nullptr, nullptr, nullptr, nullptr,
        d_xyz, nullptr, nullptr, d_dirs, d_features_dc, d_features_rest, nullptr, nullptr, d_orient_conf,
        nullptr, nullptr, nullptr, nullptr, nan_flag);
    if (!strands) return gh_launch_status(who, 1);
    // strands: dL/d midpoint through the cumulative sum into d_dirs
    gh_launch_strand_backward(S, L, d_xyz, d_dirs, nan_flag, stream);
    return gh_launch_status(who, 2);
}

}  // namespace

extern "C" int gh_hair_strands_forward_binned_capturable(
    int n_head, int S, int L, int width, int height,
    const float* head_xyz, const float* head_scaling, const float* head_rotation,
    const float* head_features_dc, const float* head_features_rest, const float* head_opacity,
    unsigned int head_flags, float head_det_eps,
    const float* origins, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    float* midpoints,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream_)
{
    const char* who = "gh_hair_strands_forward_binned_capturable";
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc == GH_OK) rc = gh_check_capacity(who, capacity);
    if (rc == GH_OK) rc = gh_strand_rows_check(who, n_head, S, L, false);
    if (rc != GH_OK) return rc;
    return gh_hair_rows_forward_capturable(
        who, n_head, S * L, S, L, width, height, head_xyz, head_scaling, head_rotation, head_features_dc,
        head_features_rest, head_opacity, head_flags, head_det_eps, origins, midpoints, midpoints, dirs, scale, features_dc,
        features_rest, orient_conf, flags, det_eps, viewmatrix, projmatrix, campos, tan_fov, scale_modifier, sh_degree,
        means2D, colors, opacities, conic, visible, radii, geom_buffer, img_buffer, binning_buffer, capacity, status,
        num_rendered, (cudaStream_t)stream_, true);
}

extern "C" int gh_hair_strands_backward_capturable(
    int n_head, int S, int L, int width, int height,
    const float* midpoints, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    const unsigned char* visible, const char* geom_buffer,
    float* d_xyz, float* d_dirs, float* d_features_dc, float* d_features_rest, float* d_orient_conf,
    unsigned int* nan_flag, int debug, gh_stream_t stream_)
{
    const char* who = "gh_hair_strands_backward_capturable";
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc == GH_OK) rc = gh_strand_rows_check(who, n_head, S, L, true);
    if (rc != GH_OK) return rc;
    return gh_hair_rows_backward_capturable(
        who, n_head, S * L, S, L, width, height, midpoints, dirs, scale, features_dc, features_rest, orient_conf, flags,
        det_eps, viewmatrix, projmatrix, campos, tan_fov, scale_modifier, sh_degree, visible, geom_buffer, d_xyz, d_dirs,
        d_features_dc, d_features_rest, d_orient_conf, nan_flag, (cudaStream_t)stream_, true);
}

// ------------------------------------------------------------------------------------------------ capturable, segments
// The latent strand model (render_hair_segments): its N segment rows come as given midpoints `xyz` and segment vectors
// `dirs` (what GaussianModelHair.generate_strands leaves in _xyz and _dir), not as polylines.
extern "C" int gh_hair_segments_forward_binned_capturable(
    int n_head, int N, int width, int height,
    const float* head_xyz, const float* head_scaling, const float* head_rotation,
    const float* head_features_dc, const float* head_features_rest, const float* head_opacity,
    unsigned int head_flags, float head_det_eps,
    const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream_)
{
    const char* who = "gh_hair_segments_forward_binned_capturable";
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc == GH_OK) rc = gh_check_capacity(who, capacity);
    if (rc == GH_OK) rc = gh_segment_rows_check(who, n_head, N, false);
    if (rc != GH_OK) return rc;
    if (!xyz || !dirs) return gh_set_error(GH_E_INVALID_ARG, "%s: xyz and dirs (the segment rows) are required", who);
    return gh_hair_rows_forward_capturable(
        who, n_head, N, 0, 0, width, height, head_xyz, head_scaling, head_rotation, head_features_dc, head_features_rest,
        head_opacity, head_flags, head_det_eps, nullptr, nullptr, xyz, dirs, scale, features_dc, features_rest, orient_conf,
        flags, det_eps, viewmatrix, projmatrix, campos, tan_fov, scale_modifier, sh_degree, means2D, colors, opacities,
        conic, visible, radii, geom_buffer, img_buffer, binning_buffer, capacity, status, num_rendered,
        (cudaStream_t)stream_, false);
}

extern "C" int gh_hair_segments_backward_capturable(
    int n_head, int N, int width, int height,
    const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    const unsigned char* visible, const char* geom_buffer,
    float* d_xyz, float* d_dirs, float* d_features_dc, float* d_features_rest, float* d_orient_conf,
    unsigned int* nan_flag, int debug, gh_stream_t stream_)
{
    const char* who = "gh_hair_segments_backward_capturable";
    gh_clear_error();
    int rc = gh_check_capturable(who, debug);
    if (rc == GH_OK) rc = gh_segment_rows_check(who, n_head, N, true);
    if (rc != GH_OK) return rc;
    if (!xyz || !dirs) return gh_set_error(GH_E_INVALID_ARG, "%s: xyz and dirs (the segment rows) are required", who);
    return gh_hair_rows_backward_capturable(
        who, n_head, N, 0, 0, width, height, xyz, dirs, scale, features_dc, features_rest, orient_conf, flags, det_eps,
        viewmatrix, projmatrix, campos, tan_fov, scale_modifier, sh_degree, visible, geom_buffer, d_xyz, d_dirs,
        d_features_dc, d_features_rest, d_orient_conf, nan_flag, (cudaStream_t)stream_, false);
}
