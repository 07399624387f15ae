// Signed distance of points to a triangle mesh, brute force (contract: include/gh_rasterizer.h; DESIGN §23):
//     gh_sdf_prepare_kernel  one thread per face: checks its three indices against V and writes the face's record
//                            (gh_mesh_math.h), or a NaN record for an index out of range
//     gh_sdf_query_kernel    one thread per point: the records stream through shared memory in tiles of GH_SDF_TILE
//                            faces, and every thread visits every face in index order, keeping min d^2 in float32 and
//                            the sum of the solid angles in double
// A point's result depends only on the point and the record array, so it is the same in any batch and any launch.
#include <climits>

#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_mesh_math.h"
#include "../../include/gh_rasterizer.h"

namespace {

#define GH_SDF_THREADS 128                 // queries per CTA
#define GH_SDF_TILE 128                    // faces per shared-memory tile: 14 KB
#define GH_SDF_VEC (sizeof(GhSdfRecord) / sizeof(float4))

static_assert(sizeof(GhSdfRecord) == 112, "record layout");

__global__ void __launch_bounds__(256)
gh_sdf_prepare_kernel(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces,
                      GhSdfRecord* __restrict__ rec, unsigned int* __restrict__ status)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= F) return;
    const int i0 = __ldg(faces + 3 * (size_t)f), i1 = __ldg(faces + 3 * (size_t)f + 1), i2 = __ldg(faces + 3 * (size_t)f + 2);
    GhSdfRecord r;
    if (!gh_mesh_face_in_range(i0, i1, i2, V)) {
        atomicOr(status, GH_STATUS_SDF_FACE_INDEX);
        for (int k = 0; k < 28; k++) r.v[k] = __int_as_float(0x7fffffff);
    } else {
        float a[3], b[3], c[3];
        for (int k = 0; k < 3; k++) {
            a[k] = __ldg(verts + 3 * (size_t)i0 + k);
            b[k] = __ldg(verts + 3 * (size_t)i1 + k);
            c[k] = __ldg(verts + 3 * (size_t)i2 + k);
        }
        gh_sdf_record(a, b, c, r);
    }
    rec[f] = r;
}

__global__ void __launch_bounds__(GH_SDF_THREADS)
gh_sdf_query_kernel(int N, const float* __restrict__ points, int F, const float4* __restrict__ rec,
                    float* __restrict__ sdf, float* __restrict__ dist, float* __restrict__ winding)
{
    __shared__ GhSdfRecord s_rec[GH_SDF_TILE];
    const int i = blockIdx.x * GH_SDF_THREADS + threadIdx.x;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (i < N) {
        px = __ldg(points + 3 * (size_t)i);
        py = __ldg(points + 3 * (size_t)i + 1);
        pz = __ldg(points + 3 * (size_t)i + 2);
    }
    float m = INFINITY;
    double w = 0.0;
    for (int f0 = 0; f0 < F; f0 += GH_SDF_TILE) {
        const int nt = min(GH_SDF_TILE, F - f0);
        __syncthreads();
        float4* s4 = reinterpret_cast<float4*>(s_rec);
        for (int k = threadIdx.x; k < nt * (int)GH_SDF_VEC; k += GH_SDF_THREADS)
            s4[k] = __ldg(rec + (size_t)f0 * GH_SDF_VEC + k);
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < nt; j++) {
            float d2, om;
            gh_sdf_pair(s_rec[j], px, py, pz, d2, om);
            m = fminf(m, d2);
            w += (double)om;
        }
    }
    if (i >= N) return;
    const double wn = w / (4.0 * 3.14159265358979323846);
    const float d = sqrtf(m);
    float o_sdf = wn > 0.5 ? d : -d, o_d = d, o_w = (float)wn;
    if (!(isfinite(px) && isfinite(py) && isfinite(pz))) o_sdf = o_d = o_w = __int_as_float(0x7fffffff);
    sdf[i] = o_sdf;
    if (dist) dist[i] = o_d;
    if (winding) winding[i] = o_w;
}

size_t gh_sdf_ws_bytes(long long F) { return (size_t)F * sizeof(GhSdfRecord); }

int gh_sdf_check_count(const char* who, const char* what, long long n, long long lo)
{
    if (n < lo || n > INT_MAX) return gh_set_error(GH_E_INVALID_ARG, "%s: %s must lie in [%lld, 2^31)", who, what, lo);
    return GH_OK;
}

int gh_sdf_check_ws(const char* who, long long F, const void* workspace, size_t bytes, int debug)
{
    if (!workspace) return gh_set_error(GH_E_INVALID_ARG, "%s: missing workspace", who);
    if ((size_t)workspace & 15) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace must be 16-byte aligned", who);
    if (bytes < gh_sdf_ws_bytes(F))
        return gh_set_error(GH_E_INVALID_ARG, "%s: workspace of %zu bytes, %zu needed", who, bytes, gh_sdf_ws_bytes(F));
    if (debug) return gh_check_capturable(who, 0);     // debug synchronises: not with the stage timer on
    return GH_OK;
}

int gh_sdf_finish(const char* who, int debug, cudaStream_t stream)
{
    int rc = gh_launch_status(who, 1);
    if (rc == GH_OK && debug) rc = gh_cuda_status(who, "synchronise (debug)", cudaStreamSynchronize(stream));
    return rc;
}

}  // namespace

extern "C" int gh_sdf_workspace_size(long long F, size_t* bytes)
{
    static const char* who = "gh_sdf_workspace_size";
    gh_clear_error();
    const int rc = gh_sdf_check_count(who, "F", F, 1);
    if (rc != GH_OK) return rc;
    if (!bytes) return gh_set_error(GH_E_INVALID_ARG, "%s: bytes is NULL", who);
    *bytes = gh_sdf_ws_bytes(F);
    return GH_OK;
}

extern "C" int gh_sdf_prepare(long long V, long long F, const float* verts, const int* faces, void* workspace,
                              size_t bytes, unsigned int* status, int debug, gh_stream_t stream_)
{
    static const char* who = "gh_sdf_prepare";
    gh_clear_error();
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = gh_sdf_check_count(who, "V", V, 1);
    if (rc == GH_OK) rc = gh_sdf_check_count(who, "F", F, 1);
    if (rc != GH_OK) return rc;
    if (!verts || !faces || !status) return gh_set_error(GH_E_INVALID_ARG, "%s: missing verts, faces or status", who);
    if (((size_t)verts | (size_t)faces | (size_t)status) & 3)
        return gh_set_error(GH_E_INVALID_ARG, "%s: verts, faces and status must be 4-byte aligned", who);
    if ((rc = gh_sdf_check_ws(who, F, workspace, bytes, debug)) != GH_OK) return rc;
    const int nf = (int)F;
    gh_sdf_prepare_kernel<<<(nf + 255) / 256, 256, 0, stream>>>((int)V, nf, verts, faces,
                                                                static_cast<GhSdfRecord*>(workspace), status);
    return gh_sdf_finish(who, debug, stream);
}

extern "C" int gh_sdf_query(long long N, const float* points, long long F, const void* workspace, size_t bytes,
                            float* sdf, float* dist, float* winding, int debug, gh_stream_t stream_)
{
    static const char* who = "gh_sdf_query";
    gh_clear_error();
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = gh_sdf_check_count(who, "N", N, 0);
    if (rc == GH_OK) rc = gh_sdf_check_count(who, "F", F, 1);
    if (rc != GH_OK) return rc;
    if (N > 0 && (!points || !sdf)) return gh_set_error(GH_E_INVALID_ARG, "%s: missing points or sdf", who);
    if (((size_t)points | (size_t)sdf | (size_t)dist | (size_t)winding) & 3)
        return gh_set_error(GH_E_INVALID_ARG, "%s: points, sdf, dist and winding must be 4-byte aligned", who);
    if ((rc = gh_sdf_check_ws(who, F, workspace, bytes, debug)) != GH_OK) return rc;
    if (N == 0) return GH_OK;
    const int n = (int)N;
    gh_sdf_query_kernel<<<(n + GH_SDF_THREADS - 1) / GH_SDF_THREADS, GH_SDF_THREADS, 0, stream>>>(
        n, points, (int)F, static_cast<const float4*>(workspace), sdf, dist, winding);
    return gh_sdf_finish(who, debug, stream);
}
