// Z-buffered triangle-mesh rasterization per view, and the per-vertex visibility counts of the scalp extraction
// (contract: include/gh_rasterizer.h; DESIGN §24).  Views run in chunks of `chunk`; per chunk, in stream order:
//     memset                      the packed z-buffer to all ones (no face, -1), the per-view vertex flags to 0
//     gh_mesh_raster_setup_kernel one thread per (view, face): projects the face into a GhRasterFace record
//                                 (gh_mesh_math.h), clears the (view, face) visibility flags and, once per view, the
//                                 per-view statistics
//     gh_mesh_raster_kernel       one warp per 32 consecutive records: the warp scans its faces' box sizes and walks
//                                 the flattened (face, pixel) pairs 32 at a time, each lane finding its face by a
//                                 binary search over the scan; a covered pixel takes atomicMin of (z bits << 32 | face)
//     gh_mesh_resolve_kernel      one thread per pixel: pix_to_face, the head-masked visibility image, the (view, face)
//                                 flags, and per view whether -1 occurs and the smallest face present
//     gh_mesh_face_verts_kernel   one thread per (view, face): flags the face's vertices, less the face `[1:]` drops
//     gh_mesh_count_kernel        one thread per vertex: adds the chunk's views, in view order, to the counts
// A pixel's answer is the smallest key, so it depends only on the mesh and its camera: bit-reproducible, independent
// of B, the chunk and the launch shape.
#include <climits>

#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_mesh_math.h"
#include "../../include/gh_rasterizer.h"

namespace {

static_assert(sizeof(GhRasterFace) == 80, "record layout");

#define GH_MR_THREADS 256
#define GH_MR_MAX_SIDE 8192                // H, W: pixel centres exact in float32, 32 boxes' pixels fit in 32 bits

struct GhMrLayout {
    size_t zbuf, rec, fvis, vvis, stats, total;
};

size_t gh_mr_align(size_t x) { return (x + 255) & ~(size_t)255; }

GhMrLayout gh_mr_layout(long long V, long long F, int H, int W, int chunk)
{
    GhMrLayout l;
    l.zbuf = 0;
    l.rec = gh_mr_align(l.zbuf + (size_t)chunk * H * W * sizeof(unsigned long long));
    l.fvis = gh_mr_align(l.rec + (size_t)chunk * F * sizeof(GhRasterFace));
    l.vvis = gh_mr_align(l.fvis + (size_t)2 * chunk * F);
    l.stats = gh_mr_align(l.vvis + (size_t)2 * chunk * V);
    l.total = gh_mr_align(l.stats + (size_t)4 * chunk * sizeof(unsigned int));
    return l;
}

// stats per view: [0] a -1 occurs in pix_to_face, [1] one occurs in the head variant, [2], [3] the smallest face
// present in each (0xffffffff: none)
__global__ void __launch_bounds__(GH_MR_THREADS)
gh_mesh_raster_setup_kernel(int Bc, int V, int F, const float* __restrict__ verts, const int* __restrict__ faces,
                            const float* __restrict__ K, const float* __restrict__ R, const float* __restrict__ t,
                            int H, int W, GhRasterFace* __restrict__ rec, unsigned char* __restrict__ fvis,
                            unsigned int* __restrict__ stats, unsigned int* __restrict__ status)
{
    const int r = blockIdx.x * GH_MR_THREADS + threadIdx.x;
    if (r >= Bc * F) return;
    const int b = r / F, f = r - b * F;
    if (fvis) {
        fvis[r] = 0;
        fvis[(size_t)Bc * F + r] = 0;
        if (f == 0) {
            stats[4 * b] = stats[4 * b + 1] = 0u;
            stats[4 * b + 2] = stats[4 * b + 3] = 0xffffffffu;
        }
    }
    const int i0 = __ldg(faces + 3 * (size_t)f), i1 = __ldg(faces + 3 * (size_t)f + 1), i2 = __ldg(faces + 3 * (size_t)f + 2);
    GhRasterFace out;
    out.j0 = out.i0 = out.nj = out.ni = 0;
    if (!gh_mesh_face_in_range(i0, i1, i2, V)) {
        atomicOr(status, GH_STATUS_SDF_FACE_INDEX);
    } else {
        float a[3], bb[3], c[3], cam[4], Rv[9], tv[3];
        for (int k = 0; k < 3; k++) {
            a[k] = __ldg(verts + 3 * (size_t)i0 + k);
            bb[k] = __ldg(verts + 3 * (size_t)i1 + k);
            c[k] = __ldg(verts + 3 * (size_t)i2 + k);
            tv[k] = __ldg(t + 3 * b + k);
        }
        for (int k = 0; k < 9; k++) Rv[k] = __ldg(R + 9 * b + k);
        cam[0] = __ldg(K + 9 * b);
        cam[1] = __ldg(K + 9 * b + 4);
        cam[2] = __ldg(K + 9 * b + 2);
        cam[3] = __ldg(K + 9 * b + 5);
        if (gh_raster_setup(cam, Rv, tv, a, bb, c, H, W, out) == GH_RASTER_NEAR) atomicOr(status, GH_STATUS_RASTER_NEAR);
    }
    rec[r] = out;
}

__global__ void __launch_bounds__(GH_MR_THREADS)
gh_mesh_raster_kernel(int n_rec, int F, int H, int W, const GhRasterFace* __restrict__ rec,
                      unsigned long long* __restrict__ zbuf)
{
    const int lane = threadIdx.x & 31;
    const int r0 = (blockIdx.x * GH_MR_THREADS + threadIdx.x) & ~31;
    if (r0 >= n_rec) return;                                   // the whole warp
    unsigned n = 0;
    if (r0 + lane < n_rec) n = (unsigned)__ldg(&rec[r0 + lane].nj) * (unsigned)__ldg(&rec[r0 + lane].ni);
    unsigned incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    const unsigned excl = incl - n;
    const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
    for (unsigned base = 0; base < total; base += 32) {
        const unsigned idx = base + lane;
        int owner = 0;                                         // the first lane whose inclusive sum exceeds idx
#pragma unroll
        for (int step = 16; step; step >>= 1)
            if (__shfl_sync(0xffffffffu, incl, owner + step - 1) <= idx) owner += step;
        const unsigned local = idx - __shfl_sync(0xffffffffu, excl, owner);
        if (idx >= total) continue;
        const GhRasterFace* fr = rec + r0 + owner;
        const int nj = __ldg(&fr->nj);
        const int di = (int)(local / (unsigned)nj), dj = (int)local - di * nj;
        const int i = __ldg(&fr->i0) + di, j = __ldg(&fr->j0) + dj;
        GhRasterFace f;
        for (int k = 0; k < 3; k++) {
            f.x[k] = __ldg(&fr->x[k]);
            f.y[k] = __ldg(&fr->y[k]);
            f.ex[k] = __ldg(&fr->ex[k]);
            f.ey[k] = __ldg(&fr->ey[k]);
            f.iz[k] = __ldg(&fr->iz[k]);
        }
        f.area = __ldg(&fr->area);
        float z;
        if (gh_raster_pixel(f, i, j, z)) {
            const int rr = r0 + owner, b = rr / F, face = rr - b * F;
            atomicMin(zbuf + ((size_t)b * H + i) * W + j,
                      ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)face);
        }
    }
}

// grid (ceil(HW / 256), Bc): one view per grid row, so the per-view reductions stay inside a warp's view
__global__ void __launch_bounds__(GH_MR_THREADS)
gh_mesh_resolve_kernel(int F, int HW, const unsigned long long* __restrict__ zbuf,
                       const unsigned char* __restrict__ head, int* __restrict__ pix_to_face,
                       unsigned char* __restrict__ vis, unsigned char* __restrict__ fvis, int Bc,
                       unsigned int* __restrict__ stats)
{
    const int b = blockIdx.y, p = blockIdx.x * GH_MR_THREADS + threadIdx.x;
    const bool valid = p < HW;
    const size_t px = (size_t)b * HW + p;
    int face = -1, face_h = -1;
    if (valid) {
        face = (int)(unsigned)zbuf[px];
        face_h = head && head[px] ? face : -1;
        if (pix_to_face) pix_to_face[px] = face;
        if (vis) vis[px] = face_h >= 0;
    }
    if (!fvis) return;
    if (face >= 0) fvis[(size_t)b * F + face] = 1;
    if (face_h >= 0) fvis[(size_t)Bc * F + (size_t)b * F + face_h] = 1;
    const unsigned neg = __ballot_sync(0xffffffffu, valid && face < 0);
    const unsigned neg_h = __ballot_sync(0xffffffffu, valid && face_h < 0);
    const unsigned mn = __reduce_min_sync(0xffffffffu, face >= 0 ? (unsigned)face : 0xffffffffu);
    const unsigned mn_h = __reduce_min_sync(0xffffffffu, face_h >= 0 ? (unsigned)face_h : 0xffffffffu);
    if ((threadIdx.x & 31) == 0) {
        unsigned int* s = stats + 4 * b;
        if (neg) s[0] = 1u;
        if (neg_h) s[1] = 1u;
        if (mn != 0xffffffffu) atomicMin(s + 2, mn);
        if (mn_h != 0xffffffffu) atomicMin(s + 3, mn_h);
    }
}

// `pix_to_face.unique()[1:]` drops the smallest value: -1 where one occurs, else the smallest face present
__global__ void __launch_bounds__(GH_MR_THREADS)
gh_mesh_face_verts_kernel(int Bc, int V, int F, const int* __restrict__ faces, const unsigned char* __restrict__ fvis,
                          const unsigned int* __restrict__ stats, unsigned char* __restrict__ vvis)
{
    const int r = blockIdx.x * GH_MR_THREADS + threadIdx.x;
    if (r >= Bc * F) return;
    const int b = r / F, f = r - b * F;
    const unsigned int* s = stats + 4 * b;
    const bool plain = fvis[r] && !(s[0] == 0u && s[2] == (unsigned)f);
    const bool head = fvis[(size_t)Bc * F + r] && !(s[1] == 0u && s[3] == (unsigned)f);
    if (!plain && !head) return;
    const int i[3] = {__ldg(faces + 3 * (size_t)f), __ldg(faces + 3 * (size_t)f + 1), __ldg(faces + 3 * (size_t)f + 2)};
    if (!gh_mesh_face_in_range(i[0], i[1], i[2], V)) return;  // never drawn, so never flagged
    for (int k = 0; k < 3; k++) {
        if (plain) vvis[(size_t)b * V + i[k]] = 1;
        if (head) vvis[(size_t)Bc * V + (size_t)b * V + i[k]] = 1;
    }
}

__global__ void __launch_bounds__(GH_MR_THREADS)
gh_mesh_count_kernel(int Bc, int V, const unsigned char* __restrict__ vvis, int* __restrict__ count,
                     int* __restrict__ count_head)
{
    const int v = blockIdx.x * GH_MR_THREADS + threadIdx.x;
    if (v >= V) return;
    int c = 0, ch = 0;
    for (int b = 0; b < Bc; b++) {
        c += vvis[(size_t)b * V + v];
        ch += vvis[(size_t)(Bc + b) * V + v];
    }
    count[v] += c;
    count_head[v] += ch;
}

int gh_mr_check_sizes(const char* who, long long V, long long F, int H, int W, int chunk)
{
    if (V < 1 || V > INT_MAX || F < 1 || F > INT_MAX)
        return gh_set_error(GH_E_INVALID_ARG, "%s: V and F must lie in [1, 2^31)", who);
    if (H < 1 || W < 1 || H > GH_MR_MAX_SIDE || W > GH_MR_MAX_SIDE)
        return gh_set_error(GH_E_INVALID_ARG, "%s: H and W must lie in [1, %d]", who, GH_MR_MAX_SIDE);
    if (chunk < 1 || (long long)chunk * H * W > INT_MAX || (long long)chunk * F > INT_MAX ||
        (long long)chunk * V > INT_MAX)
        return gh_set_error(GH_E_INVALID_ARG, "%s: chunk must be >= 1 with chunk*H*W, chunk*F and chunk*V below 2^31",
                            who);
    return GH_OK;
}

}  // namespace

extern "C" int gh_mesh_raster_workspace_size(long long V, long long F, int H, int W, int chunk, size_t* bytes)
{
    static const char* who = "gh_mesh_raster_workspace_size";
    gh_clear_error();
    const int rc = gh_mr_check_sizes(who, V, F, H, W, chunk);
    if (rc != GH_OK) return rc;
    if (!bytes) return gh_set_error(GH_E_INVALID_ARG, "%s: bytes is NULL", who);
    *bytes = gh_mr_layout(V, F, H, W, chunk).total;
    return GH_OK;
}

extern "C" int gh_mesh_raster(long long V, long long F, const float* verts, const int* faces, int B, const float* K,
                              const float* R, const float* t, int H, int W, const unsigned char* head_mask,
                              int* pix_to_face, unsigned char* vis_head, int* vis_count, int* vis_count_head, int chunk,
                              void* workspace, size_t bytes, unsigned int* status, int debug, gh_stream_t stream_)
{
    static const char* who = "gh_mesh_raster";
    gh_clear_error();
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = gh_mr_check_sizes(who, V, F, H, W, chunk);
    if (rc != GH_OK) return rc;
    if (B < 1) return gh_set_error(GH_E_INVALID_ARG, "%s: B must be >= 1", who);
    if (!verts || !faces || !K || !R || !t || !status)
        return gh_set_error(GH_E_INVALID_ARG, "%s: missing verts, faces, K, R, t or status", who);
    if (((size_t)verts | (size_t)faces | (size_t)K | (size_t)R | (size_t)t | (size_t)status | (size_t)pix_to_face |
         (size_t)vis_count | (size_t)vis_count_head) & 3)
        return gh_set_error(GH_E_INVALID_ARG, "%s: float and int arrays must be 4-byte aligned", who);
    if (!vis_count != !vis_count_head)
        return gh_set_error(GH_E_INVALID_ARG, "%s: vis_count and vis_count_head go together", who);
    if (!pix_to_face && !vis_head && !vis_count)
        return gh_set_error(GH_E_INVALID_ARG, "%s: no output (pix_to_face, vis_head or vis_count)", who);
    const GhMrLayout l = gh_mr_layout(V, F, H, W, chunk);
    if (!workspace) return gh_set_error(GH_E_INVALID_ARG, "%s: missing workspace", who);
    if ((size_t)workspace & 255) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace must be 256-byte aligned", who);
    if (bytes < l.total) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace of %zu bytes, %zu needed", who, bytes, l.total);
    if (debug && (rc = gh_check_capturable(who, 0)) != GH_OK) return rc;    // debug synchronises: not with the stage timer on

    const int nv = (int)V, nf = (int)F, HW = H * W;
    char* ws = static_cast<char*>(workspace);
    unsigned long long* zbuf = reinterpret_cast<unsigned long long*>(ws + l.zbuf);
    GhRasterFace* rec = reinterpret_cast<GhRasterFace*>(ws + l.rec);
    unsigned char* fvis = vis_count ? reinterpret_cast<unsigned char*>(ws + l.fvis) : nullptr;
    unsigned char* vvis = reinterpret_cast<unsigned char*>(ws + l.vvis);
    unsigned int* stats = reinterpret_cast<unsigned int*>(ws + l.stats);
    int launches = 0;
    if (vis_count) {
        if ((rc = gh_cuda_status(who, "memset", cudaMemsetAsync(vis_count, 0, sizeof(int) * (size_t)nv, stream))) ||
            (rc = gh_cuda_status(who, "memset", cudaMemsetAsync(vis_count_head, 0, sizeof(int) * (size_t)nv, stream))))
            return rc;
    }
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int Bc = min(chunk, B - b0);
        const size_t px0 = (size_t)b0 * HW;
        if ((rc = gh_cuda_status(who, "memset", cudaMemsetAsync(zbuf, 0xff, (size_t)Bc * HW * 8, stream)))) return rc;
        const int n_rec = Bc * nf;
        const int g_rec = (n_rec + GH_MR_THREADS - 1) / GH_MR_THREADS;
        gh_mesh_raster_setup_kernel<<<g_rec, GH_MR_THREADS, 0, stream>>>(
            Bc, nv, nf, verts, faces, K + 9 * (size_t)b0, R + 9 * (size_t)b0, t + 3 * (size_t)b0, H, W, rec, fvis,
            stats, status);
        gh_mesh_raster_kernel<<<g_rec, GH_MR_THREADS, 0, stream>>>(n_rec, nf, H, W, rec, zbuf);
        gh_mesh_resolve_kernel<<<dim3((HW + GH_MR_THREADS - 1) / GH_MR_THREADS, Bc), GH_MR_THREADS, 0, stream>>>(
            nf, HW, zbuf, head_mask ? head_mask + px0 : nullptr, pix_to_face ? pix_to_face + px0 : nullptr,
            vis_head ? vis_head + px0 : nullptr, fvis, Bc, stats);
        launches += 3;
        if (vis_count) {
            if ((rc = gh_cuda_status(who, "memset", cudaMemsetAsync(vvis, 0, (size_t)2 * Bc * nv, stream)))) return rc;
            gh_mesh_face_verts_kernel<<<g_rec, GH_MR_THREADS, 0, stream>>>(Bc, nv, nf, faces, fvis, stats, vvis);
            gh_mesh_count_kernel<<<(nv + GH_MR_THREADS - 1) / GH_MR_THREADS, GH_MR_THREADS, 0, stream>>>(
                Bc, nv, vvis, vis_count, vis_count_head);
            launches += 2;
        }
    }
    rc = gh_launch_status(who, launches);
    if (rc == GH_OK && debug) rc = gh_cuda_status(who, "synchronise (debug)", cudaStreamSynchronize(stream));
    return rc;
}
