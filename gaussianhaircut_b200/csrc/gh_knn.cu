// Exact 3-nearest-neighbour mean squared distance of a point cloud: `simple_knn._C.distCUDA2`, which
// `GaussianModel.create_from_pcd` (src/scene/gaussian_model.py:409) calls once to size the initial Gaussians.
//
// d[i] = ((b0 + b1) + b2) / 3 over the three smallest float32 squared distances from point i to the other finite points
// (DESIGN §14 states the contract).  Stages, all on the caller's stream:
//   gh_knn_morton      bounding box of the finite points (per-CTA reduction + integer atomics on an order-preserving
//                      encoding: exact), then 63-bit Morton codes quantised on that box; non-finite points get
//                      INT64_MAX, above every finite code, so they sort to the end.
//   (caller)           order = torch.sort(codes, stable=True).indices
//   gh_knn_mean_dist3  gather the points in Morton order (non-finite ones as NaN) and build tight boxes of 32
//                      consecutive points, an implicit binary tree over them (heap order, root 1, children 2h and 2h+1,
//                      min/max only), then one thread per point in Morton order: seed b2 from the +-4 neighbours in
//                      sorted order, walk the tree nearest child first, prune a node whose lower bound
//                      (gh_knn_box_bound) is >= b2, stop at b2 == 0, write d[order[i]].
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_knn_math.h"
#include "../../include/gh_rasterizer.h"

#include <climits>

namespace {

constexpr int GH_KNN_LEAF = 32;       // points per leaf box: one warp builds one
constexpr int GH_KNN_SEED = 4;        // neighbours on each side in sorted order that seed b2
constexpr int GH_KNN_TREE_CTA = 256;  // nodes of one row reduced by a CTA of the tree kernel (8 rows up)
constexpr unsigned int GH_KNN_QMAX = (1u << 21) - 2;   // quantised coordinate limit: finite codes stay < INT64_MAX

// Workspace: the bounding box (6 encoded words), the points in sorted order, the tree's boxes (lo, hi as two float4
// per node, heap order; 2^D leaves with 2^D >= ceil(P / 32), so the tree has 2^(D+1) slots, slot 0 unused).
struct GhKnnWS {
    unsigned int* box;
    float4* pts;
    float4* nodes;
    int depth;

    static int depth_for(size_t P) {
        const size_t leaves = (P + GH_KNN_LEAF - 1) / GH_KNN_LEAF;
        int d = 0;
        while (((size_t)1 << d) < leaves) d++;
        return d;
    }
    static size_t bytes(size_t P) {
        return 256 + gh_align_up(P * sizeof(float4), 256) + gh_align_up(((size_t)2 << depth_for(P)) * 2 * sizeof(float4), 256) + 256;
    }
    static GhKnnWS carve(char* base, size_t P) {
        GhKnnWS w;
        size_t off = gh_align_up((size_t)base, 256) - (size_t)base;
        w.box = (unsigned int*)(base + off); off += 256;
        w.pts = (float4*)(base + off); off += gh_align_up(P * sizeof(float4), 256);
        w.nodes = (float4*)(base + off);
        w.depth = depth_for(P);
        return w;
    }
};

// float -> unsigned with the same order (negative values complemented, positive ones with the sign bit set)
__device__ __forceinline__ unsigned int gh_knn_ord(float f) {
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float gh_knn_unord(unsigned int e) {
    return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

__device__ __forceinline__ bool gh_knn_finite(float x, float y, float z) {
    return isfinite(x) && isfinite(y) && isfinite(z);
}

// 21 bits -> every third bit of 63
__device__ __forceinline__ unsigned long long gh_knn_spread(unsigned int v) {
    unsigned long long x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

// box[0..2] = max of ~ord(min candidates) (so that one zero memset initialises min and max alike), box[3..5] = max ord.
// For finite values neither encoding is 0, so 0 is the identity of both.
__global__ void __launch_bounds__(256)
gh_knn_bbox_kernel(int P, const float* __restrict__ pts, unsigned int* __restrict__ box)
{
    unsigned int m[6] = {0u, 0u, 0u, 0u, 0u, 0u};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        if (!gh_knn_finite(x, y, z)) continue;
        const unsigned int ex = gh_knn_ord(x), ey = gh_knn_ord(y), ez = gh_knn_ord(z);
        m[0] = max(m[0], ~ex); m[1] = max(m[1], ~ey); m[2] = max(m[2], ~ez);
        m[3] = max(m[3], ex);  m[4] = max(m[4], ey);  m[5] = max(m[5], ez);
    }
    __shared__ unsigned int part[8][6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 6; k++) m[k] = __reduce_max_sync(0xffffffffu, m[k]);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 6; k++) part[warp][k] = m[k];
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        unsigned int v = 0u;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) v = max(v, part[w][threadIdx.x]);
        if (v != 0u) atomicMax(&box[threadIdx.x], v);
    }
}

__global__ void __launch_bounds__(256)
gh_knn_morton_kernel(int P, const float* __restrict__ pts, const unsigned int* __restrict__ box, long long* __restrict__ codes)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    if (!gh_knn_finite(x, y, z)) { codes[i] = LLONG_MAX; return; }
    // at least this point is finite, so the box is
    const float lx = gh_knn_unord(~box[0]), ly = gh_knn_unord(~box[1]), lz = gh_knn_unord(~box[2]);
    const float ext = fmaxf(fmaxf(gh_knn_unord(box[3]) - lx, gh_knn_unord(box[4]) - ly), gh_knn_unord(box[5]) - lz);
    // one scale for all axes keeps cells cubic; an extent that overflows to +inf gives scale 0 (all codes 0: slower
    // queries, same results -- the order only decides how fast the tree prunes, never what it finds)
    const float scale = ext > 0.f ? (float)GH_KNN_QMAX / ext : 0.f;
    const float qm = (float)GH_KNN_QMAX;
    const unsigned int qx = (unsigned int)fminf(fmaxf((x - lx) * scale, 0.f), qm);
    const unsigned int qy = (unsigned int)fminf(fmaxf((y - ly) * scale, 0.f), qm);
    const unsigned int qz = (unsigned int)fminf(fmaxf((z - lz) * scale, 0.f), qm);
    codes[i] = (long long)((gh_knn_spread(qx) << 2) | (gh_knn_spread(qy) << 1) | gh_knn_spread(qz));
}

// One warp per leaf: gather its 32 points in sorted order (.w = original index; non-finite points as NaN, which no
// comparison admits as a neighbour) and reduce their tight box.  Leaves past P get the empty box (+inf, -inf).
__global__ void __launch_bounds__(256)
gh_knn_leaves_kernel(int P, unsigned int nleaf, const float* __restrict__ pts, const long long* __restrict__ order,
                     float4* __restrict__ sorted, float4* __restrict__ nodes)
{
    const unsigned int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (leaf >= nleaf) return;
    const long long i = (long long)leaf * GH_KNN_LEAF + lane;
    float lx = INFINITY, ly = INFINITY, lz = INFINITY, hx = -INFINITY, hy = -INFINITY, hz = -INFINITY;
    if (i < P) {
        const long long o = order[i];
        float4 v = make_float4(NAN, NAN, NAN, __int_as_float(-1));    // an index outside [0, P) is never written
        if (o >= 0 && o < P) {
            const float x = pts[3 * o], y = pts[3 * o + 1], z = pts[3 * o + 2];
            v.w = __int_as_float((int)o);
            if (gh_knn_finite(x, y, z)) {
                v.x = x; v.y = y; v.z = z;
                lx = hx = x; ly = hy = y; lz = hz = z;
            }
        }
        sorted[i] = v;
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        lx = fminf(lx, __shfl_xor_sync(0xffffffffu, lx, s));
        ly = fminf(ly, __shfl_xor_sync(0xffffffffu, ly, s));
        lz = fminf(lz, __shfl_xor_sync(0xffffffffu, lz, s));
        hx = fmaxf(hx, __shfl_xor_sync(0xffffffffu, hx, s));
        hy = fmaxf(hy, __shfl_xor_sync(0xffffffffu, hy, s));
        hz = fmaxf(hz, __shfl_xor_sync(0xffffffffu, hz, s));
    }
    if (lane == 0) {
        const size_t h = (size_t)nleaf + leaf;
        nodes[2 * h] = make_float4(lx, ly, lz, 0.f);
        nodes[2 * h + 1] = make_float4(hx, hy, hz, 0.f);
    }
}

// Rows `row - 1` .. `row - steps` of the tree from row `row` (2^row nodes, heap slots [2^row, 2^(row+1))): each CTA
// reduces 256 consecutive nodes, i.e. complete subtrees up to 8 rows high, in shared memory.
__global__ void __launch_bounds__(GH_KNN_TREE_CTA)
gh_knn_tree_kernel(float4* __restrict__ nodes, int row, int steps)
{
    __shared__ float4 slo[GH_KNN_TREE_CTA], shi[GH_KNN_TREE_CTA];
    const unsigned int n = 1u << row, t = threadIdx.x;
    const unsigned int k = blockIdx.x * GH_KNN_TREE_CTA + t;
    if (k < n) { slo[t] = nodes[2 * ((size_t)n + k)]; shi[t] = nodes[2 * ((size_t)n + k) + 1]; }
    __syncthreads();
    unsigned int width = min(n, (unsigned int)GH_KNN_TREE_CTA);
    for (int s = 1; s <= steps; s++) {
        width >>= 1;
        float4 lo, hi;
        if (t < width) {
            const float4 a = slo[2 * t], b = slo[2 * t + 1], c = shi[2 * t], d = shi[2 * t + 1];
            lo = make_float4(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z), 0.f);
            hi = make_float4(fmaxf(c.x, d.x), fmaxf(c.y, d.y), fmaxf(c.z, d.z), 0.f);
        }
        __syncthreads();
        if (t < width) {
            slo[t] = lo; shi[t] = hi;
            const size_t h = ((size_t)n >> s) + (size_t)blockIdx.x * (GH_KNN_TREE_CTA >> s) + t;
            nodes[2 * h] = lo; nodes[2 * h + 1] = hi;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ float gh_knn_node_bound(const float4* __restrict__ nodes, unsigned int h, float px, float py, float pz)
{
    const float4 lo = __ldg(nodes + 2 * (size_t)h), hi = __ldg(nodes + 2 * (size_t)h + 1);
    return gh_knn_box_bound(px, py, pz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
}

// One thread per point in sorted order.  The walk needs no stack: in heap order the parent of h is h >> 1 and its
// sibling h ^ 1, and bit k of `second` says whether the node at depth k is the second child visited.
__global__ void __launch_bounds__(128)
gh_knn_query_kernel(int P, int depth, const float4* __restrict__ pts, const float4* __restrict__ nodes, float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float4 p = __ldg(pts + i);
    const int o = __float_as_int(p.w);
    if (o < 0) return;
    if (p.x != p.x) { out[o] = NAN; return; }      // a non-finite point has no distance and is no neighbour
    float b0 = INFINITY, b1 = INFINITY, b2 = INFINITY;
    const int j0 = max(i - GH_KNN_SEED, 0), j1 = min(i + GH_KNN_SEED, P - 1);
    for (int j = j0; j <= j1; j++) {
        if (j == i) continue;
        const float4 q = __ldg(pts + j);
        gh_knn_insert(gh_knn_dist2(p.x, p.y, p.z, q.x, q.y, q.z), b0, b1, b2);
    }
    const unsigned int nleaf = 1u << depth;
    unsigned int h = 1u, second = 0u;
    int dep = 0;
    float lb = gh_knn_node_bound(nodes, 1u, p.x, p.y, p.z);
    for (;;) {
        if (lb < b2) {
            if (h >= nleaf) {
                const int a = (int)(h - nleaf) * GH_KNN_LEAF, e = min(a + GH_KNN_LEAF, P);
                for (int j = a; j < e; j++) {
                    if ((unsigned int)(j - i + GH_KNN_SEED) <= 2u * GH_KNN_SEED) continue;   // the seeds and i itself
                    const float4 q = __ldg(pts + j);
                    gh_knn_insert(gh_knn_dist2(p.x, p.y, p.z, q.x, q.y, q.z), b0, b1, b2);
                }
            } else {
                const float l0 = gh_knn_node_bound(nodes, 2u * h, p.x, p.y, p.z);
                const float l1 = gh_knn_node_bound(nodes, 2u * h + 1u, p.x, p.y, p.z);
                dep++;
                second &= ~(1u << dep);
                h = 2u * h + (l1 < l0 ? 1u : 0u);
                lb = fminf(l0, l1);
                continue;
            }
        }
        while (dep > 0 && ((second >> dep) & 1u)) { h >>= 1; dep--; }
        if (dep == 0 || b2 == 0.f) break;       // b2 == 0: nothing can come closer (all-duplicate clouds stay linear)
        second |= 1u << dep;
        h ^= 1u;
        lb = gh_knn_node_bound(nodes, h, p.x, p.y, p.z);
    }
    out[o] = gh_knn_mean3(b0, b1, b2);
}

int gh_knn_check(const char* who, long long P, const void* points, const void* workspace, size_t bytes)
{
    if (P < 0 || P > INT_MAX) return gh_set_error(GH_E_INVALID_ARG, "%s: P must lie in [0, 2^31)", who);
    if (P > 0 && (!points || !workspace)) return gh_set_error(GH_E_INVALID_ARG, "%s: missing points or workspace", who);
    if (P > 0 && ((size_t)points & 3)) return gh_set_error(GH_E_INVALID_ARG, "%s: points must be 4-byte aligned", who);
    if (P > 0 && bytes < GhKnnWS::bytes((size_t)P))
        return gh_set_error(GH_E_INVALID_ARG, "%s: workspace smaller than gh_knn_workspace_size", who);
    return GH_OK;
}

}  // namespace

extern "C" int gh_knn_workspace_size(long long P, size_t* bytes)
{
    gh_clear_error();
    if (P < 0 || P > INT_MAX) return gh_set_error(GH_E_INVALID_ARG, "gh_knn_workspace_size: P must lie in [0, 2^31)");
    if (bytes) *bytes = GhKnnWS::bytes((size_t)P);
    return GH_OK;
}

extern "C" int gh_knn_morton(long long P, const float* points, long long* codes, void* workspace, size_t bytes,
                             gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_knn_check("gh_knn_morton", P, points, workspace, bytes);
    if (rc != GH_OK) return rc;
    if (P == 0) return GH_OK;
    if (!codes || ((size_t)codes & 7)) return gh_set_error(GH_E_INVALID_ARG, "gh_knn_morton: codes must be an 8-byte aligned int64 array");
    const GhKnnWS ws = GhKnnWS::carve((char*)workspace, (size_t)P);
    const cudaError_t e = cudaMemsetAsync(ws.box, 0, 6 * sizeof(unsigned int), stream);
    if (e != cudaSuccess) return gh_cuda_status("gh_knn_morton", "memset(bounding box)", e);
    const int n = (int)P;
    const int blocks = (n + 255) / 256;
    gh_knn_bbox_kernel<<<min(blocks, 1024), 256, 0, stream>>>(n, points, ws.box);
    gh_knn_morton_kernel<<<blocks, 256, 0, stream>>>(n, points, ws.box, codes);
    return gh_launch_status("gh_knn_morton", 2);
}

extern "C" int gh_knn_mean_dist3(long long P, const float* points, const long long* order, float* out, void* workspace,
                                 size_t bytes, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_knn_check("gh_knn_mean_dist3", P, points, workspace, bytes);
    if (rc != GH_OK) return rc;
    if (P == 0) return GH_OK;
    if (!order || ((size_t)order & 7)) return gh_set_error(GH_E_INVALID_ARG, "gh_knn_mean_dist3: order must be an 8-byte aligned int64 array");
    if (!out || ((size_t)out & 3)) return gh_set_error(GH_E_INVALID_ARG, "gh_knn_mean_dist3: out must be a 4-byte aligned float array");
    const GhKnnWS ws = GhKnnWS::carve((char*)workspace, (size_t)P);
    const int n = (int)P;
    const unsigned int nleaf = 1u << ws.depth;
    gh_knn_leaves_kernel<<<(unsigned int)(((size_t)nleaf * 32 + 255) / 256), 256, 0, stream>>>(n, nleaf, points, order, ws.pts, ws.nodes);
    int launches = 1;
    for (int row = ws.depth; row > 0;) {
        const int steps = min(row, 8);
        const unsigned int blocks = ((1u << row) + GH_KNN_TREE_CTA - 1) / GH_KNN_TREE_CTA;
        gh_knn_tree_kernel<<<blocks, GH_KNN_TREE_CTA, 0, stream>>>(ws.nodes, row, steps);
        launches++;
        row -= steps;
    }
    gh_knn_query_kernel<<<(n + 127) / 128, 128, 0, stream>>>(n, ws.depth, ws.pts, ws.nodes, out);
    return gh_launch_status("gh_knn_mean_dist3", launches + 1);
}
