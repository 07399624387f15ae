// Per-point arithmetic of the exact 3-nearest-neighbour kernels (gh_knn.cu), written once for device AND host: the
// CUDA kernels call these functions, and tests/host_harness/knn_host.cpp compiles this very header with g++ so that
// the pruning bound is checked against the distance it bounds on a machine without a GPU (tests/test_knn_cpu.py).
// The host build is test infrastructure only; libgh_raster.so contains no CPU path.
//
// Every operation is rounded on its own (no FMA contraction): the intrinsics on the device, -ffp-contract=off on the
// host.  The result of a query is a function of the multiset of float32 squared distances alone (DESIGN §14).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define GH_KNN_HD __host__ __device__ __forceinline__
#else
#define GH_KNN_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define GH_KNN_SUB(a, b) __fsub_rn((a), (b))
#define GH_KNN_ADD(a, b) __fadd_rn((a), (b))
#define GH_KNN_MUL(a, b) __fmul_rn((a), (b))
#define GH_KNN_DIV(a, b) __fdiv_rn((a), (b))
#else
#define GH_KNN_SUB(a, b) ((a) - (b))
#define GH_KNN_ADD(a, b) ((a) + (b))
#define GH_KNN_MUL(a, b) ((a) * (b))
#define GH_KNN_DIV(a, b) ((a) / (b))
#endif

// s = (dx*dx + dy*dy) + dz*dz with dx = q.x - p.x, ...
GH_KNN_HD float gh_knn_dist2(float px, float py, float pz, float qx, float qy, float qz)
{
    const float dx = GH_KNN_SUB(qx, px), dy = GH_KNN_SUB(qy, py), dz = GH_KNN_SUB(qz, pz);
    return GH_KNN_ADD(GH_KNN_ADD(GH_KNN_MUL(dx, dx), GH_KNN_MUL(dy, dy)), GH_KNN_MUL(dz, dz));
}

// Per-axis gap from p to [lo, hi]: max(lo - p, p - hi, 0), each difference rounded like dx.
GH_KNN_HD float gh_knn_gap(float p, float lo, float hi)
{
    return fmaxf(fmaxf(GH_KNN_SUB(lo, p), GH_KNN_SUB(p, hi)), 0.f);
}

// Lower bound of gh_knn_dist2(p, q) over every q with lo <= q <= hi (componentwise).
//
// Why it is a bound of the float32 distances, not only of the real ones: take one axis and q in [lo, hi].  If p < lo,
// the real q - p >= lo - p, and rounding to nearest is monotone, so fl(q - p) >= fl(lo - p) = gap.  If p > hi,
// fl(p - q) >= fl(p - hi) = gap, and fl(q - p) = -fl(p - q) (round to nearest is symmetric).  Otherwise gap = 0.  So
// |dx| >= gap on every axis, hence fl(dx*dx) >= fl(gap*gap), and the two additions, done in the same order as in
// gh_knn_dist2 on operands that are each no smaller, give a sum that is no smaller.  An empty box (lo = +inf,
// hi = -inf) gives +inf.  A node whose bound is >= the current third-smallest distance b2 cannot hold a point with
// s < b2, so pruning it never drops one of the three smallest float32 distances.
GH_KNN_HD float gh_knn_box_bound(float px, float py, float pz, float lox, float loy, float loz,
                                 float hix, float hiy, float hiz)
{
    const float gx = gh_knn_gap(px, lox, hix), gy = gh_knn_gap(py, loy, hiy), gz = gh_knn_gap(pz, loz, hiz);
    return GH_KNN_ADD(GH_KNN_ADD(GH_KNN_MUL(gx, gx), GH_KNN_MUL(gy, gy)), GH_KNN_MUL(gz, gz));
}

// Keep b0 <= b1 <= b2, the three smallest values seen.  A NaN never enters (s < b2 is false), and neither does a value
// equal to b2: the multiset of the three smallest is the same either way.
GH_KNN_HD void gh_knn_insert(float s, float& b0, float& b1, float& b2)
{
    if (s < b2) {
        if (s < b1) {
            b2 = b1;
            if (s < b0) { b1 = b0; b0 = s; } else { b1 = s; }
        } else {
            b2 = s;
        }
    }
}

GH_KNN_HD float gh_knn_mean3(float b0, float b1, float b2)
{
    return GH_KNN_DIV(GH_KNN_ADD(GH_KNN_ADD(b0, b1), b2), 3.0f);
}
