// TEST INFRASTRUCTURE: compiles the product's nearest-neighbour arithmetic (gaussianhaircut_b200/csrc/gh_knn_math.h,
// the functions the CUDA kernels call) for the host, so that the pruning bound can be checked against the distances
// it bounds where there is no GPU (tests/test_knn_cpu.py).  Build with -ffp-contract=off, like the oracle.
// Not part of libgh_raster.so; the product has no CPU path.
#include "../../gaussianhaircut_b200/csrc/gh_knn_math.h"

extern "C" void gh_host_knn_dist2(int n, const float* p, const float* q, float* out)
{
    for (int i = 0; i < n; i++)
        out[i] = gh_knn_dist2(p[3 * i], p[3 * i + 1], p[3 * i + 2], q[3 * i], q[3 * i + 1], q[3 * i + 2]);
}

extern "C" void gh_host_knn_box_bound(int n, const float* p, const float* lo, const float* hi, float* out)
{
    for (int i = 0; i < n; i++)
        out[i] = gh_knn_box_bound(p[3 * i], p[3 * i + 1], p[3 * i + 2], lo[3 * i], lo[3 * i + 1], lo[3 * i + 2],
                                  hi[3 * i], hi[3 * i + 1], hi[3 * i + 2]);
}
