// TEST INFRASTRUCTURE: compiles the product's per-face arithmetic (gaussianhaircut_b200/csrc/gh_mesh_math.h, the
// functions the CUDA kernels call) for the host, so that the face record and the per-pair distance and solid angle are
// checked against the float64 oracle where there is no GPU (tests/test_sdf_cpu.py).  Build with -ffp-contract=off.
// Not part of libgh_raster.so; the product has no CPU path.
#include "../../gaussianhaircut_b200/csrc/gh_mesh_math.h"

// tri (F,9): a, b, c of each face -> rec (F,28)
extern "C" void gh_host_sdf_record(int F, const float* tri, float* rec)
{
    for (int f = 0; f < F; f++) {
        GhSdfRecord r;
        gh_sdf_record(tri + 9 * f, tri + 9 * f + 3, tri + 9 * f + 6, r);
        for (int k = 0; k < 28; k++) rec[28 * f + k] = r.v[k];
    }
}

// pair i = (p[i], rec[i]) -> d2[i], omega[i]
extern "C" void gh_host_sdf_pair(int n, const float* p, const float* rec, float* d2, float* omega)
{
    for (int i = 0; i < n; i++) {
        GhSdfRecord r;
        for (int k = 0; k < 28; k++) r.v[k] = rec[28 * i + k];
        gh_sdf_pair(r, p[3 * i], p[3 * i + 1], p[3 * i + 2], d2[i], omega[i]);
    }
}
