// Per-pixel epilogue of the orientation-map kernels (gh_orient.cu), written once for device AND host: the Gabor kernel
// calls these functions, and tests/host_harness/orient_host.cpp compiles this very header with g++ so that it is
// checked bit for bit against a numpy float32 restatement of the reference's torch expressions (tests/test_orient_cpu.py).
// The host build is test infrastructure only; libgh_raster.so contains no CPU path.
//
// For one group g of one pixel, with F_j = |response_j| (j < num_filters, theta-major channel j*G + g):
//   idx = argmax_j F_j (first on ties),  a = (idx / num_filters) * pi,
//   d_j = min(|a - theta_j|, min(|(a - theta_j) - pi|, |(a - theta_j) + pi|)),
//   S = max(sum_j F_j, 1e-12),  var = sum_j (d_j * d_j) * (F_j / S),
// both sums in increasing j, every operation rounded on its own in float32 (DESIGN §15).  Across groups the pixel keeps
// the first group with the smallest var.  All-zero responses give idx 0 and var 0.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define GH_OR_HD __host__ __device__ __forceinline__
#else
#define GH_OR_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define GH_OR_SUB(a, b) __fsub_rn((a), (b))
#define GH_OR_ADD(a, b) __fadd_rn((a), (b))
#define GH_OR_MUL(a, b) __fmul_rn((a), (b))
#define GH_OR_DIV(a, b) __fdiv_rn((a), (b))
#else
#define GH_OR_SUB(a, b) ((a) - (b))
#define GH_OR_ADD(a, b) ((a) + (b))
#define GH_OR_MUL(a, b) ((a) * (b))
#define GH_OR_DIV(a, b) ((a) / (b))
#endif

#define GH_OR_PI 3.14159265358979323846f   // math.pi as torch rounds a Python scalar for a float32 tensor
#define GH_OR_EPS 1e-12f                    // F.normalize's eps

// The angular distance between the winning orientation a and theta_j, with the wrap-around at pi.
GH_OR_HD float gh_orient_dist(float a, float theta)
{
    const float t = GH_OR_SUB(a, theta);
    return fminf(fabsf(t), fminf(fabsf(GH_OR_SUB(t, GH_OR_PI)), fabsf(GH_OR_ADD(t, GH_OR_PI))));
}

// One group: F[j * stride] for j < nf.  Writes idx and var.
GH_OR_HD void gh_orient_group(const float* F, int stride, int nf, const float* thetas, int* idx_out, float* var_out)
{
    float fmax = F[0], sum = 0.f;
    int idx = 0;
    for (int j = 0; j < nf; j++) {
        const float f = F[(long long)j * stride];
        if (f > fmax) { fmax = f; idx = j; }
        sum = GH_OR_ADD(sum, f);
    }
    const float S = fmaxf(sum, GH_OR_EPS);
    const float a = GH_OR_MUL(GH_OR_DIV((float)idx, (float)nf), GH_OR_PI);
    float var = 0.f;
    for (int j = 0; j < nf; j++) {
        const float d = gh_orient_dist(a, thetas[j]);
        var = GH_OR_ADD(var, GH_OR_MUL(GH_OR_MUL(d, d), GH_OR_DIV(F[(long long)j * stride], S)));
    }
    *idx_out = idx;
    *var_out = var;
}

// Across groups: keep the first group with the smallest var (torch.argmin's tie rule).
GH_OR_HD void gh_orient_keep(int g, int idx, float var, int& best_idx, float& best_var)
{
    if (g == 0 || var < best_var) { best_idx = idx; best_var = var; }
}
