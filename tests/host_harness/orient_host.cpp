// TEST INFRASTRUCTURE: compiles the product's orientation-map epilogue (gaussianhaircut_b200/csrc/gh_orient_math.h, the
// functions the Gabor kernel calls) for the host, so that it is checked bit for bit against a numpy float32 restatement
// of the reference's torch expressions where there is no GPU (tests/test_orient_cpu.py).  Build with -ffp-contract=off.
// Not part of libgh_raster.so; the product has no CPU path.
#include "../../gaussianhaircut_b200/csrc/gh_orient_math.h"

// F (npix, N) in the bank's channel order c = j*G + g; writes the pixel's orientation index and variance.
extern "C" void gh_host_orient_epilogue(int npix, int nf, int G, const float* F, const float* thetas, long long* idx,
                                        float* var)
{
    for (int p = 0; p < npix; p++) {
        int bi = 0;
        float bv = 0.f;
        for (int g = 0; g < G; g++) {
            int i;
            float v;
            gh_orient_group(F + (long long)p * nf * G + g, G, nf, thetas, &i, &v);
            gh_orient_keep(g, i, v, bi, bv);
        }
        idx[p] = bi;
        var[p] = bv;
    }
}
