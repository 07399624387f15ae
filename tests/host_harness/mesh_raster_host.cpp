// TEST INFRASTRUCTURE: compiles the mesh rasterizer's per-face and per-pixel arithmetic (gaussianhaircut_b200/csrc/
// gh_mesh_math.h, the functions the CUDA kernels call) for the host, so that coverage decisions and depth bits are
// checked against the float64 oracle (tests/_meshraster64.py) where there is no GPU, and so that the kernel's
// pix_to_face can be compared with a brute-force z-buffer bit for bit (tests/test_mesh_raster_cpu.py,
// tests/test_gpu_mesh_raster.py).  Build with -ffp-contract=off.  Not part of libgh_raster.so.
#include <stdint.h>

#include "../../gaussianhaircut_b200/csrc/gh_mesh_math.h"

static void camera(const float* K, float* cam) { cam[0] = K[0]; cam[1] = K[4]; cam[2] = K[2]; cam[3] = K[5]; }

// one view: K (3,3), R (3,3), t (3) -> rec (F,20) as raw words, code (F): GH_RASTER_* or -1 for a face index out of
// range
extern "C" void gh_host_raster_setup(int V, int F, const float* verts, const int* faces, const float* K, const float* R,
                                     const float* t, int H, int W, GhRasterFace* rec, int* code)
{
    float cam[4];
    camera(K, cam);
    for (int f = 0; f < F; f++) {
        const int* i = faces + 3 * f;
        rec[f] = GhRasterFace{};
        if (!gh_mesh_face_in_range(i[0], i[1], i[2], V)) { code[f] = -1; continue; }
        code[f] = gh_raster_setup(cam, R, t, verts + 3 * i[0], verts + 3 * i[1], verts + 3 * i[2], H, W, rec[f]);
    }
}

// pair n = (face[n], pixel (row[n], col[n])) of one view's records -> w (n,3), covered (n), z (n)
extern "C" void gh_host_raster_pairs(int n, const GhRasterFace* rec, const int* face, const int* row, const int* col,
                                     float* w, int* covered, float* z)
{
    for (int k = 0; k < n; k++) {
        const GhRasterFace& r = rec[face[k]];
        gh_raster_edges(r, row[k], col[k], w + 3 * k);
        covered[k] = gh_raster_pixel(r, row[k], col[k], z[k]);
    }
}

// brute-force z-buffer of B views in the kernels' rule (the smallest (z bits, face) key over each face's box) ->
// pix_to_face (B,H,W); status |= GH_STATUS_* bits as the kernels set them
extern "C" void gh_host_raster_brute(int V, int F, const float* verts, const int* faces, int B, const float* K,
                                     const float* R, const float* t, int H, int W, int* pix_to_face, unsigned* status)
{
    uint64_t* key = new uint64_t[(size_t)H * W];
    for (int b = 0; b < B; b++) {
        float cam[4];
        camera(K + 9 * b, cam);
        for (size_t p = 0; p < (size_t)H * W; p++) key[p] = ~(uint64_t)0;
        for (int f = 0; f < F; f++) {
            const int* i = faces + 3 * f;
            if (!gh_mesh_face_in_range(i[0], i[1], i[2], V)) { *status |= 4u; continue; }
            GhRasterFace r;
            const int code = gh_raster_setup(cam, R + 9 * b, t + 3 * b, verts + 3 * i[0], verts + 3 * i[1],
                                             verts + 3 * i[2], H, W, r);
            if (code == GH_RASTER_NEAR) *status |= 8u;
            for (int y = r.i0; y < r.i0 + r.ni; y++)
                for (int x = r.j0; x < r.j0 + r.nj; x++) {
                    float z;
                    if (!gh_raster_pixel(r, y, x, z)) continue;
                    uint32_t zb;
                    __builtin_memcpy(&zb, &z, 4);
                    const uint64_t k = ((uint64_t)zb << 32) | (uint32_t)f;
                    if (k < key[(size_t)y * W + x]) key[(size_t)y * W + x] = k;
                }
        }
        for (size_t p = 0; p < (size_t)H * W; p++) pix_to_face[(size_t)b * H * W + p] = (int)(uint32_t)key[p];
    }
    delete[] key;
}
