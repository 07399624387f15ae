// TEST INFRASTRUCTURE: compiles the product's camera model (gaussianhaircut_b200/csrc/gh_camera_math.h, the functions
// the camera kernels call) for the host, so that it is checked against a float64 restatement and float64 autograd where
// there is no GPU (tests/test_cameras_cpu.py).  Build with -ffp-contract=off.  Not part of libgh_raster.so.
#include "../../gaussianhaircut_b200/csrc/gh_camera_math.h"

// n cameras: base (n, 18), r (n, 8) -> view (n, 16), proj (n, 16), campos (n, 3), tan_fov (n, 2)
extern "C" void gh_host_camera_forward(int n, const float* base, const float* r, float* view, float* proj, float* campos,
                                       float* tan_fov)
{
    for (int i = 0; i < n; i++)
        gh_camera_forward_math(base + i * GH_CAM_BASE, r + i * GH_CAM_ROW, view + i * 16, proj + i * 16, campos + i * 3,
                               tan_fov + i * 2);
}

// n cameras: base (n, 18), r (n, 8), g (n, 37) -> dr (n, 8)
extern "C" void gh_host_camera_backward(int n, const float* base, const float* r, const float* g, int intrinsics, float* dr)
{
    for (int i = 0; i < n; i++)
        gh_camera_backward_math(base + i * GH_CAM_BASE, r + i * GH_CAM_ROW, g + i * GH_CAM_DCAMERA, intrinsics,
                                dr + i * GH_CAM_ROW);
}
