// TEST INFRASTRUCTURE: the strand instantiation of the product's per-Gaussian projection arithmetic
// (gaussianhaircut_b200/csrc/gh_project_math.h with STRAND = true, what the strand-mode kernels call) compiled for the
// host, so that the derived geometry and the folded backward are checked against PyTorch autograd without a GPU
// (tests/test_strands_cpu.py).  Not part of libgh_raster.so.
#include "../../gaussianhaircut_b200/csrc/gh_project_math.h"

#include <cstring>

static GhProjArgs make_args(int P, int W, int H, const float* xyz, const float* scale, const float* dirs, const float* f_dc,
                            const float* f_rest, const float* conf, const float* V, const float* Pm, const float* campos,
                            float tanx, float tany, float mod, int sh_degree, unsigned int flags, float det_eps)
{
    GhProjArgs A;
    A.P = P; A.W = W; A.H = H; A.mod = mod; A.det_eps = det_eps; A.tanx = tanx; A.tany = tany; A.sh_degree = sh_degree;
    A.scale_act = (int)(flags & 3u); A.opacity_act = (int)((flags >> 2) & 3u); A.label_act = (int)((flags >> 4) & 3u);
    A.conf_act = (int)((flags >> 6) & 3u); A.dir_mode = (int)((flags >> 8) & 3u);
    A.xyz = xyz; A.scaling = scale; A.rotation = nullptr; A.dirs = dirs; A.f_dc = f_dc; A.f_rest = f_rest;
    A.opacity = nullptr; A.label = nullptr; A.conf = conf; A.V = V; A.Pm = Pm; A.campos = campos;
    return A;
}

extern "C" void gh_host_strand_forward(
    int P, int W, int H, const float* xyz, const float* scale, const float* dirs, const float* f_dc, const float* f_rest,
    const float* conf, const float* V, const float* Pm, const float* campos, float tanx, float tany, float mod, int sh_degree,
    unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opac, float* conic, float* cov3D, unsigned char* visible)
{
    GhProjArgs A = make_args(P, W, H, xyz, scale, dirs, f_dc, f_rest, conf, V, Pm, campos, tanx, tany, mod, sh_degree, flags, det_eps);
    for (int i = 0; i < P; i++) {
        GhProjOut o;
        gh_project_forward_one<true>(A, i, f_rest + (size_t)i * GH_PJ_REST, true, o);
        for (int k = 0; k < 3; k++) { means2D[3 * i + k] = o.m2[k]; conic[3 * i + k] = o.conic[k]; }
        opac[i] = o.opacity;
        for (int k = 0; k < GH_PJ_CHANNELS; k++) colors[GH_PJ_CHANNELS * i + k] = o.color[k];
        for (int k = 0; k < 6; k++) cov3D[6 * i + k] = o.cov3D[k];
        visible[i] = o.visible ? 1 : 0;
    }
}

// g_conic3 is the PUBLIC 3-vector conic gradient [g00, 2 g01, g11].  d_dirs = the direct term of each segment (scale
// and rotation folded in), d_xyz = the gradient w.r.t. its midpoint; d_scaling_rotation receives the 7 values the
// strand path leaves in go.scaling / go.rotation (all zero).
extern "C" void gh_host_strand_backward(
    int P, int W, int H, const float* xyz, const float* scale, const float* dirs, const float* f_dc, const float* f_rest,
    const float* conf, const float* V, const float* Pm, const float* campos, float tanx, float tany, float mod, int sh_degree,
    unsigned int flags, float det_eps, const unsigned char* visible,
    const float* g_means2D, const float* g_conic3, const float* g_colors,
    float* d_xyz, float* d_dirs, float* d_fdc, float* d_frest, float* d_conf, float* d_scaling_rotation, double* d_cam29)
{
    GhProjArgs A = make_args(P, W, H, xyz, scale, dirs, f_dc, f_rest, conf, V, Pm, campos, tanx, tany, mod, sh_degree, flags, det_eps);
    for (int k = 0; k < GH_PJ_NCAM; k++) d_cam29[k] = 0.0;
    for (int i = 0; i < P; i++) {
        GhProjGradOut go;
        std::memset(&go, 0, sizeof go);
        float cam[GH_PJ_NCAM] = {0};
        if (visible[i]) {
            GhProjGradIn gi;
            gi.m2x = g_means2D[3 * i]; gi.m2y = g_means2D[3 * i + 1];
            for (int k = 0; k < 3; k++) gi.con[k] = g_conic3[3 * i + k];
            for (int k = 0; k < GH_PJ_CHANNELS; k++) gi.color[k] = g_colors[GH_PJ_CHANNELS * i + k];
            gi.opacity = 0.f;
            gh_project_backward_one<true>(A, i, f_rest + (size_t)i * GH_PJ_REST, gi, go, cam);
        }
        for (int k = 0; k < 3; k++) { d_xyz[3 * i + k] = go.xyz[k]; d_dirs[3 * i + k] = go.dirs[k]; d_fdc[3 * i + k] = go.f_dc[k]; }
        for (int k = 0; k < GH_PJ_REST; k++) d_frest[(size_t)GH_PJ_REST * i + k] = go.rest[k];
        d_conf[i] = go.conf;
        for (int k = 0; k < 3; k++) d_scaling_rotation[7 * i + k] = go.scaling[k];
        for (int k = 0; k < 4; k++) d_scaling_rotation[7 * i + 3 + k] = go.rotation[k];
        for (int k = 0; k < GH_PJ_NCAM; k++) d_cam29[k] += (double)cam[k];
    }
}
