// Per-Gaussian arithmetic of the fused projection preamble (gh_project.cu), written once for device AND host:
// the CUDA kernels call these functions, and tests/host_harness compiles this very header with g++ so that the
// hand-derived backward is checked against PyTorch autograd on a machine without a GPU (tests/test_project_cpu.py).
// The host build is test infrastructure only; libgh_raster.so contains no CPU path.
//
// What is computed (row-vector convention of the reference's Python: t = x . V[:3,:3] + V[3,:3]):
//   s = exp(log s) * mod (or the activated scale)          gaussian_model.py:231-233 / latent_strands :110-115
//   R = build_rotation(q / |q|)                            general_utils.py:79-109 (normalises, transposed layout)
//   Sigma = sum_i s_i^2 R[i]^T R[i]                        (S R)^T (S R), gaussian_model.py:242-245
//   u0 = T[:,0], u1 = T[:,1], T = V[:3,:3] @ J             gaussian_model.py:252-297 (J from the clamped position)
//   a = sum_i s_i^2 (R[i].u0)^2 + 0.3, b = sum_i s_i^2 (R[i].u0)(R[i].u1), c = sum_i s_i^2 (R[i].u1)^2 + 0.3
//   conic = (c, -b, a) / (ac - b^2 + eps)                  :303-315, eps 1e-12; strand models eps 1e-7 (:355)
//   means2D = (x . Pm[:3] + Pm[3])[:3] / (w + 1e-7)        :317-337          depth = t.z  :339-342
//   dir2D = d3 . T, d3 = s_max R[argmax s] (:385-391) or normalize(dir) (latent_strands :437-438)
//   rgb = max(SH(normalize(x - campos)) + 0.5, 0)          sh_utils.py:57-112, gaussian_renderer/__init__.py:58-66
//   visible = filter_points                                gaussian_model.py:143-228
#pragma once
#include <math.h>
#include <stddef.h>

#ifdef __CUDACC__
#define GH_HD __host__ __device__ __forceinline__
#else
#define GH_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define GH_LDG(p) __ldg(p)
#else
#define GH_LDG(p) (*(p))
#endif

#define GH_PJ_REST 45          // floats per f_rest row: 15 coefficients x RGB
#define GH_PJ_NCAM 29          // camera-gradient accumulators: V[i][j<3] 12, Pm[i][0,1,3] 12, campos 3, tan(fov/2) 2
#define GH_PJ_CHANNELS 10

#define GH_SH_C0 0.28209479177387814f
#define GH_SH_C1 0.4886025119029199f
#define GH_SH_C20 1.0925484305920792f
#define GH_SH_C21 (-1.0925484305920792f)
#define GH_SH_C22 0.31539156525252005f
#define GH_SH_C23 (-1.0925484305920792f)
#define GH_SH_C24 0.5462742152960396f
#define GH_SH_C30 (-0.5900435899266435f)
#define GH_SH_C31 2.890611442640554f
#define GH_SH_C32 (-0.4570457994644658f)
#define GH_SH_C33 0.3731763325901154f
#define GH_SH_C34 (-0.4570457994644658f)
#define GH_SH_C35 1.445305721320277f
#define GH_SH_C36 (-0.5900435899266435f)

struct GhProjArgs {
    int P, W, H;
    float mod, det_eps, tanx, tany;
    int sh_degree;
    int scale_act;      // 0: scales are activated values, 1: exp()
    int opacity_act;    // 0: identity, 1: sigmoid, 2: constant 1 (input ignored)
    int label_act;      // 0: identity, 1: sigmoid, 2: constant 1, 3: constant 0
    int conf_act;       // 0: identity, 1: exp, 3: constant 0
    int dir_mode;       // 0: s_max * R[argmax s], 1: normalize(dirs[i]), 2: zero
    const float* xyz; const float* scaling; const float* rotation; const float* dirs;
    const float* f_dc; const float* f_rest; const float* opacity; const float* label; const float* conf;
    const float* V; const float* Pm; const float* campos;
};

GH_HD float gh_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
GH_HD int gh_imin(int a, int b) { return a < b ? a : b; }
GH_HD int gh_imax(int a, int b) { return a > b ? a : b; }
GH_HD float gh_sel3(float a0, float a1, float a2, int j) { return j == 0 ? a0 : (j == 1 ? a1 : a2); }

// SH basis values B[16] (sh_utils.py:57-112) for the unit direction (x, y, z)
GH_HD void gh_sh_basis(int deg, float x, float y, float z, float* B) {
#pragma unroll
    for (int k = 0; k < 16; k++) B[k] = 0.f;
    B[0] = GH_SH_C0;
    if (deg > 0) {
        B[1] = -GH_SH_C1 * y; B[2] = GH_SH_C1 * z; B[3] = -GH_SH_C1 * x;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            B[4] = GH_SH_C20 * xy; B[5] = GH_SH_C21 * yz; B[6] = GH_SH_C22 * (2.0f * zz - xx - yy);
            B[7] = GH_SH_C23 * xz; B[8] = GH_SH_C24 * (xx - yy);
            if (deg > 2) {
                B[9] = GH_SH_C30 * y * (3.f * xx - yy); B[10] = GH_SH_C31 * xy * z;
                B[11] = GH_SH_C32 * y * (4.f * zz - xx - yy); B[12] = GH_SH_C33 * z * (2.f * zz - 3.f * xx - 3.f * yy);
                B[13] = GH_SH_C34 * x * (4.f * zz - xx - yy); B[14] = GH_SH_C35 * z * (xx - yy);
                B[15] = GH_SH_C36 * x * (xx - 3.f * yy);
            }
        }
    }
}

// d B_k / d(x, y, z), the components treated as independent variables (what autograd sees)
GH_HD void gh_sh_basis_grad(int deg, float x, float y, float z, float* Bx, float* By, float* Bz) {
#pragma unroll
    for (int k = 0; k < 16; k++) { Bx[k] = 0.f; By[k] = 0.f; Bz[k] = 0.f; }
    if (deg > 0) {
        By[1] = -GH_SH_C1; Bz[2] = GH_SH_C1; Bx[3] = -GH_SH_C1;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            Bx[4] = GH_SH_C20 * y; By[4] = GH_SH_C20 * x;
            By[5] = GH_SH_C21 * z; Bz[5] = GH_SH_C21 * y;
            Bx[6] = -2.f * GH_SH_C22 * x; By[6] = -2.f * GH_SH_C22 * y; Bz[6] = 4.f * GH_SH_C22 * z;
            Bx[7] = GH_SH_C23 * z; Bz[7] = GH_SH_C23 * x;
            Bx[8] = 2.f * GH_SH_C24 * x; By[8] = -2.f * GH_SH_C24 * y;
            if (deg > 2) {
                Bx[9] = 6.f * GH_SH_C30 * xy; By[9] = GH_SH_C30 * (3.f * xx - 3.f * yy);
                Bx[10] = GH_SH_C31 * yz; By[10] = GH_SH_C31 * xz; Bz[10] = GH_SH_C31 * xy;
                Bx[11] = -2.f * GH_SH_C32 * xy; By[11] = GH_SH_C32 * (4.f * zz - xx - 3.f * yy); Bz[11] = 8.f * GH_SH_C32 * yz;
                Bx[12] = -6.f * GH_SH_C33 * xz; By[12] = -6.f * GH_SH_C33 * yz; Bz[12] = GH_SH_C33 * (6.f * zz - 3.f * xx - 3.f * yy);
                Bx[13] = GH_SH_C34 * (4.f * zz - 3.f * xx - yy); By[13] = -2.f * GH_SH_C34 * xy; Bz[13] = 8.f * GH_SH_C34 * xz;
                Bx[14] = 2.f * GH_SH_C35 * xz; By[14] = -2.f * GH_SH_C35 * yz; Bz[14] = GH_SH_C35 * (xx - yy);
                Bx[15] = GH_SH_C36 * (3.f * xx - 3.f * yy); By[15] = -6.f * GH_SH_C36 * xy;
            }
        }
    }
}

// Geometry shared by forward and backward: everything up to the 2-D covariance.
struct GhProjGeo {
    float x[3];          // position
    float s[3];          // activated scale * modifier
    float qn[4], qlen;   // normalised quaternion, |q|
    float R[3][3];       // build_rotation layout (row i = axis i)
    float t[3];          // view-space position
    float txc, tyc;      // clamped tx, ty (times tz)
    bool clx, cly;       // x / y clamp active
    float sgx, sgy;      // sign of the active clamp
    float fx, fy;
    float j00, j20, j11, j21;
    float u0[3], u1[3];
    float w0[3], w1[3];  // R[i].u0, R[i].u1
    float a, b, c;       // cov2D incl. the 0.3 low-pass
};

// STRAND: the Gaussian is segment i of a polyline (gaussian_model_strands.py:435-454).  Its scales and rotation are
// derived in registers from the segment vector d = dirs[i]: scales (|d|/2, scale, scale) with the strand thickness
// `scale` = scaling[0] (one float for the whole model), rotation parallel_transport(e_x, d) = (1 + b.x, 0, -b.z, b.y)
// with b = d / max(|d|, 1e-12) (general_utils.py:150-160).  `rotation` is not read.
template <bool STRAND = false>
GH_HD void gh_proj_geometry(const GhProjArgs& A, int i, GhProjGeo& g) {
    g.x[0] = A.xyz[3 * (size_t)i]; g.x[1] = A.xyz[3 * (size_t)i + 1]; g.x[2] = A.xyz[3 * (size_t)i + 2];
    float q0, q1, q2, q3;
    if constexpr (STRAND) {
        const float dx = A.dirs[3 * (size_t)i], dy = A.dirs[3 * (size_t)i + 1], dz = A.dirs[3 * (size_t)i + 2];
        const float dn = sqrtf(dx * dx + dy * dy + dz * dz);
        const float th = GH_LDG(A.scaling) * A.mod;
        g.s[0] = (dn * 0.5f) * A.mod; g.s[1] = th; g.s[2] = th;
        const float ib = 1.0f / fmaxf(dn, 1e-12f);
        q0 = 1.0f + dx * ib; q1 = 0.f; q2 = -(dz * ib); q3 = dy * ib;
    } else {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float v = A.scaling[3 * (size_t)i + k];
            g.s[k] = (A.scale_act == 1 ? expf(v) : v) * A.mod;
        }
        const float* qp = A.rotation + 4 * (size_t)i;
        q0 = qp[0]; q1 = qp[1]; q2 = qp[2]; q3 = qp[3];
    }
    g.qlen = sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
    const float il = 1.0f / g.qlen;
    const float r = q0 * il, x = q1 * il, y = q2 * il, z = q3 * il;
    g.qn[0] = r; g.qn[1] = x; g.qn[2] = y; g.qn[3] = z;
    g.R[0][0] = 1.f - 2.f * (y * y + z * z); g.R[1][0] = 2.f * (x * y - r * z); g.R[2][0] = 2.f * (x * z + r * y);
    g.R[0][1] = 2.f * (x * y + r * z); g.R[1][1] = 1.f - 2.f * (x * x + z * z); g.R[2][1] = 2.f * (y * z - r * x);
    g.R[0][2] = 2.f * (x * z - r * y); g.R[1][2] = 2.f * (y * z + r * x); g.R[2][2] = 1.f - 2.f * (x * x + y * y);
    const float* V = A.V;
#pragma unroll
    for (int j = 0; j < 3; j++)
        g.t[j] = g.x[0] * GH_LDG(V + j) + g.x[1] * GH_LDG(V + 4 + j) + g.x[2] * GH_LDG(V + 8 + j) + GH_LDG(V + 12 + j);
    const float tz = g.t[2];
    const float limx = 1.3f * A.tanx, limy = 1.3f * A.tany;
    const float txtz = g.t[0] / tz, tytz = g.t[1] / tz;
    g.clx = (txtz < -limx) || (txtz > limx); g.cly = (tytz < -limy) || (tytz > limy);
    g.sgx = txtz < 0.f ? -1.f : 1.f; g.sgy = tytz < 0.f ? -1.f : 1.f;
    g.txc = fminf(limx, fmaxf(-limx, txtz)) * tz;
    g.tyc = fminf(limy, fmaxf(-limy, tytz)) * tz;
    g.fx = A.W / (2.0f * A.tanx); g.fy = A.H / (2.0f * A.tany);
    const float itz = 1.0f / tz, itz2 = itz * itz;
    g.j00 = g.fx * itz; g.j20 = -(g.fx * g.txc) * itz2;
    g.j11 = g.fy * itz; g.j21 = -(g.fy * g.tyc) * itz2;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        g.u0[k] = GH_LDG(V + 4 * k + 0) * g.j00 + GH_LDG(V + 4 * k + 2) * g.j20;
        g.u1[k] = GH_LDG(V + 4 * k + 1) * g.j11 + GH_LDG(V + 4 * k + 2) * g.j21;
    }
    float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        g.w0[k] = g.R[k][0] * g.u0[0] + g.R[k][1] * g.u0[1] + g.R[k][2] * g.u0[2];
        g.w1[k] = g.R[k][0] * g.u1[0] + g.R[k][1] * g.u1[1] + g.R[k][2] * g.u1[2];
        const float s2 = g.s[k] * g.s[k];
        a += s2 * g.w0[k] * g.w0[k]; b += s2 * g.w0[k] * g.w1[k]; c += s2 * g.w1[k] * g.w1[k];
    }
    g.a = a + 0.3f; g.b = b; g.c = c + 0.3f;
}

// torch.argsort(descending=True)[0]: the largest scale (first index on exact ties)
GH_HD int gh_argmax3(float s0, float s1, float s2) {
    int j = 0;
    float m = s0;
    if (s1 > m) { j = 1; m = s1; }
    if (s2 > m) j = 2;
    return j;
}

// the caller's prefilter (gaussian_model.py:143-228)
GH_HD bool gh_proj_visible(const GhProjArgs& A, const GhProjGeo& g, float m2x, float m2y) {
    const float det = g.a * g.c - g.b * g.b;
    if (!(g.t[2] > 0.2f) || det == 0.f) return false;
    const float mid = 0.5f * (g.a + g.c);
    const float sq = sqrtf(fmaxf(mid * mid - det, 0.1f));
    const float rad = ceilf(3.f * sqrtf(fmaxf(mid + sq, mid - sq)));
    const float px = ((m2x + 1.f) * A.W - 1.0f) * 0.5f, py = ((m2y + 1.f) * A.H - 1.0f) * 0.5f;
    const int gx = (A.W + 15) / 16, gy = (A.H + 15) / 16;
    const int x0 = gh_imin(gx, gh_imax(0, (int)((px - rad) / 16.f))), y0 = gh_imin(gy, gh_imax(0, (int)((py - rad) / 16.f)));
    const int x1 = gh_imin(gx, gh_imax(0, (int)((px + rad + 15.f) / 16.f))), y1 = gh_imin(gy, gh_imax(0, (int)((py + rad + 15.f) / 16.f)));
    return (x1 - x0) * (y1 - y0) != 0;
}

struct GhProjOut {
    float m2[3];                      // NDC mean
    float conic[3];                   // zeros when culled
    float opacity;
    float color[GH_PJ_CHANNELS];
    float cov3D[6];
    bool visible;
};

// One Gaussian, forward.  `rest` = this Gaussian's f_rest row (45 floats, coefficient-major, RGB-minor).
template <bool STRAND = false>
GH_HD void gh_project_forward_one(const GhProjArgs& A, int i, const float* rest, bool want_cov3D, GhProjOut& o) {
    GhProjGeo g;
    gh_proj_geometry<STRAND>(A, i, g);
    const float* Pm = A.Pm;
    float h[4];
#pragma unroll
    for (int j = 0; j < 4; j++)
        h[j] = g.x[0] * GH_LDG(Pm + j) + g.x[1] * GH_LDG(Pm + 4 + j) + g.x[2] * GH_LDG(Pm + 8 + j) + GH_LDG(Pm + 12 + j);
    const float p_w = 1.0f / (h[3] + 0.0000001f);
    o.m2[0] = h[0] * p_w; o.m2[1] = h[1] * p_w; o.m2[2] = h[2] * p_w;
    o.visible = gh_proj_visible(A, g, o.m2[0], o.m2[1]);
    const float det = g.a * g.c - g.b * g.b;
    const float inv = 1.0f / (det + A.det_eps);
    // a culled Gaussian gets a zero conic: the rasterizer drops it (zero determinant, forward.cu:243-245)
    o.conic[0] = o.visible ? g.c * inv : 0.f; o.conic[1] = o.visible ? -g.b * inv : 0.f; o.conic[2] = o.visible ? g.a * inv : 0.f;
    if (want_cov3D) {
        // Sigma = sum_k s_k^2 R[k]^T R[k], stored [xx, xy, xz, yy, yz, zz] (strip_symmetric)
#pragma unroll
        for (int k = 0; k < 6; k++) o.cov3D[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float s2 = g.s[k] * g.s[k];
            o.cov3D[0] += s2 * g.R[k][0] * g.R[k][0]; o.cov3D[1] += s2 * g.R[k][0] * g.R[k][1]; o.cov3D[2] += s2 * g.R[k][0] * g.R[k][2];
            o.cov3D[3] += s2 * g.R[k][1] * g.R[k][1]; o.cov3D[4] += s2 * g.R[k][1] * g.R[k][2]; o.cov3D[5] += s2 * g.R[k][2] * g.R[k][2];
        }
    }
    const float op = A.opacity_act == 2 ? 1.0f : A.opacity[i];
    o.opacity = A.opacity_act == 1 ? gh_sigmoid(op) : op;

    float d3[3] = {0.f, 0.f, 0.f};
    if (A.dir_mode == 0) {
        const int jm = gh_argmax3(g.s[0], g.s[1], g.s[2]);
        const float sj = gh_sel3(g.s[0], g.s[1], g.s[2], jm);
#pragma unroll
        for (int k = 0; k < 3; k++) d3[k] = gh_sel3(g.R[0][k], g.R[1][k], g.R[2][k], jm) * sj;
    } else if (A.dir_mode == 1) {
        const float dx = A.dirs[3 * (size_t)i], dy = A.dirs[3 * (size_t)i + 1], dz = A.dirs[3 * (size_t)i + 2];
        const float il = 1.0f / fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);    // F.normalize eps
        d3[0] = dx * il; d3[1] = dy * il; d3[2] = dz * il;
    }
    const float dir2x = d3[0] * g.u0[0] + d3[1] * g.u0[1] + d3[2] * g.u0[2];
    const float dir2y = d3[0] * g.u1[0] + d3[1] * g.u1[1] + d3[2] * g.u1[2];

    float vx = g.x[0] - GH_LDG(A.campos), vy = g.x[1] - GH_LDG(A.campos + 1), vz = g.x[2] - GH_LDG(A.campos + 2);
    const float ivl = 1.0f / sqrtf(vx * vx + vy * vy + vz * vz);
    vx *= ivl; vy *= ivl; vz *= ivl;
    float B[16];
    gh_sh_basis(A.sh_degree, vx, vy, vz, B);
    const int ncoef = (A.sh_degree + 1) * (A.sh_degree + 1);
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        float acc = B[0] * A.f_dc[3 * (size_t)i + ch];
#pragma unroll
        for (int k = 1; k < 16; k++)
            if (k < ncoef) acc += B[k] * rest[3 * (k - 1) + ch];
        o.color[ch] = fmaxf(acc + 0.5f, 0.0f);
    }
    float lab = 0.f, cf = 0.f;
    if (A.label_act == 2) lab = 1.f; else if (A.label_act != 3) { lab = A.label[i]; if (A.label_act == 1) lab = gh_sigmoid(lab); }
    if (A.conf_act != 3) { cf = A.conf[i]; if (A.conf_act == 1) cf = expf(cf); }
    o.color[3] = lab; o.color[4] = 1.0f; o.color[5] = dir2x; o.color[6] = dir2y; o.color[7] = 0.0f; o.color[8] = cf; o.color[9] = g.t[2];
}

struct GhProjGradIn {
    float m2x, m2y;                   // dL/d NDC mean (x, y)
    float con[3];                     // dL/d conic (a, b, c) -- the PUBLIC 3-vector gradient [g00, 2 g01, g11]
    float color[GH_PJ_CHANNELS];
    float opacity;
};

struct GhProjGradOut {
    float xyz[3], scaling[3], rotation[4], dirs[3], f_dc[3];
    float opacity, label, conf;
    float rest[GH_PJ_REST];
};

// One Gaussian, backward.  `cam[29]` is ACCUMULATED into (caller zero-initialises):
//   [0..11]  dL/dV[i][j]  (i = 0..3 rows, j = 0..2)          index 3*i + j
//   [12..23] dL/dPm[i][c] (i = 0..3 rows, c in {0, 1, 3})    index 12 + 3*i + {0, 1, 2}
//   [24..26] dL/dcampos, [27..28] dL/dtan(fovx/2), dL/dtan(fovy/2)
// STRAND: the scale and rotation gradients are folded into go.dirs (the segment vector's direct term) and
// go.scaling / go.rotation come back as zeros; go.xyz is the gradient w.r.t. the segment's midpoint.
template <bool STRAND = false>
GH_HD void gh_project_backward_one(const GhProjArgs& A, int i, const float* rest, const GhProjGradIn& gi,
                                   GhProjGradOut& go, float* cam) {
    GhProjGeo g;
    gh_proj_geometry<STRAND>(A, i, g);
    const float* V = A.V;
    const float* Pm = A.Pm;
    float dx[3] = {0.f, 0.f, 0.f}, ds[3] = {0.f, 0.f, 0.f};
    float gt[3] = {0.f, 0.f, gi.color[9]};               // depth = t.z
    go.opacity = 0.f; go.label = 0.f; go.conf = 0.f;
    go.dirs[0] = 0.f; go.dirs[1] = 0.f; go.dirs[2] = 0.f;
    // ---- activations
    if (A.opacity_act == 1) { const float s = gh_sigmoid(A.opacity[i]); go.opacity = gi.opacity * s * (1.f - s); }
    else if (A.opacity_act == 0) go.opacity = gi.opacity;
    if (A.label_act == 1) { const float s = gh_sigmoid(A.label[i]); go.label = gi.color[3] * s * (1.f - s); }
    else if (A.label_act == 0) go.label = gi.color[3];
    if (A.conf_act == 1) go.conf = gi.color[8] * expf(A.conf[i]);
    else if (A.conf_act == 0) go.conf = gi.color[8];

    // ---- SH colour
    {
        float vx = g.x[0] - GH_LDG(A.campos), vy = g.x[1] - GH_LDG(A.campos + 1), vz = g.x[2] - GH_LDG(A.campos + 2);
        const float vl = sqrtf(vx * vx + vy * vy + vz * vz), ivl = 1.0f / vl;
        vx *= ivl; vy *= ivl; vz *= ivl;
        float B[16];
        gh_sh_basis(A.sh_degree, vx, vy, vz, B);
        const int ncoef = (A.sh_degree + 1) * (A.sh_degree + 1);
        float grgb[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            float acc = B[0] * A.f_dc[3 * (size_t)i + ch];
#pragma unroll
            for (int k = 1; k < 16; k++)
                if (k < ncoef) acc += B[k] * rest[3 * (k - 1) + ch];
            grgb[ch] = (acc + 0.5f >= 0.0f) ? gi.color[ch] : 0.f;     // clamp_min(., 0)
            go.f_dc[ch] = B[0] * grgb[ch];
        }
        float gv[3] = {0.f, 0.f, 0.f};
        if (A.sh_degree > 0) {
            float Bx[16], By[16], Bz[16];
            gh_sh_basis_grad(A.sh_degree, vx, vy, vz, Bx, By, Bz);
#pragma unroll
            for (int k = 1; k < 16; k++) {
                if (k < ncoef) {
                    const float c = rest[3 * (k - 1)] * grgb[0] + rest[3 * (k - 1) + 1] * grgb[1] + rest[3 * (k - 1) + 2] * grgb[2];
                    gv[0] += Bx[k] * c; gv[1] += By[k] * c; gv[2] += Bz[k] * c;
                }
            }
        }
#pragma unroll
        for (int k = 1; k < 16; k++) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) go.rest[3 * (k - 1) + ch] = (k < ncoef) ? B[k] * grgb[ch] : 0.f;
        }
        const float dot = vx * gv[0] + vy * gv[1] + vz * gv[2];
        const float gd0 = (gv[0] - vx * dot) * ivl, gd1 = (gv[1] - vy * dot) * ivl, gd2 = (gv[2] - vz * dot) * ivl;
        dx[0] += gd0; dx[1] += gd1; dx[2] += gd2;
        cam[24] -= gd0; cam[25] -= gd1; cam[26] -= gd2;
    }

    float gu0[3] = {0.f, 0.f, 0.f}, gu1[3] = {0.f, 0.f, 0.f};
    float gR[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    // ---- dir2D = d3 . (u0, u1)
    {
        float d3[3] = {0.f, 0.f, 0.f};
        int jm = 0;
        float sjm = 0.f, dl = 1.f;
        if (A.dir_mode == 0) {
            jm = gh_argmax3(g.s[0], g.s[1], g.s[2]);
            sjm = gh_sel3(g.s[0], g.s[1], g.s[2], jm);
#pragma unroll
            for (int k = 0; k < 3; k++) d3[k] = gh_sel3(g.R[0][k], g.R[1][k], g.R[2][k], jm) * sjm;
        } else if (A.dir_mode == 1) {
            const float n0 = A.dirs[3 * (size_t)i], n1 = A.dirs[3 * (size_t)i + 1], n2 = A.dirs[3 * (size_t)i + 2];
            dl = fmaxf(sqrtf(n0 * n0 + n1 * n1 + n2 * n2), 1e-12f);
            d3[0] = n0 / dl; d3[1] = n1 / dl; d3[2] = n2 / dl;
        }
        const float g5 = gi.color[5], g6 = gi.color[6];
        float gd3[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            gd3[k] = g5 * g.u0[k] + g6 * g.u1[k];
            gu0[k] += g5 * d3[k]; gu1[k] += g6 * d3[k];
        }
        if (A.dir_mode == 0) {
            float dsj = 0.f;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                dsj += gh_sel3(g.R[0][k], g.R[1][k], g.R[2][k], jm) * gd3[k];
#pragma unroll
                for (int r = 0; r < 3; r++) gR[r][k] += (r == jm) ? sjm * gd3[k] : 0.f;
            }
#pragma unroll
            for (int r = 0; r < 3; r++) ds[r] += (r == jm) ? dsj : 0.f;
        } else if (A.dir_mode == 1) {
            const float dot = d3[0] * gd3[0] + d3[1] * gd3[1] + d3[2] * gd3[2];
#pragma unroll
            for (int k = 0; k < 3; k++) go.dirs[k] = (gd3[k] - d3[k] * dot) / dl;
        }
    }
    // ---- conic -> cov2D
    float ga, gb, gc;
    {
        const float det = g.a * g.c - g.b * g.b;
        const float inv = 1.0f / (det + A.det_eps);
        ga = gi.con[2] * inv; gc = gi.con[0] * inv; gb = -gi.con[1] * inv;
        const float ginv = gi.con[0] * g.c - gi.con[1] * g.b + gi.con[2] * g.a;
        const float gdet = -inv * inv * ginv;
        ga += gdet * g.c; gc += gdet * g.a; gb += -2.f * g.b * gdet;
    }
    // ---- cov2D -> scales, rotation rows, u0 / u1
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float s2 = g.s[k] * g.s[k];
        const float gw0 = s2 * (2.f * ga * g.w0[k] + gb * g.w1[k]);
        const float gw1 = s2 * (2.f * gc * g.w1[k] + gb * g.w0[k]);
        ds[k] += 2.f * g.s[k] * (ga * g.w0[k] * g.w0[k] + gb * g.w0[k] * g.w1[k] + gc * g.w1[k] * g.w1[k]);
#pragma unroll
        for (int m = 0; m < 3; m++) {
            gR[k][m] += gw0 * g.u0[m] + gw1 * g.u1[m];
            gu0[m] += gw0 * g.R[k][m]; gu1[m] += gw1 * g.R[k][m];
        }
    }
    // ---- u0 / u1 -> J entries and the view matrix
    float gj00 = 0.f, gj20 = 0.f, gj11 = 0.f, gj21 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        gj00 += gu0[k] * GH_LDG(V + 4 * k + 0); gj20 += gu0[k] * GH_LDG(V + 4 * k + 2);
        gj11 += gu1[k] * GH_LDG(V + 4 * k + 1); gj21 += gu1[k] * GH_LDG(V + 4 * k + 2);
        cam[3 * k + 0] += gu0[k] * g.j00;
        cam[3 * k + 1] += gu1[k] * g.j11;
        cam[3 * k + 2] += gu0[k] * g.j20 + gu1[k] * g.j21;
    }
    {
        const float tz = g.t[2], itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float gfx = gj00 * itz - g.txc * itz2 * gj20;
        const float gfy = gj11 * itz - g.tyc * itz2 * gj21;
        gt[2] += -g.fx * itz2 * gj00 + 2.f * g.fx * g.txc * itz3 * gj20 - g.fy * itz2 * gj11 + 2.f * g.fy * g.tyc * itz3 * gj21;
        const float gtxc = -g.fx * itz2 * gj20, gtyc = -g.fy * itz2 * gj21;
        float glimx = 0.f, glimy = 0.f;
        if (g.clx) { gt[2] += g.sgx * 1.3f * A.tanx * gtxc; glimx = g.sgx * tz * gtxc; } else gt[0] += gtxc;
        if (g.cly) { gt[2] += g.sgy * 1.3f * A.tany * gtyc; glimy = g.sgy * tz * gtyc; } else gt[1] += gtyc;
        cam[27] += -g.fx / A.tanx * gfx + 1.3f * glimx;
        cam[28] += -g.fy / A.tany * gfy + 1.3f * glimy;
    }
    // ---- view transform
#pragma unroll
    for (int k = 0; k < 3; k++) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
            dx[k] += gt[j] * GH_LDG(V + 4 * k + j);
            cam[3 * k + j] += g.x[k] * gt[j];
        }
    }
    cam[9] += gt[0]; cam[10] += gt[1]; cam[11] += gt[2];
    // ---- NDC mean
    {
        float h[4];
#pragma unroll
        for (int j = 0; j < 4; j++)
            h[j] = g.x[0] * GH_LDG(Pm + j) + g.x[1] * GH_LDG(Pm + 4 + j) + g.x[2] * GH_LDG(Pm + 8 + j) + GH_LDG(Pm + 12 + j);
        const float p_w = 1.0f / (h[3] + 0.0000001f);
        const float gh0 = gi.m2x * p_w, gh1 = gi.m2y * p_w;
        const float gh3 = -p_w * p_w * (gi.m2x * h[0] + gi.m2y * h[1]);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            dx[k] += gh0 * GH_LDG(Pm + 4 * k + 0) + gh1 * GH_LDG(Pm + 4 * k + 1) + gh3 * GH_LDG(Pm + 4 * k + 3);
            cam[12 + 3 * k + 0] += g.x[k] * gh0; cam[12 + 3 * k + 1] += g.x[k] * gh1; cam[12 + 3 * k + 2] += g.x[k] * gh3;
        }
        cam[21] += gh0; cam[22] += gh1; cam[23] += gh3;
    }
    // ---- rotation matrix -> normalised quaternion -> raw quaternion
    {
        const float r = g.qn[0], x = g.qn[1], y = g.qn[2], z = g.qn[3];
        float gq[4];
        gq[0] = 2.f * (-z * gR[1][0] + y * gR[2][0] + z * gR[0][1] - x * gR[2][1] - y * gR[0][2] + x * gR[1][2]);
        gq[1] = 2.f * (y * gR[1][0] + z * gR[2][0] + y * gR[0][1] - r * gR[2][1] + z * gR[0][2] + r * gR[1][2]) - 4.f * x * (gR[1][1] + gR[2][2]);
        gq[2] = 2.f * (x * gR[1][0] + r * gR[2][0] + x * gR[0][1] + z * gR[2][1] - r * gR[0][2] + z * gR[1][2]) - 4.f * y * (gR[0][0] + gR[2][2]);
        gq[3] = 2.f * (-r * gR[1][0] + x * gR[2][0] + r * gR[0][1] + y * gR[2][1] + x * gR[0][2] + y * gR[1][2]) - 4.f * z * (gR[0][0] + gR[1][1]);
        const float dot = r * gq[0] + x * gq[1] + y * gq[2] + z * gq[3];
        const float il = 1.0f / g.qlen;
        go.rotation[0] = (gq[0] - r * dot) * il; go.rotation[1] = (gq[1] - x * dot) * il;
        go.rotation[2] = (gq[2] - y * dot) * il; go.rotation[3] = (gq[3] - z * dot) * il;
    }
    // ---- scale activation
#pragma unroll
    for (int k = 0; k < 3; k++) go.scaling[k] = (A.scale_act == 1) ? ds[k] * g.s[k] : ds[k] * A.mod;
    go.xyz[0] = dx[0]; go.xyz[1] = dx[1]; go.xyz[2] = dx[2];
    if constexpr (STRAND) {
        // q = (1 + b.x, 0, -b.z, b.y): dL/db from the raw-quaternion gradient, through b = d / max(|d|, 1e-12);
        // scale 0 = |d| / 2 adds 0.5 dL/ds0 d / |d|.  The thickness is not a parameter: its gradient is dropped.
        const float n0 = A.dirs[3 * (size_t)i], n1 = A.dirs[3 * (size_t)i + 1], n2 = A.dirs[3 * (size_t)i + 2];
        const float dl = fmaxf(sqrtf(n0 * n0 + n1 * n1 + n2 * n2), 1e-12f);
        const float b0 = n0 / dl, b1 = n1 / dl, b2 = n2 / dl;
        const float gb0 = go.rotation[0], gb1 = go.rotation[3], gb2 = -go.rotation[2];
        const float dot = b0 * gb0 + b1 * gb1 + b2 * gb2;
        const float hs = 0.5f * go.scaling[0];
        go.dirs[0] += (gb0 - b0 * dot) / dl + hs * b0;
        go.dirs[1] += (gb1 - b1 * dot) / dl + hs * b1;
        go.dirs[2] += (gb2 - b2 * dot) / dl + hs * b2;
#pragma unroll
        for (int k = 0; k < 3; k++) go.scaling[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) go.rotation[k] = 0.f;
    }
}
