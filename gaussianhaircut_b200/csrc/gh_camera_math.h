// The trainable-camera model of the reference (src/scene/cameras.py:95-152, BARF parameterisation), written once for
// device AND host: the kernels of gh_camera.cu call these functions, and tests/host_harness/camera_host.cpp compiles
// this very header with g++ so that it is checked against a float64 restatement and float64 autograd
// (tests/test_cameras_cpu.py).  The host build is test infrastructure only; libgh_raster.so contains no CPU path.
//
// Camera i: base state `base` = C (the float32 _colmap_transform, 16, row-major), FoVx, FoVy (GH_CAM_BASE floats) and
// trained row r = [w(3), u(3), f(2)] (_rotation_res, _translation_res, _fov_res; f = 0 without trainable intrinsics).
//   Res[:3] = lie.se3_to_SE3(cat(w, u)), Res[3] = (0, 0, 0, 1)      (utils/camera_opt_utils.py:84-141)
//   viewmatrix = (C @ Res)^T
//   projmatrix = viewmatrix @ getProjectionMatrix(0.01, 100, FoVx + f0, FoVy + f1)^T   (utils/graphics_utils.py:51)
//   campos     = inverse(viewmatrix)[3, :3]
//   tan_fov    = tan((FoV + f) / 2), per axis
// The forward follows the reference's float32 operation order where that is cheap: the three 11-term Taylor sums term
// by term (x**2i, then * (1 / float(denominator)) -- torch's `tensor / python_float` on CUDA), `(B * wx) @ wx`, and the
// top / right / reciprocal sequence of getProjectionMatrix.  The 4x4 inverse is computed in double and rounded once.
// The backward (the chain of all of the above) runs in double from the float32 inputs and rounds each of the 8
// gradients once; the series are differentiated in s = |w|^2, so w = 0 (the reference's initial value) is regular.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define GH_CAM_HD __host__ __device__ __forceinline__
#else
#define GH_CAM_HD static inline
#endif

#define GH_CAM_BASE 18        // floats per camera of the base table: C (16, row-major), FoVx, FoVy
#define GH_CAM_ROW 8          // floats per camera of the trained table: w (3), u (3), f (2)
#define GH_CAM_DCAMERA 37     // dL/dviewmatrix (16), dL/dprojmatrix (16), dL/dcampos (3), dL/dtan_fov (2)
#define GH_CAM_TERMS 11       // Taylor terms of taylor_A / taylor_B / taylor_C (nth = 10)

// The denominators of taylor_A (sin x / x), taylor_B ((1 - cos x) / x^2) and taylor_C ((x - sin x) / x^3), accumulated
// in double like the reference's Python floats: k = 0, 1, 2.
GH_CAM_HD double gh_cam_denominator(int k, int i) {
    double d = 1.0;
    for (int j = 0; j <= i; j++) {
        if (k == 0) { if (j > 0) d *= (double)(2 * j) * (double)(2 * j + 1); }
        else if (k == 1) d *= (double)(2 * j + 1) * (double)(2 * j + 2);
        else d *= (double)(2 * j + 2) * (double)(2 * j + 3);
    }
    return d;
}

// torch's float32 `x ** e` on CUDA for the even exponents of the series: 0 -> 1, 2 -> x * x, otherwise powf
GH_CAM_HD float gh_cam_pow(float x, int e) {
    return e == 0 ? 1.0f : (e == 2 ? x * x : powf(x, (float)e));
}

// taylor_{A,B,C}(theta) in float32, term by term
GH_CAM_HD float gh_cam_taylor_f(int k, float theta) {
    float ans = 0.0f;
    for (int i = 0; i < GH_CAM_TERMS; i++) {
        const float p = gh_cam_pow(theta, 2 * i);
        const float inv = 1.0f / (float)gh_cam_denominator(k, i);
        ans = ans + ((i & 1) ? -p : p) * inv;
    }
    return ans;
}

// the same series as a function of s = theta^2, in double, and its derivative d/ds
GH_CAM_HD void gh_cam_taylor_d(int k, double s, double& val, double& dval) {
    val = 0.0; dval = 0.0;
    double sp = 1.0;          // s^i
    double spm = 0.0;         // i * s^(i-1)
    for (int i = 0; i < GH_CAM_TERMS; i++) {
        const double d = gh_cam_denominator(k, i);
        const double sg = (i & 1) ? -1.0 : 1.0;
        val += sg * sp / d;
        dval += sg * spm / d;
        spm = (double)(i + 1) * sp;
        sp *= s;
    }
}

// 4x4 inverse (row-major) by cofactors, in double; returns the determinant
GH_CAM_HD double gh_cam_inverse4(const double a[16], double b[16]) {
    const double s0 = a[0] * a[5] - a[4] * a[1], s1 = a[0] * a[6] - a[4] * a[2], s2 = a[0] * a[7] - a[4] * a[3];
    const double s3 = a[1] * a[6] - a[5] * a[2], s4 = a[1] * a[7] - a[5] * a[3], s5 = a[2] * a[7] - a[6] * a[3];
    const double c5 = a[10] * a[15] - a[14] * a[11], c4 = a[9] * a[15] - a[13] * a[11], c3 = a[9] * a[14] - a[13] * a[10];
    const double c2 = a[8] * a[15] - a[12] * a[11], c1 = a[8] * a[14] - a[12] * a[10], c0 = a[8] * a[13] - a[12] * a[9];
    const double det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
    const double r = 1.0 / det;
    b[0] = (a[5] * c5 - a[6] * c4 + a[7] * c3) * r;
    b[1] = (-a[1] * c5 + a[2] * c4 - a[3] * c3) * r;
    b[2] = (a[13] * s5 - a[14] * s4 + a[15] * s3) * r;
    b[3] = (-a[9] * s5 + a[10] * s4 - a[11] * s3) * r;
    b[4] = (-a[4] * c5 + a[6] * c2 - a[7] * c1) * r;
    b[5] = (a[0] * c5 - a[2] * c2 + a[3] * c1) * r;
    b[6] = (-a[12] * s5 + a[14] * s2 - a[15] * s1) * r;
    b[7] = (a[8] * s5 - a[10] * s2 + a[11] * s1) * r;
    b[8] = (a[4] * c4 - a[5] * c2 + a[7] * c0) * r;
    b[9] = (-a[0] * c4 + a[1] * c2 - a[3] * c0) * r;
    b[10] = (a[12] * s4 - a[13] * s2 + a[15] * s0) * r;
    b[11] = (-a[8] * s4 + a[9] * s2 - a[11] * s0) * r;
    b[12] = (-a[4] * c3 + a[5] * c1 - a[6] * c0) * r;
    b[13] = (a[0] * c3 - a[1] * c1 + a[2] * c0) * r;
    b[14] = (-a[12] * s3 + a[13] * s1 - a[14] * s0) * r;
    b[15] = (a[8] * s3 - a[9] * s1 + a[10] * s0) * r;
    return det;
}

// the constant entries of getProjectionMatrix(znear = 0.01, zfar = 100), computed in double and stored as float32
#define GH_CAM_P22 ((float)(100.0 / (100.0 - 0.01)))
#define GH_CAM_P23 ((float)(-(100.0 * 0.01) / (100.0 - 0.01)))

// Forward: the four outputs of the reference Camera, row-major like the torch tensors.
GH_CAM_HD void gh_camera_forward_math(const float* base, const float* r, float view[16], float proj[16],
                                      float campos[3], float tan_fov[2]) {
    const float w0 = r[0], w1 = r[1], w2 = r[2];
    // skew_symmetric(w) and its square (B * wx) @ wx, (C * wx) @ wx
    const float K[9] = {0.0f, -w2, w1, w2, 0.0f, -w0, -w1, w0, 0.0f};
    const float theta = sqrtf(w0 * w0 + w1 * w1 + w2 * w2);
    const float A = gh_cam_taylor_f(0, theta), B = gh_cam_taylor_f(1, theta), Cc = gh_cam_taylor_f(2, theta);
    float R[9], V[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            float bk = 0.0f, ck = 0.0f;
            for (int k = 0; k < 3; k++) { bk = bk + (B * K[i * 3 + k]) * K[k * 3 + j]; ck = ck + (Cc * K[i * 3 + k]) * K[k * 3 + j]; }
            const float I = (i == j) ? 1.0f : 0.0f;
            R[i * 3 + j] = (I + A * K[i * 3 + j]) + bk;
            V[i * 3 + j] = (I + B * K[i * 3 + j]) + ck;
        }
    float Res[16];
    for (int i = 0; i < 3; i++) {
        float t = 0.0f;
        for (int k = 0; k < 3; k++) t = t + V[i * 3 + k] * r[3 + k];
        Res[i * 4 + 0] = R[i * 3 + 0]; Res[i * 4 + 1] = R[i * 3 + 1]; Res[i * 4 + 2] = R[i * 3 + 2]; Res[i * 4 + 3] = t;
    }
    Res[12] = 0.0f; Res[13] = 0.0f; Res[14] = 0.0f; Res[15] = 1.0f;
    // viewmatrix = (C @ Res)^T
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            float m = 0.0f;
            for (int k = 0; k < 4; k++) m = m + base[i * 4 + k] * Res[k * 4 + j];
            view[j * 4 + i] = m;
        }
    // getProjectionMatrix(..., FoVx + f0, FoVy + f1).T
    const float tx = tanf((base[16] + r[6]) * 0.5f), ty = tanf((base[17] + r[7]) * 0.5f);
    const float top = ty * 0.01f, right = tx * 0.01f;
    float PT[16];
    for (int i = 0; i < 16; i++) PT[i] = 0.0f;
    PT[0] = (1.0f / (right - (-right))) * 0.02f;                 // P[0,0] = 2 znear / (right - left)
    PT[5] = (1.0f / (top - (-top))) * 0.02f;                     // P[1,1]
    PT[8] = (right + (-right)) / (right - (-right));             // P[0,2] (= 0)
    PT[9] = (top + (-top)) / (top - (-top));                     // P[1,2] (= 0)
    PT[11] = 1.0f;                                               // P[3,2] = z_sign
    PT[10] = GH_CAM_P22;                                         // P[2,2]
    PT[14] = GH_CAM_P23;                                         // P[2,3]
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            float m = 0.0f;
            for (int k = 0; k < 4; k++) m = m + view[i * 4 + k] * PT[k * 4 + j];
            proj[i * 4 + j] = m;
        }
    double Wd[16], Inv[16];
    for (int i = 0; i < 16; i++) Wd[i] = (double)view[i];
    gh_cam_inverse4(Wd, Inv);
    campos[0] = (float)Inv[12]; campos[1] = (float)Inv[13]; campos[2] = (float)Inv[14];
    tan_fov[0] = tx; tan_fov[1] = ty;
}

// Backward: g = the 37 upstream gradients (d_camera layout) -> dr[8] = dL/d[w, u, f] (dr[6..7] = 0 without intrinsics).
GH_CAM_HD void gh_camera_backward_math(const float* base, const float* r, const float* g, int intrinsics, float dr[8]) {
    const double w[3] = {r[0], r[1], r[2]}, u[3] = {r[3], r[4], r[5]};
    const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
    double K2[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) K2[i * 3 + j] = K[i * 3] * K[j] + K[i * 3 + 1] * K[3 + j] + K[i * 3 + 2] * K[6 + j];
    const double s = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    double A, dA_ds, B, dB_ds, Cc, dC_ds;
    gh_cam_taylor_d(0, s, A, dA_ds);
    gh_cam_taylor_d(1, s, B, dB_ds);
    gh_cam_taylor_d(2, s, Cc, dC_ds);
    double Res[16];
    for (int i = 0; i < 3; i++) {
        double t = 0.0;
        for (int j = 0; j < 3; j++) {
            const double I = (i == j) ? 1.0 : 0.0;
            Res[i * 4 + j] = I + A * K[i * 3 + j] + B * K2[i * 3 + j];
            t += (I + B * K[i * 3 + j] + Cc * K2[i * 3 + j]) * u[j];
        }
        Res[i * 4 + 3] = t;
    }
    Res[12] = 0.0; Res[13] = 0.0; Res[14] = 0.0; Res[15] = 1.0;
    double W[16];                                     // (C @ Res)^T
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double m = 0.0;
            for (int k = 0; k < 4; k++) m += (double)base[i * 4 + k] * Res[k * 4 + j];
            W[j * 4 + i] = m;
        }
    const double tx = tan(((double)base[16] + r[6]) * 0.5), ty = tan(((double)base[17] + r[7]) * 0.5);
    // dL/dW: the direct term, projmatrix = W @ PT (PT[0] = 1/tx, PT[5] = 1/ty, PT[10], PT[11] = 1, PT[14]) and campos
    double dW[16];
    const float* gF = g + 16;
    const double PT0 = 1.0 / tx, PT5 = 1.0 / ty, PT10 = (double)GH_CAM_P22, PT14 = (double)GH_CAM_P23;
    for (int i = 0; i < 4; i++) {
        // dW[i][k] = g_view[i][k] + sum_j gF[i][j] PT[k][j]
        dW[i * 4 + 0] = (double)g[i * 4 + 0] + (double)gF[i * 4 + 0] * PT0;
        dW[i * 4 + 1] = (double)g[i * 4 + 1] + (double)gF[i * 4 + 1] * PT5;
        dW[i * 4 + 2] = (double)g[i * 4 + 2] + (double)gF[i * 4 + 2] * PT10 + (double)gF[i * 4 + 3];
        dW[i * 4 + 3] = (double)g[i * 4 + 3] + (double)gF[i * 4 + 2] * PT14;
    }
    // dL/dPT[0][0] and dL/dPT[1][1] = (W^T gF)[0][0], (W^T gF)[1][1]: the only entries of PT that depend on tan fov
    double dPT0 = 0.0, dPT5 = 0.0;
    for (int i = 0; i < 4; i++) { dPT0 += W[i * 4 + 0] * (double)gF[i * 4 + 0]; dPT5 += W[i * 4 + 1] * (double)gF[i * 4 + 1]; }
    // campos = inverse(W)[3, :3]: dW -= Inv^T G Inv^T with G[3][j] = g_campos[j]
    double Inv[16];
    gh_cam_inverse4(W, Inv);
    {
        const float* gc = g + 32;
        // Inv^T G Inv^T: (Inv^T)[a][3] * gc[j] * (Inv^T)[j][b] = Inv[3][a] * gc[j] * Inv[b][j]
        for (int b = 0; b < 4; b++) {
            const double q = (double)gc[0] * Inv[b * 4 + 0] + (double)gc[1] * Inv[b * 4 + 1] + (double)gc[2] * Inv[b * 4 + 2];
            for (int a = 0; a < 4; a++) dW[a * 4 + b] -= Inv[12 + a] * q;
        }
    }
    // M = C @ Res = W^T: dM = dW^T; dRes = C^T dM (rows 0..2)
    double dRes[12];
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 4; b++) {
            double m = 0.0;
            for (int k = 0; k < 4; k++) m += (double)base[k * 4 + a] * dW[b * 4 + k];   // C[k][a] * dM[k][b], dM[k][b] = dW[b][k]
            dRes[a * 4 + b] = m;
        }
    // t = V u: du = V^T dt, dV = dt u^T; R = I + A K + B K^2, V = I + B K + C K^2
    double du[3] = {0.0, 0.0, 0.0}, dV[9], dR[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            const double I = (i == j) ? 1.0 : 0.0;
            const double Vij = I + B * K[i * 3 + j] + Cc * K2[i * 3 + j];
            du[j] += Vij * dRes[i * 4 + 3];
            dV[i * 3 + j] = dRes[i * 4 + 3] * u[j];
            dR[i * 3 + j] = dRes[i * 4 + j];
        }
    double gA = 0.0, gB = 0.0, gC = 0.0;
    for (int i = 0; i < 9; i++) { gA += dR[i] * K[i]; gB += dR[i] * K2[i] + dV[i] * K[i]; gC += dV[i] * K2[i]; }
    // dK = A dR + B dV + (B dR + C dV) K^T + K^T (B dR + C dV)
    double G2[9], dK[9];
    for (int i = 0; i < 9; i++) G2[i] = B * dR[i] + Cc * dV[i];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double m = A * dR[i * 3 + j] + B * dV[i * 3 + j];
            for (int k = 0; k < 3; k++) m += G2[i * 3 + k] * K[j * 3 + k] + K[k * 3 + i] * G2[k * 3 + j];
            dK[i * 3 + j] = m;
        }
    const double ds2 = 2.0 * (gA * dA_ds + gB * dB_ds + gC * dC_ds);
    dr[0] = (float)(dK[7] - dK[5] + ds2 * w[0]);
    dr[1] = (float)(dK[2] - dK[6] + ds2 * w[1]);
    dr[2] = (float)(dK[3] - dK[1] + ds2 * w[2]);
    dr[3] = (float)du[0]; dr[4] = (float)du[1]; dr[5] = (float)du[2];
    if (intrinsics) {
        // PT[0] = 1 / tan_x, PT[5] = 1 / tan_y; d tan / d fov = (1 + tan^2) / 2
        const double dtx = (double)g[35] - dPT0 / (tx * tx), dty = (double)g[36] - dPT5 / (ty * ty);
        dr[6] = (float)(dtx * 0.5 * (1.0 + tx * tx));
        dr[7] = (float)(dty * 0.5 * (1.0 + ty * ty));
    } else {
        dr[6] = 0.0f; dr[7] = 0.0f;
    }
}
