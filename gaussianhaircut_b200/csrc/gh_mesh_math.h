// Per-triangle arithmetic of the mesh signed-distance kernels (gh_sdf.cu), written once for device AND host: the CUDA
// kernels call these functions, and tests/host_harness/sdf_host.cpp compiles this very header with g++ so that the
// per-pair distance and solid angle are checked against the float64 oracle (tests/_sdf64.py) on a machine without a
// GPU.  The host build is test infrastructure only; libgh_raster.so contains no CPU path.  DESIGN §23.
//
// gh_sdf_record rounds every operation on its own (intrinsics on the device, -ffp-contract=off on the host), so the
// record is the same bits wherever it is built, and the oracle can restate it in numpy float32.  gh_sdf_pair leaves
// contraction to the compiler: its error bound (tests/_sdf64.py) counts one rounding per multiply and per add, which
// an FMA's single rounding satisfies.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define GH_MESH_HD __host__ __device__ __forceinline__
#else
#define GH_MESH_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define GH_MESH_SUB(a, b) __fsub_rn((a), (b))
#define GH_MESH_ADD(a, b) __fadd_rn((a), (b))
#define GH_MESH_MUL(a, b) __fmul_rn((a), (b))
#define GH_MESH_RCP(a) __fdiv_rn(1.f, (a))
#else
#define GH_MESH_SUB(a, b) ((a) - (b))
#define GH_MESH_ADD(a, b) ((a) + (b))
#define GH_MESH_MUL(a, b) ((a) * (b))
#define GH_MESH_RCP(a) (1.f / (a))
#endif

// One face as the query loop reads it: 7 x 16 bytes.
//   v[0..2]  a     v[3]  inv_nn  = 1 / |n|^2, or 0 when that is not a positive finite number (the triangle is
//                                  degenerate: only its edges count)
//   v[4..6]  b     v[7]  inv_ab  = 1 / |ab|^2, or 0 likewise (the edge is a point: t = 0)
//   v[8..10] c     v[11] inv_bc
//   v[12..14] ab = b - a,  v[15] inv_ca
//   v[16..18] bc = c - b,  v[20..22] ca = a - c,  v[24..26] n = ca x ab (= ab x ac),  v[19], v[23], v[27] = 0
struct alignas(16) GhSdfRecord { float v[28]; };

GH_MESH_HD float gh_mesh_safe_rcp(float x)
{
    const float r = GH_MESH_RCP(x);
    return (r > 0.f && r < INFINITY) ? r : 0.f;
}

GH_MESH_HD float gh_mesh_norm2_rn(float x, float y, float z)
{
    return GH_MESH_ADD(GH_MESH_ADD(GH_MESH_MUL(x, x), GH_MESH_MUL(y, y)), GH_MESH_MUL(z, z));
}

// The record of triangle (a, b, c); every operation rounded on its own.
GH_MESH_HD void gh_sdf_record(const float* a, const float* b, const float* c, GhSdfRecord& r)
{
    float ab[3], bc[3], ca[3];
    for (int k = 0; k < 3; k++) {
        ab[k] = GH_MESH_SUB(b[k], a[k]);
        bc[k] = GH_MESH_SUB(c[k], b[k]);
        ca[k] = GH_MESH_SUB(a[k], c[k]);
    }
    const float n[3] = {GH_MESH_SUB(GH_MESH_MUL(ca[1], ab[2]), GH_MESH_MUL(ca[2], ab[1])),
                        GH_MESH_SUB(GH_MESH_MUL(ca[2], ab[0]), GH_MESH_MUL(ca[0], ab[2])),
                        GH_MESH_SUB(GH_MESH_MUL(ca[0], ab[1]), GH_MESH_MUL(ca[1], ab[0]))};
    for (int k = 0; k < 3; k++) {
        r.v[k] = a[k];
        r.v[4 + k] = b[k];
        r.v[8 + k] = c[k];
        r.v[12 + k] = ab[k];
        r.v[16 + k] = bc[k];
        r.v[20 + k] = ca[k];
        r.v[24 + k] = n[k];
    }
    r.v[3] = gh_mesh_safe_rcp(gh_mesh_norm2_rn(n[0], n[1], n[2]));
    r.v[7] = gh_mesh_safe_rcp(gh_mesh_norm2_rn(ab[0], ab[1], ab[2]));
    r.v[11] = gh_mesh_safe_rcp(gh_mesh_norm2_rn(bc[0], bc[1], bc[2]));
    r.v[15] = gh_mesh_safe_rcp(gh_mesh_norm2_rn(ca[0], ca[1], ca[2]));
    r.v[19] = r.v[23] = r.v[27] = 0.f;
}

GH_MESH_HD float gh_mesh_dot(float ax, float ay, float az, float bx, float by, float bz)
{
    return ax * bx + ay * by + az * bz;
}

// Squared distance from the origin to the segment {X + t E : 0 <= t <= 1}, X = (x, y, z) = vertex - p; inv = the
// record's 1 / |E|^2 (0: the segment is the point X).
GH_MESH_HD float gh_mesh_seg_d2(float x, float y, float z, float ex, float ey, float ez, float inv)
{
    const float t = fminf(fmaxf(-gh_mesh_dot(x, y, z, ex, ey, ez) * inv, 0.f), 1.f);
    const float qx = x + t * ex, qy = y + t * ey, qz = z + t * ez;
    return gh_mesh_dot(qx, qy, qz, qx, qy, qz);
}

// One (point, face) pair: d2 = the squared distance from p to the triangle, omega = its signed solid angle seen from p.
//   distance: Ericson's Voronoi regions of a triangle (Real-Time Collision Detection, 5.1.5) evaluated as the smallest
//     of the three edge-segment distances (the vertex and edge regions: t clamped to [0, 1]) and, when p's projection
//     lies in the face region (B x C, C x A and A x B all on n's side) of a non-degenerate face, the plane distance
//     (A . n)^2 / |n|^2.  A degenerate face (inv_nn = 0) is its edges, a zero-length edge its vertex.
//   solid angle: 2 atan2(A . (B x C), |A||B||C| + (A.B)|C| + (A.C)|B| + (B.C)|A|) (Van Oosterom-Strackee).
GH_MESH_HD void gh_sdf_pair(const GhSdfRecord& r, float px, float py, float pz, float& d2, float& omega)
{
    const float Ax = r.v[0] - px, Ay = r.v[1] - py, Az = r.v[2] - pz;
    const float Bx = r.v[4] - px, By = r.v[5] - py, Bz = r.v[6] - pz;
    const float Cx = r.v[8] - px, Cy = r.v[9] - py, Cz = r.v[10] - pz;
    const float bcx = By * Cz - Bz * Cy, bcy = Bz * Cx - Bx * Cz, bcz = Bx * Cy - By * Cx;      // B x C
    const float cax = Cy * Az - Cz * Ay, cay = Cz * Ax - Cx * Az, caz = Cx * Ay - Cy * Ax;      // C x A
    const float abx = Ay * Bz - Az * By, aby = Az * Bx - Ax * Bz, abz = Ax * By - Ay * Bx;      // A x B
    const float la = sqrtf(gh_mesh_dot(Ax, Ay, Az, Ax, Ay, Az));
    const float lb = sqrtf(gh_mesh_dot(Bx, By, Bz, Bx, By, Bz));
    const float lc = sqrtf(gh_mesh_dot(Cx, Cy, Cz, Cx, Cy, Cz));
    const float num = gh_mesh_dot(Ax, Ay, Az, bcx, bcy, bcz);
    const float den = la * lb * lc + gh_mesh_dot(Ax, Ay, Az, Bx, By, Bz) * lc + gh_mesh_dot(Ax, Ay, Az, Cx, Cy, Cz) * lb +
                      gh_mesh_dot(Bx, By, Bz, Cx, Cy, Cz) * la;
    omega = 2.f * atan2f(num, den);

    float m = gh_mesh_seg_d2(Ax, Ay, Az, r.v[12], r.v[13], r.v[14], r.v[7]);
    m = fminf(m, gh_mesh_seg_d2(Bx, By, Bz, r.v[16], r.v[17], r.v[18], r.v[11]));
    m = fminf(m, gh_mesh_seg_d2(Cx, Cy, Cz, r.v[20], r.v[21], r.v[22], r.v[15]));
    const float nx = r.v[24], ny = r.v[25], nz = r.v[26], inv_nn = r.v[3];
    const bool face = inv_nn > 0.f && gh_mesh_dot(bcx, bcy, bcz, nx, ny, nz) >= 0.f &&
                      gh_mesh_dot(cax, cay, caz, nx, ny, nz) >= 0.f && gh_mesh_dot(abx, aby, abz, nx, ny, nz) >= 0.f;
    const float s = gh_mesh_dot(Ax, Ay, Az, nx, ny, nz);
    d2 = face ? fminf(m, s * s * inv_nn) : m;
}
