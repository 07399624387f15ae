// Per-triangle arithmetic of the mesh signed-distance kernels (gh_sdf.cu) and the mesh rasterizer (gh_mesh_raster.cu),
// written once for device AND host: the CUDA kernels call these functions, and tests/host_harness/sdf_host.cpp and
// mesh_raster_host.cpp compile this very header with g++ so that the per-pair results are checked against the float64
// oracles (tests/_sdf64.py, tests/_meshraster64.py) on a machine without a GPU.  The host builds are test
// infrastructure only; libgh_raster.so contains no CPU path.  DESIGN §23, §24.
//
// The rasterizer's functions (gh_raster_*) round every operation on their own, FMAs included (GH_MESH_FMA), so the
// host build with -ffp-contract=off reproduces the device's coverage decisions and depth bits exactly.
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
#define GH_MESH_DIV(a, b) __fdiv_rn((a), (b))
#define GH_MESH_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#else
#define GH_MESH_SUB(a, b) ((a) - (b))
#define GH_MESH_ADD(a, b) ((a) + (b))
#define GH_MESH_MUL(a, b) ((a) * (b))
#define GH_MESH_RCP(a) (1.f / (a))
#define GH_MESH_DIV(a, b) ((a) / (b))
#define GH_MESH_FMA(a, b, c) fmaf((a), (b), (c))
#endif

// The face-index rule of every mesh kernel: a face reads its vertices only when all three indices lie in [0, V).
GH_MESH_HD bool gh_mesh_face_in_range(int i0, int i1, int i2, int V)
{
    return i0 >= 0 && i0 < V && i1 >= 0 && i1 < V && i2 >= 0 && i2 < V;
}

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

// ------------------------------------------------------------------------------------------------ mesh rasterizer
// One (view, face) as the raster kernel reads it: 80 bytes.  x, y: the screen vertices; ex[k], ey[k] = vertex k2 -
// vertex k1 with (k1, k2) = (k + 1, k + 2) mod 3, the edge opposite vertex k; iz[k] = 1 / z_k (view-space z); area =
// the signed doubled screen area; the pixel box [i0, i0 + ni) x [j0, j0 + nj), empty (ni = nj = 0) for a skipped face.
struct alignas(16) GhRasterFace {
    float x[3], y[3], ex[3], ey[3], iz[3], area;
    int j0, i0, nj, ni;
};

#define GH_RASTER_DRAWN 0
#define GH_RASTER_SKIPPED 1     // a non-finite vertex or projection, zero area, or the whole face at z <= 0
#define GH_RASTER_NEAR 2        // some vertices at z <= 0, others in front: skipped (pytorch3d would clip it)

// cam = fx, fy, cx, cy; R row-major 3x3 (world to camera); t (3).  a, b, c: the world vertices.  Every operation
// rounded on its own, in this order:
//   x_cam = fma(R0, X, fma(R1, Y, fma(R2, Z, t0)))          (y_cam, z_cam likewise with R3..5, t1 and R6..8, t2)
//   u = fma(fx, x_cam / z_cam, cx),  v = fma(fy, y_cam / z_cam, cy),  iz = 1 / z_cam
//   ex[k] = x[k2] - x[k1],  ey[k] = y[k2] - y[k1]
//   area = fma(x1 - x0, y2 - y0, -((y1 - y0) * (x2 - x0)))
//   box: columns [max(floor(min u) - 1, 0), min(ceil(max u), W - 1)], rows likewise -- it holds every pixel centre of
//        the triangle with a pixel to spare, so the box never decides coverage where the edge tests are near a tie.
GH_MESH_HD int gh_raster_setup(const float* cam, const float* R, const float* t, const float* a, const float* b,
                               const float* c, int H, int W, GhRasterFace& r)
{
    r.j0 = r.i0 = r.nj = r.ni = 0;
    const float* P[3] = {a, b, c};
    float zc[3];
    bool finite = true;
    int n_front = 0;
    for (int k = 0; k < 3; k++) {
        const float X = P[k][0], Y = P[k][1], Z = P[k][2];
        finite = finite && isfinite(X) && isfinite(Y) && isfinite(Z);
        const float xc = GH_MESH_FMA(R[0], X, GH_MESH_FMA(R[1], Y, GH_MESH_FMA(R[2], Z, t[0])));
        const float yc = GH_MESH_FMA(R[3], X, GH_MESH_FMA(R[4], Y, GH_MESH_FMA(R[5], Z, t[1])));
        zc[k] = GH_MESH_FMA(R[6], X, GH_MESH_FMA(R[7], Y, GH_MESH_FMA(R[8], Z, t[2])));
        n_front += zc[k] > 0.f;
        r.x[k] = GH_MESH_FMA(cam[0], GH_MESH_DIV(xc, zc[k]), cam[2]);
        r.y[k] = GH_MESH_FMA(cam[1], GH_MESH_DIV(yc, zc[k]), cam[3]);
        r.iz[k] = GH_MESH_RCP(zc[k]);
    }
    if (!finite) return GH_RASTER_SKIPPED;
    if (n_front < 3) return n_front == 0 ? GH_RASTER_SKIPPED : GH_RASTER_NEAR;
    for (int k = 0; k < 3; k++) {
        const int k1 = k == 2 ? 0 : k + 1, k2 = k == 0 ? 2 : k - 1;
        r.ex[k] = GH_MESH_SUB(r.x[k2], r.x[k1]);
        r.ey[k] = GH_MESH_SUB(r.y[k2], r.y[k1]);
    }
    r.area = GH_MESH_FMA(GH_MESH_SUB(r.x[1], r.x[0]), GH_MESH_SUB(r.y[2], r.y[0]),
                         -GH_MESH_MUL(GH_MESH_SUB(r.y[1], r.y[0]), GH_MESH_SUB(r.x[2], r.x[0])));
    bool ok = r.area != 0.f && isfinite(r.area);
    for (int k = 0; k < 3; k++) ok = ok && isfinite(r.x[k]) && isfinite(r.y[k]);
    if (!ok) return GH_RASTER_SKIPPED;
    const float j_lo = fmaxf(floorf(fminf(r.x[0], fminf(r.x[1], r.x[2]))) - 1.f, 0.f);
    const float j_hi = fminf(ceilf(fmaxf(r.x[0], fmaxf(r.x[1], r.x[2]))), (float)(W - 1));
    const float i_lo = fmaxf(floorf(fminf(r.y[0], fminf(r.y[1], r.y[2]))) - 1.f, 0.f);
    const float i_hi = fminf(ceilf(fmaxf(r.y[0], fmaxf(r.y[1], r.y[2]))), (float)(H - 1));
    if (j_lo <= j_hi && i_lo <= i_hi) {
        r.j0 = (int)j_lo;
        r.i0 = (int)i_lo;
        r.nj = (int)j_hi - r.j0 + 1;
        r.ni = (int)i_hi - r.i0 + 1;
    }
    return GH_RASTER_DRAWN;
}

// The three edge functions at the centre (j + 0.5, i + 0.5) of pixel (i, j):
//   w[k] = fma(ex[k], py - y[k1], -(ey[k] * (px - x[k1]))),  w[k] / area = the screen barycentric of vertex k.
GH_MESH_HD void gh_raster_edges(const GhRasterFace& r, int i, int j, float* w)
{
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    for (int k = 0; k < 3; k++) {
        const int k1 = k == 2 ? 0 : k + 1;
        w[k] = GH_MESH_FMA(r.ex[k], GH_MESH_SUB(py, r.y[k1]), -GH_MESH_MUL(r.ey[k], GH_MESH_SUB(px, r.x[k1])));
    }
}

// Coverage of pixel (i, j): every barycentric strictly positive (each w[k] strictly of the area's sign), so a centre
// on an edge is not covered and back faces are drawn.  When covered, z = area / fma(w0, iz0, fma(w1, iz1, w2 * iz2)):
// the perspective-correct view-space z, 1 / z the barycentric blend of the vertices' 1 / z.
GH_MESH_HD bool gh_raster_pixel(const GhRasterFace& r, int i, int j, float& z)
{
    float w[3];
    gh_raster_edges(r, i, j, w);
    const bool in = r.area > 0.f ? (w[0] > 0.f && w[1] > 0.f && w[2] > 0.f) : (w[0] < 0.f && w[1] < 0.f && w[2] < 0.f);
    z = GH_MESH_DIV(r.area, GH_MESH_FMA(w[0], r.iz[0], GH_MESH_FMA(w[1], r.iz[1], GH_MESH_MUL(w[2], r.iz[2]))));
    return in;
}
