/*
 * gh_oracle.c -- TEST INFRASTRUCTURE ONLY (Oracle-B).
 *
 * A plain-C, CPU restatement of the reference rasterizer's algorithm
 * (/root/reference/ext/diff_gaussian_rasterization_hair/cuda_rasterizer/{forward,backward,
 * rasterizer_impl}.cu, auxiliary.h).  It exists to CHECK the CUDA product; nothing on the product
 * path may include, link or call it (only tests/, __graft_entry__.smoke() and bench.py's baseline
 * leg do).  Every function names the reference lines it follows.
 *
 * Pinning.  The reference ships no tests or golden vectors for this path.  This restatement is
 * pinned against (a) tests/golden/ *.npz, outputs of the reference extension itself executed on a
 * GPU (tests/golden/make_golden.py), and (b) the reference authors' own PyTorch restatement of
 * stage 1 (src/scene/gaussian_model.py:143-337), see tests/test_oracle_cpu.py.
 *
 * Rounding.  Everything that feeds a decision of the reference (depth key bits, tile rectangle,
 * alpha and transmittance thresholds) is evaluated in float32 in the operation order nvcc + ptxas
 * emit for the reference sources with its default flags (read off the SASS of the reference build):
 * in `a*b + c*d (+ e*f)` the LEFT product is fused into the add (fmaf(a,b,c*d)); `a*b - c*d`
 * becomes fmaf(a,b,-(c*d)); `m*m - d` becomes fmaf(m,m,-d); `1.f/x` is a correctly rounded
 * reciprocal, sqrt/div are IEEE.  Compile with -ffp-contract=off so that only the fmaf()
 * written here contracts.  The one thing a CPU cannot reproduce bit for bit is CUDA's expf
 * (ex2.approx based, <= 2 ulp); exp is evaluated in double and rounded, so blended values agree to
 * ~1e-7 relative and a decision can flip only for a pair sitting within an ulp of a threshold.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NUM_CHANNELS 10 /* config.h:15 */
#define BLOCK_X 16      /* config.h:16 */
#define BLOCK_Y 16      /* config.h:17 */

#ifdef __cplusplus
extern "C" {
#endif

static inline float f_rcp(float x) { return 1.0f / x; }

/* float -> int like PTX cvt.rzi.s32.f32 (saturating, NaN -> 0); a C cast is UB out of range */
static inline int f2i_rz(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return 2147483647;
    if (v <= -2147483648.0f) return (-2147483647 - 1);
    return (int)v;
}
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* auxiliary.h:41-44 -- the literals are doubles, so this is FP64 arithmetic (PTX: add.f64, fma.rn.f64, mul.f64) */
static inline float ndc2Pix(float v, int S) {
    double t = (double)v + 1.0;
    t = fma(t, (double)S, -1.0);
    t = t * 0.5;
    return (float)t;
}

/* auxiliary.h:46-56 */
static inline void getRect(float px, float py, int max_radius, int gx, int gy, int* rmin, int* rmax) {
    const float rf = (float)max_radius;
    rmin[0] = imin(gx, imax(0, f2i_rz((px - rf) * 0.0625f)));
    rmin[1] = imin(gy, imax(0, f2i_rz((py - rf) * 0.0625f)));
    rmax[0] = imin(gx, imax(0, f2i_rz((((px + rf) + 16.0f) + -1.0f) * 0.0625f)));
    rmax[1] = imin(gy, imax(0, f2i_rz((((py + rf) + 16.0f) + -1.0f) * 0.0625f)));
}

/* auxiliary.h:58-77 : m[0]*x + m[4]*y + m[8]*z + m[12]  ->  m12 + fma(z, m8, fma(x, m0, y*m4)) */
static inline float xform_row(const float* m, int r, float x, float y, float z) {
    return m[12 + r] + fmaf(z, m[8 + r], fmaf(x, m[r], y * m[4 + r]));
}

/* forward.cu:118-152 (computeCov3D) with the glm product order of oracle/glm_shim */
static void computeCov3D(const float* scale, float mod, const float* rot, float* cov3D) {
    const float sx = mod * scale[0], sy = mod * scale[1], sz = mod * scale[2];
    const float r = rot[0], x = rot[1], y = rot[2], z = rot[3]; /* NOT normalised (forward.cu:127) */
    const float yy = y * y, zz = z * z, xz = x * z, rx = r * x, rz = r * z;
    const float yy_zz = yy + zz;
    const float xx_zz = fmaf(x, x, zz);
    const float xx_yy = fmaf(x, x, yy);
    float t;
    const float R00 = 1.0f - (yy_zz + yy_zz);
    t = fmaf(x, y, -rz); const float R01 = t + t; /* 2(xy - rz) */
    t = fmaf(r, y, xz);  const float R02 = t + t; /* 2(xz + ry) */
    t = fmaf(x, y, rz);  const float R10 = t + t; /* 2(xy + rz) */
    const float R11 = 1.0f - (xx_zz + xx_zz);
    t = fmaf(y, z, -rx); const float R12 = t + t; /* 2(yz - rx) */
    t = fmaf(-r, y, xz); const float R20 = t + t; /* 2(xz - ry) */
    t = fmaf(y, z, rx);  const float R21 = t + t; /* 2(yz + rx) */
    const float R22 = 1.0f - (xx_yy + xx_yy);
    /* M = S * R (glm, column-major): M[c][r] = s_r * R[c][r] */
    const float M00 = sx * R00, M01 = sy * R01, M02 = sz * R02;
    const float M10 = sx * R10, M11 = sy * R11, M12 = sz * R12;
    const float M20 = sx * R20, M21 = sy * R21, M22 = sz * R22;
    /* Sigma = transpose(M) * M, upper triangle (forward.cu:141-151) */
    cov3D[0] = fmaf(M02, M02, fmaf(M00, M00, M01 * M01));
    cov3D[1] = fmaf(M02, M12, fmaf(M00, M10, M01 * M11));
    cov3D[2] = fmaf(M02, M22, fmaf(M00, M20, M01 * M21));
    cov3D[3] = fmaf(M12, M12, fmaf(M10, M10, M11 * M11));
    cov3D[4] = fmaf(M12, M22, fmaf(M10, M20, M11 * M21));
    cov3D[5] = fmaf(M22, M22, fmaf(M20, M20, M21 * M21));
}

/* forward.cu:74-113 (computeCov2D): returns (cov[0][0]+0.3, cov[0][1], cov[1][1]+0.3) */
static void computeCov2D(const float* mean, float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                         const float* c3, const float* vm, float* cov) {
    const float tx0 = xform_row(vm, 0, mean[0], mean[1], mean[2]);
    const float ty0 = xform_row(vm, 1, mean[0], mean[1], mean[2]);
    const float tz = xform_row(vm, 2, mean[0], mean[1], mean[2]);
    const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
    const float txtz = tx0 / tz, tytz = ty0 / tz;
    const float tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    const float ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
    const float tz2 = tz * tz;
    const float J00 = focal_x / tz, J02 = -((focal_x * tx) / tz2);
    const float J11 = focal_y / tz, J12 = -((focal_y * ty) / tz2);
    /* T = W * J, W = mat3(vm[0],vm[4],vm[8], vm[1],vm[5],vm[9], vm[2],vm[6],vm[10]) */
    const float T00 = fmaf(vm[2], J02, vm[0] * J00);
    const float T01 = fmaf(vm[6], J02, vm[4] * J00);
    const float T02 = fmaf(vm[10], J02, vm[8] * J00);
    const float T10 = fmaf(vm[2], J12, vm[1] * J11);
    const float T11 = fmaf(vm[6], J12, vm[5] * J11);
    const float T12 = fmaf(vm[10], J12, vm[9] * J11);
    /* cov = transpose(T) * transpose(Vrk) * T, evaluated left to right */
    const float A00 = fmaf(T02, c3[2], fmaf(T00, c3[0], T01 * c3[1]));
    const float A01 = fmaf(T12, c3[2], fmaf(T10, c3[0], T11 * c3[1]));
    const float A10 = fmaf(T02, c3[4], fmaf(T00, c3[1], T01 * c3[3]));
    const float A11 = fmaf(T12, c3[4], fmaf(T10, c3[1], T11 * c3[3]));
    const float A20 = fmaf(T02, c3[5], fmaf(T00, c3[2], T01 * c3[4]));
    const float A21 = fmaf(T12, c3[5], fmaf(T10, c3[2], T11 * c3[4]));
    const float c00 = fmaf(T02, A20, fmaf(T00, A00, T01 * A10));
    const float c01 = fmaf(T02, A21, fmaf(T00, A01, T01 * A11));
    const float c11 = fmaf(T12, A21, fmaf(T10, A01, T11 * A11));
    cov[0] = c00 + 0.3f; /* low-pass, forward.cu:110-111 */
    cov[1] = c01;
    cov[2] = c11 + 0.3f;
}

/*
 * K1: preprocessCUDA forward (forward.cu:155-282) + in_frustum (auxiliary.h:139-164).
 * Optional inputs are NULL when absent.  Outputs (all length-P arrays, zero where the Gaussian is
 * dropped): radii, depths, means2D[2P] (pixel coords), conic_opacity[4P], cov3D[6P] (native mode
 * only, else untouched), tiles_touched.  Returns the number of points that failed the near cull
 * (the reference traps on the first one when `prefiltered` is set).
 */
int gho_preprocess(int P, int W, int H,
                   const float* means3D, const float* opacities,
                   const float* scales, float scale_modifier, const float* rotations,
                   const float* cov3D_precomp, const float* conic_precomp,
                   const float* viewmatrix, const float* projmatrix,
                   float tan_fovx, float tan_fovy,
                   int* radii, float* depths, float* means2D, float* conic_opacity, float* cov3D_out,
                   uint32_t* tiles_touched)
{
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const float focal_y = H / (2.0f * tan_fovy); /* rasterizer_impl.cu:224-225 */
    const float focal_x = W / (2.0f * tan_fovx);
    int culled = 0;
    for (int idx = 0; idx < P; idx++) {
        radii[idx] = 0; tiles_touched[idx] = 0; /* forward.cu:190-191 */
        depths[idx] = 0.f; means2D[2 * idx] = means2D[2 * idx + 1] = 0.f;
        conic_opacity[4 * idx] = conic_opacity[4 * idx + 1] = conic_opacity[4 * idx + 2] = conic_opacity[4 * idx + 3] = 0.f;
        const float* p = means3D + 3 * idx;
        const float zview = xform_row(viewmatrix, 2, p[0], p[1], p[2]);
        if (zview <= 0.2f) { culled++; continue; } /* auxiliary.h:154 */
        /* forward.cu:201-206: projection is always recomputed */
        const float hx = xform_row(projmatrix, 0, p[0], p[1], p[2]);
        const float hy = xform_row(projmatrix, 1, p[0], p[1], p[2]);
        const float hw = xform_row(projmatrix, 3, p[0], p[1], p[2]);
        const float p_w = f_rcp(hw + 0.0000001f);
        const float projx = hx * p_w, projy = hy * p_w;

        float covx, covz, det, conx, cony, conz;
        if (conic_precomp == NULL) {
            float c3buf[6];
            const float* c3;
            if (cov3D_precomp != NULL) {
                c3 = cov3D_precomp + 6 * idx;
            } else {
                computeCov3D(scales + 3 * idx, scale_modifier, rotations + 4 * idx, c3buf);
                c3 = c3buf;
                if (cov3D_out) memcpy(cov3D_out + 6 * idx, c3buf, sizeof(c3buf));
            }
            float cov[3];
            computeCov2D(p, focal_x, focal_y, tan_fovx, tan_fovy, c3, viewmatrix, cov);
            covx = cov[0]; covz = cov[2];
            det = fmaf(covx, covz, -(cov[1] * cov[1])); /* forward.cu:231; SASS: FMUL, FFMA */
            if (det == 0.0f) continue;
            const float det_inv = f_rcp(det);
            conx = covz * det_inv; cony = det_inv * (-cov[1]); conz = covx * det_inv;
        } else { /* forward.cu:238-248 */
            conx = conic_precomp[3 * idx]; cony = conic_precomp[3 * idx + 1]; conz = conic_precomp[3 * idx + 2];
            const float det_inv = fmaf(conx, conz, -(cony * cony));
            if (det_inv == 0.0f) continue;
            det = f_rcp(det_inv);
            covx = conz * det; covz = conx * det;
        }
        /* forward.cu:254-257 */
        const float mid = (covx + covz) * 0.5f;
        const float sq = sqrtf(fmaxf(fmaf(mid, mid, -det), 0.1f));
        const float lam = fmaxf(mid + sq, mid - sq);
        const float my_radius = ceilf(sqrtf(lam) * 3.0f);
        const float pix_x = ndc2Pix(projx, W), pix_y = ndc2Pix(projy, H);
        const int ri = f2i_rz(my_radius);
        int rmin[2], rmax[2];
        getRect(pix_x, pix_y, ri, gx, gy, rmin, rmax);
        if ((rmax[0] - rmin[0]) * (rmax[1] - rmin[1]) == 0) continue; /* forward.cu:261-262 */
        depths[idx] = zview;
        radii[idx] = ri;
        means2D[2 * idx] = pix_x; means2D[2 * idx + 1] = pix_y;
        conic_opacity[4 * idx] = conx; conic_opacity[4 * idx + 1] = cony; conic_opacity[4 * idx + 2] = conz;
        conic_opacity[4 * idx + 3] = opacities[idx];
        tiles_touched[idx] = (uint32_t)((rmax[1] - rmin[1]) * (rmax[0] - rmin[0]));
    }
    return culled;
}

/* rasterizer_impl.cu:35-50 */
static uint32_t getHigherMsb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

/*
 * K2..K5: inclusive scan, duplicateWithKeys, STABLE sort of (key,value) on bits [0, 32+bit),
 * identifyTileRanges (rasterizer_impl.cu:70-138, 281-321).
 * keys_sorted[R], point_list[R], ranges[2*T] (zero-initialised, tiles without instances keep (0,0)).
 */
int gho_binning(int P, int W, int H, const int* radii, const float* depths, const float* means2D,
                const uint32_t* tiles_touched, long long R,
                uint64_t* keys_sorted, uint32_t* point_list, uint32_t* ranges)
{
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const int T = gx * gy;
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)T);
    if (R == 0) return 0;
    uint64_t* keys = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)R);
    uint32_t* vals = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)R);
    uint64_t* keys2 = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)R);
    uint32_t* vals2 = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)R);
    if (!keys || !vals || !keys2 || !vals2) { free(keys); free(vals); free(keys2); free(vals2); return -1; }
    /* duplicateWithKeys: offsets = prefix sum over Gaussian index; y outer, x inner */
    size_t off = 0;
    for (int idx = 0; idx < P; idx++) {
        if (radii[idx] > 0) {
            int rmin[2], rmax[2];
            getRect(means2D[2 * idx], means2D[2 * idx + 1], radii[idx], gx, gy, rmin, rmax);
            uint32_t dbits;
            memcpy(&dbits, depths + idx, 4);
            for (int y = rmin[1]; y < rmax[1]; y++)
                for (int x = rmin[0]; x < rmax[0]; x++) {
                    uint64_t key = (uint64_t)(y * gx + x);
                    key <<= 32;
                    key |= dbits;
                    keys[off] = key; vals[off] = (uint32_t)idx; off++;
                }
        }
        (void)tiles_touched;
    }
    if ((long long)off != R) { free(keys); free(vals); free(keys2); free(vals2); return -2; }
    /* stable LSD radix sort, 8-bit digits, over bits [0, 32 + bit) */
    const int end_bit = 32 + (int)getHigherMsb((uint32_t)T);
    for (int shift = 0; shift < end_bit; shift += 8) {
        size_t count[257];
        memset(count, 0, sizeof(count));
        const int nb = (end_bit - shift) < 8 ? (end_bit - shift) : 8;
        const uint64_t mask = ((uint64_t)1 << nb) - 1;
        for (long long i = 0; i < R; i++) count[((keys[i] >> shift) & mask) + 1]++;
        for (int d = 0; d < 256; d++) count[d + 1] += count[d];
        for (long long i = 0; i < R; i++) {
            const size_t d = (size_t)((keys[i] >> shift) & mask);
            keys2[count[d]] = keys[i]; vals2[count[d]] = vals[i]; count[d]++;
        }
        uint64_t* tk = keys; keys = keys2; keys2 = tk;
        uint32_t* tv = vals; vals = vals2; vals2 = tv;
    }
    memcpy(keys_sorted, keys, sizeof(uint64_t) * (size_t)R);
    memcpy(point_list, vals, sizeof(uint32_t) * (size_t)R);
    /* identifyTileRanges */
    for (long long i = 0; i < R; i++) {
        const uint32_t cur = (uint32_t)(keys[i] >> 32);
        if (i == 0) ranges[2 * cur] = 0;
        else {
            const uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
            if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * cur] = (uint32_t)i; }
        }
        if (i == R - 1) ranges[2 * cur + 1] = (uint32_t)R;
    }
    free(keys); free(vals); free(keys2); free(vals2);
    return 0;
}

/* forward.cu:358-361 in nvcc's rounding order */
static inline float power_of(float dx, float dy, float ca, float cb, float cc) {
    const float s = fmaf(dx, dx * ca, dy * (dy * cc));
    return fmaf(s, -0.5f, -(dy * (dx * cb))); /* SASS: FFMA R, s, -0.5, -t */
}

static inline float exp_f(float x) { return (float)exp((double)x); }

/*
 * K6: renderCUDA forward (forward.cu:287-400).  Per-pixel semantics; the block-level batching of the
 * kernel only decides when a whole tile may stop, it never changes a pixel.  n_contrib is the
 * 1-based list position of the last blended Gaussian (forward.cu:354,387,396).
 * Also counts evaluated / contributing (pixel, Gaussian) pairs for diagnostics (may be NULL).
 */
void gho_render_forward(int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                        const float* means2D, const float* conic_opacity, const float* features,
                        const float* bg, float* out_color, float* final_T, uint32_t* n_contrib,
                        long long* pairs_evaluated, long long* pairs_contributing)
{
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    long long n_eval = 0, n_con = 0;
#pragma omp parallel for schedule(dynamic, 4) reduction(+ : n_eval, n_con)
    for (int tile = 0; tile < gx * gy; tile++) {
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int ly = 0; ly < BLOCK_Y; ly++)
            for (int lx = 0; lx < BLOCK_X; lx++) {
                const int px = tx * BLOCK_X + lx, py = ty * BLOCK_Y + ly;
                if (px >= W || py >= H) continue;
                const float pxf = (float)px, pyf = (float)py;
                float T = 1.0f;
                float C[NUM_CHANNELS] = {0};
                uint32_t contributor = 0, last_contributor = 0;
                for (uint32_t i = r0; i < r1; i++) {
                    contributor++;
                    n_eval++;
                    const uint32_t id = point_list[i];
                    const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                    const float* co = conic_opacity + 4 * id;
                    const float power = power_of(dx, dy, co[0], co[1], co[2]);
                    if (power > 0.0f) continue;
                    const float alpha = fminf(0.99f, co[3] * exp_f(power));
                    if (alpha < 1.0f / 255.0f) continue;
                    const float test_T = T * (1.0f - alpha);
                    if (test_T < 0.0001f) break; /* done = true */
                    n_con++;
                    for (int ch = 0; ch < NUM_CHANNELS; ch++)
                        C[ch] = fmaf(T, alpha * features[(size_t)id * NUM_CHANNELS + ch], C[ch]);
                    T = test_T;
                    last_contributor = contributor;
                }
                const size_t pix = (size_t)py * W + px;
                final_T[pix] = T;
                n_contrib[pix] = last_contributor;
                for (int ch = 0; ch < NUM_CHANNELS; ch++)
                    out_color[(size_t)ch * H * W + pix] = fmaf(T, bg[ch], C[ch]); /* forward.cu:398 */
            }
    }
    if (pairs_evaluated) *pairs_evaluated = n_eval;
    if (pairs_contributing) *pairs_contributing = n_con;
}

/*
 * K7: renderCUDA backward (backward.cu:403-561).  Per-pair terms are formed in float32 exactly as the
 * kernel forms them; the per-Gaussian sums (float atomicAdd in arbitrary order in the reference) are
 * accumulated in double.  dL_dmean2D is (P,3) with z untouched, dL_dconic (P,4) with .z untouched.
 */
void gho_render_backward(int P, int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                         const float* means2D, const float* conic_opacity, const float* features,
                         const float* bg, const float* final_T, const uint32_t* n_contrib,
                         const float* dL_dpixels,
                         float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolors)
{
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    double* acc = (double*)calloc((size_t)P * 16, sizeof(double));
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H; /* backward.cu:464-465 */
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < gx * gy; tile++) {
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t r0 = ranges[2 * tile];
        for (int ly = 0; ly < BLOCK_Y; ly++)
            for (int lx = 0; lx < BLOCK_X; lx++) {
                const int px = tx * BLOCK_X + lx, py = ty * BLOCK_Y + ly;
                if (px >= W || py >= H) continue;
                const size_t pix = (size_t)py * W + px;
                const float pxf = (float)px, pyf = (float)py;
                const float T_final = final_T[pix];
                float T = T_final;
                const uint32_t last_contributor = n_contrib[pix];
                float accum_rec[NUM_CHANNELS] = {0}, last_color[NUM_CHANNELS] = {0}, dL_dpixel[NUM_CHANNELS];
                for (int ch = 0; ch < NUM_CHANNELS; ch++) dL_dpixel[ch] = dL_dpixels[(size_t)ch * H * W + pix];
                float last_alpha = 0.f;
                /* back to front over list positions last_contributor-1 .. 0 (backward.cu:476,490-492) */
                for (long long pos = (long long)last_contributor - 1; pos >= 0; pos--) {
                    const uint32_t id = point_list[r0 + pos];
                    const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                    const float* co = conic_opacity + 4 * id;
                    const float power = power_of(dx, dy, co[0], co[1], co[2]);
                    if (power > 0.0f) continue;
                    const float G = exp_f(power);
                    const float alpha = fminf(0.99f, co[3] * G);
                    if (alpha < 1.0f / 255.0f) continue;
                    T = T / (1.f - alpha);
                    const float dchannel_dcolor = alpha * T;
                    float dL_dalpha = 0.0f;
                    double* a = acc + (size_t)id * 16;
                    for (int ch = 0; ch < NUM_CHANNELS; ch++) {
                        const float c = features[(size_t)id * NUM_CHANNELS + ch];
                        accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                        last_color[ch] = c;
                        const float dL_dchannel = dL_dpixel[ch];
                        dL_dalpha += (c - accum_rec[ch]) * dL_dchannel;
                        const float v = dchannel_dcolor * dL_dchannel;
#pragma omp atomic
                        a[ch] += (double)v;
                    }
                    dL_dalpha *= T;
                    last_alpha = alpha;
                    float bg_dot_dpixel = 0;
                    for (int i = 0; i < NUM_CHANNELS; i++) bg_dot_dpixel += bg[i] * dL_dpixel[i];
                    dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot_dpixel;
                    const float dL_dG = co[3] * dL_dalpha;
                    const float gdx = G * dx, gdy = G * dy;
                    const float dG_ddelx = -gdx * co[0] - gdy * co[1];
                    const float dG_ddely = -gdy * co[2] - gdx * co[1];
                    const float v10 = dL_dG * dG_ddelx * ddelx_dx, v11 = dL_dG * dG_ddely * ddely_dy;
                    const float v12 = -0.5f * gdx * dx * dL_dG, v13 = -0.5f * gdx * dy * dL_dG, v14 = -0.5f * gdy * dy * dL_dG;
                    const float v15 = G * dL_dalpha;
#pragma omp atomic
                    a[10] += (double)v10;
#pragma omp atomic
                    a[11] += (double)v11;
#pragma omp atomic
                    a[12] += (double)v12;
#pragma omp atomic
                    a[13] += (double)v13;
#pragma omp atomic
                    a[14] += (double)v14;
#pragma omp atomic
                    a[15] += (double)v15;
                }
            }
    }
    for (int i = 0; i < P; i++) {
        const double* a = acc + (size_t)i * 16;
        for (int ch = 0; ch < NUM_CHANNELS; ch++) dL_dcolors[(size_t)i * NUM_CHANNELS + ch] = (float)a[ch];
        dL_dmean2D[3 * i + 0] = (float)a[10]; dL_dmean2D[3 * i + 1] = (float)a[11]; dL_dmean2D[3 * i + 2] = 0.f;
        dL_dconic[4 * i + 0] = (float)a[12]; dL_dconic[4 * i + 1] = (float)a[13]; dL_dconic[4 * i + 2] = 0.f;
        dL_dconic[4 * i + 3] = (float)a[14];
        dL_dopacity[i] = (float)a[15];
    }
    free(acc);
}

/*
 * K8 + K9: computeCov2DCUDA (backward.cu:144-274), preprocessCUDA backward (:346-400) and the
 * backward of computeCov3D (:278-341).  Only runs when conic_precomp == NULL, like the reference
 * (backward.cu:371,398,588).  Outputs must be zero-initialised by the caller.
 */
void gho_preprocess_backward(int P, int W, int H, const float* means3D, const int* radii,
                             const float* scales, float mod, const float* rotations,
                             const float* cov3D_precomp, const float* conic_precomp,
                             const float* view, const float* proj, float tan_fovx, float tan_fovy,
                             const float* dL_dmean2D, const float* dL_dconics,
                             float* dL_dmeans, float* dL_dcov, float* dL_dscale, float* dL_drot)
{
    if (conic_precomp != NULL) return;
    const float h_y = H / (2.0f * tan_fovy), h_x = W / (2.0f * tan_fovx);
    for (int idx = 0; idx < P; idx++) {
        if (!(radii[idx] > 0)) continue;
        const float* mean = means3D + 3 * idx;
        float c3buf[6];
        const float* cov3D;
        if (cov3D_precomp) cov3D = cov3D_precomp + 6 * idx;
        else { computeCov3D(scales + 3 * idx, mod, rotations + 4 * idx, c3buf); cov3D = c3buf; }
        const float dLc[3] = {dL_dconics[4 * idx], dL_dconics[4 * idx + 1], dL_dconics[4 * idx + 3]};
        float t[3] = {view[0] * mean[0] + view[4] * mean[1] + view[8] * mean[2] + view[12],
                      view[1] * mean[0] + view[5] * mean[1] + view[9] * mean[2] + view[13],
                      view[2] * mean[0] + view[6] * mean[1] + view[10] * mean[2] + view[14]};
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float txtz = t[0] / t[2], tytz = t[1] / t[2];
        t[0] = fminf(limx, fmaxf(-limx, txtz)) * t[2];
        t[1] = fminf(limy, fmaxf(-limy, tytz)) * t[2];
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        /* glm column-major matrices as arrays M[c][r] */
        const float J[3][3] = {{h_x / t[2], 0.f, -(h_x * t[0]) / (t[2] * t[2])},
                               {0.f, h_y / t[2], -(h_y * t[1]) / (t[2] * t[2])},
                               {0.f, 0.f, 0.f}};
        const float Wm[3][3] = {{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}};
        const float Vrk[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}};
        float Tm[3][3], A[3][3], c2[3][3];
        for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++)
            Tm[j][i] = Wm[0][i] * J[j][0] + Wm[1][i] * J[j][1] + Wm[2][i] * J[j][2];
        /* A = transpose(T) * transpose(Vrk):  A[j][i] = sum_k T[i][k] * Vrk[k][j] */
        for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++)
            A[j][i] = Tm[i][0] * Vrk[0][j] + Tm[i][1] * Vrk[1][j] + Tm[i][2] * Vrk[2][j];
        for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++)
            c2[j][i] = A[0][i] * Tm[j][0] + A[1][i] * Tm[j][1] + A[2][i] * Tm[j][2];
        const float a = c2[0][0] + 0.3f, b = c2[0][1], c = c2[1][1] + 0.3f;
        const float denom = a * c - b * b;
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float* dc = dL_dcov + 6 * idx;
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c * c * dLc[0] + 2 * b * c * dLc[1] + (denom - a * c) * dLc[2]);
            dL_dc = denom2inv * (-a * a * dLc[2] + 2 * a * b * dLc[1] + (denom - a * c) * dLc[0]);
            dL_db = denom2inv * 2 * (b * c * dLc[0] - (denom + 2 * b * b) * dLc[1] + a * b * dLc[2]);
            dc[0] = (Tm[0][0] * Tm[0][0] * dL_da + Tm[0][0] * Tm[1][0] * dL_db + Tm[1][0] * Tm[1][0] * dL_dc);
            dc[3] = (Tm[0][1] * Tm[0][1] * dL_da + Tm[0][1] * Tm[1][1] * dL_db + Tm[1][1] * Tm[1][1] * dL_dc);
            dc[5] = (Tm[0][2] * Tm[0][2] * dL_da + Tm[0][2] * Tm[1][2] * dL_db + Tm[1][2] * Tm[1][2] * dL_dc);
            dc[1] = 2 * Tm[0][0] * Tm[0][1] * dL_da + (Tm[0][0] * Tm[1][1] + Tm[0][1] * Tm[1][0]) * dL_db + 2 * Tm[1][0] * Tm[1][1] * dL_dc;
            dc[2] = 2 * Tm[0][0] * Tm[0][2] * dL_da + (Tm[0][0] * Tm[1][2] + Tm[0][2] * Tm[1][0]) * dL_db + 2 * Tm[1][0] * Tm[1][2] * dL_dc;
            dc[4] = 2 * Tm[0][2] * Tm[0][1] * dL_da + (Tm[0][1] * Tm[1][2] + Tm[0][2] * Tm[1][1]) * dL_db + 2 * Tm[1][1] * Tm[1][2] * dL_dc;
        } else {
            for (int i = 0; i < 6; i++) dc[i] = 0;
        }
        const float dL_dT00 = 2 * (Tm[0][0] * Vrk[0][0] + Tm[0][1] * Vrk[0][1] + Tm[0][2] * Vrk[0][2]) * dL_da +
                              (Tm[1][0] * Vrk[0][0] + Tm[1][1] * Vrk[0][1] + Tm[1][2] * Vrk[0][2]) * dL_db;
        const float dL_dT01 = 2 * (Tm[0][0] * Vrk[1][0] + Tm[0][1] * Vrk[1][1] + Tm[0][2] * Vrk[1][2]) * dL_da +
                              (Tm[1][0] * Vrk[1][0] + Tm[1][1] * Vrk[1][1] + Tm[1][2] * Vrk[1][2]) * dL_db;
        const float dL_dT02 = 2 * (Tm[0][0] * Vrk[2][0] + Tm[0][1] * Vrk[2][1] + Tm[0][2] * Vrk[2][2]) * dL_da +
                              (Tm[1][0] * Vrk[2][0] + Tm[1][1] * Vrk[2][1] + Tm[1][2] * Vrk[2][2]) * dL_db;
        const float dL_dT10 = 2 * (Tm[1][0] * Vrk[0][0] + Tm[1][1] * Vrk[0][1] + Tm[1][2] * Vrk[0][2]) * dL_dc +
                              (Tm[0][0] * Vrk[0][0] + Tm[0][1] * Vrk[0][1] + Tm[0][2] * Vrk[0][2]) * dL_db;
        const float dL_dT11 = 2 * (Tm[1][0] * Vrk[1][0] + Tm[1][1] * Vrk[1][1] + Tm[1][2] * Vrk[1][2]) * dL_dc +
                              (Tm[0][0] * Vrk[1][0] + Tm[0][1] * Vrk[1][1] + Tm[0][2] * Vrk[1][2]) * dL_db;
        const float dL_dT12 = 2 * (Tm[1][0] * Vrk[2][0] + Tm[1][1] * Vrk[2][1] + Tm[1][2] * Vrk[2][2]) * dL_dc +
                              (Tm[0][0] * Vrk[2][0] + Tm[0][1] * Vrk[2][1] + Tm[0][2] * Vrk[2][2]) * dL_db;
        const float dL_dJ00 = Wm[0][0] * dL_dT00 + Wm[0][1] * dL_dT01 + Wm[0][2] * dL_dT02;
        const float dL_dJ02 = Wm[2][0] * dL_dT00 + Wm[2][1] * dL_dT01 + Wm[2][2] * dL_dT02;
        const float dL_dJ11 = Wm[1][0] * dL_dT10 + Wm[1][1] * dL_dT11 + Wm[1][2] * dL_dT12;
        const float dL_dJ12 = Wm[2][0] * dL_dT10 + Wm[2][1] * dL_dT11 + Wm[2][2] * dL_dT12;
        const float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
        const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t[0]) * tz3 * dL_dJ02 + (2 * h_y * t[1]) * tz3 * dL_dJ12;
        /* transformVec4x3Transpose (auxiliary.h:88-97); ASSIGNED, backward.cu:273 */
        float dm[3] = {view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz,
                       view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz,
                       view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz};
        /* preprocessCUDA backward, projection part (backward.cu:371-391) */
        {
            const float m_hom_w = proj[3] * mean[0] + proj[7] * mean[1] + proj[11] * mean[2] + proj[15];
            const float m_w = 1.0f / (m_hom_w + 0.0000001f);
            const float mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
            const float g0 = dL_dmean2D[3 * idx], g1 = dL_dmean2D[3 * idx + 1];
            dm[0] += (proj[0] * m_w - proj[3] * mul1) * g0 + (proj[1] * m_w - proj[3] * mul2) * g1;
            dm[1] += (proj[4] * m_w - proj[7] * mul1) * g0 + (proj[5] * m_w - proj[7] * mul2) * g1;
            dm[2] += (proj[8] * m_w - proj[11] * mul1) * g0 + (proj[9] * m_w - proj[11] * mul2) * g1;
        }
        dL_dmeans[3 * idx] = dm[0]; dL_dmeans[3 * idx + 1] = dm[1]; dL_dmeans[3 * idx + 2] = dm[2];

        /* computeCov3D backward (backward.cu:278-341); only when scales are given */
        if (scales && !cov3D_precomp) {
            const float* q = rotations + 4 * idx;
            const float r = q[0], x = q[1], y = q[2], z = q[3];
            const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                   {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                   {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
            const float s[3] = {mod * scales[3 * idx], mod * scales[3 * idx + 1], mod * scales[3 * idx + 2]};
            float M[3][3], D[3][3], dM[3][3];
            for (int cc = 0; cc < 3; cc++) for (int rr = 0; rr < 3; rr++) M[cc][rr] = s[rr] * R[cc][rr];
            D[0][0] = dc[0]; D[1][1] = dc[3]; D[2][2] = dc[5];
            D[0][1] = D[1][0] = 0.5f * dc[1]; D[0][2] = D[2][0] = 0.5f * dc[2]; D[1][2] = D[2][1] = 0.5f * dc[4];
            /* dL_dM = 2.0f * M * dL_dSigma */
            for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++)
                dM[j][i] = (2.0f * M[0][i]) * D[j][0] + (2.0f * M[1][i]) * D[j][1] + (2.0f * M[2][i]) * D[j][2];
            /* Rt = transpose(R), dL_dMt = transpose(dL_dM); dL_dscale.k = dot(Rt[k], dL_dMt[k]) */
            float Y[3][3];
            for (int cc = 0; cc < 3; cc++) for (int rr = 0; rr < 3; rr++) Y[cc][rr] = dM[rr][cc];
            for (int k = 0; k < 3; k++)
                dL_dscale[3 * idx + k] = R[0][k] * Y[k][0] + R[1][k] * Y[k][1] + R[2][k] * Y[k][2];
            for (int k = 0; k < 3; k++) for (int rr = 0; rr < 3; rr++) Y[k][rr] *= s[k];
            float* dq = dL_drot + 4 * idx;
            dq[0] = 2 * z * (Y[0][1] - Y[1][0]) + 2 * y * (Y[2][0] - Y[0][2]) + 2 * x * (Y[1][2] - Y[2][1]);
            dq[1] = 2 * y * (Y[1][0] + Y[0][1]) + 2 * z * (Y[2][0] + Y[0][2]) + 2 * r * (Y[1][2] - Y[2][1]) - 4 * x * (Y[2][2] + Y[1][1]);
            dq[2] = 2 * x * (Y[1][0] + Y[0][1]) + 2 * r * (Y[2][0] - Y[0][2]) + 2 * z * (Y[1][2] + Y[2][1]) - 4 * y * (Y[2][2] + Y[0][0]);
            dq[3] = 2 * r * (Y[0][1] - Y[1][0]) + 2 * x * (Y[2][0] + Y[0][2]) + 2 * y * (Y[1][2] + Y[2][1]) - 4 * z * (Y[1][1] + Y[0][0]);
        }
    }
}

/* rasterizer_impl.cu:54-66 (checkFrustum): near-plane test only */
void gho_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present) {
    for (int i = 0; i < P; i++) {
        const float* p = means3D + 3 * i;
        present[i] = !(xform_row(viewmatrix, 2, p[0], p[1], p[2]) <= 0.2f);
    }
}

#ifdef __cplusplus
}
#endif
