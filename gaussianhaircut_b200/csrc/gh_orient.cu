// Hair orientation maps: the reference's `calc_orients` (src/preprocessing/calc_orientation_maps.py:53-97) evaluated on
// the whole image (DESIGN §15 states the contract).  Two calls on the caller's stream, one workspace:
//   gh_orient_dog    grayscale (0.2989 r + 0.5870 g + 0.1140 b) and the difference of two Gaussians, both in float64
//                    with scipy.ndimage.correlate1d's operation order (mode 'nearest', axis 0 then axis 1): writes the
//                    float64 DoG and, into the workspace, its float32 rounding that the Gabor stage reads.
//   gh_orient_gabor  (1) re-lays the bank out per chunk of 64 filters of one group, tap-major, and records for every 8
//                    consecutive filters the smallest rectangle that holds all their non-zero taps; (2) one fused pass
//                    per 8x8 pixel tile: the zero-padded cross-correlation with every filter in FP32 FMA (SIMT pipe, no
//                    tensor cores), |response| kept in shared memory for a whole group, then the per-pixel epilogue
//                    (gh_orient_math.h): argmax, sum, variance, and the argmin over groups.
// No atomics: every output is a fixed sequence of rounded operations, so the maps are bit-reproducible.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "gh_orient_math.h"
#include "../../include/gh_rasterizer.h"

#include <climits>

namespace {

constexpr int GH_OR_TILE = 8;                   // output tile: 8 x 8 pixels per CTA
constexpr int GH_OR_PIX = GH_OR_TILE * GH_OR_TILE;
constexpr int GH_OR_CHUNK = 64;                 // filters of one group per shared-memory chunk
constexpr int GH_OR_THREADS = 256;              // 8 warps; warp w computes filters [8w, 8w + 8) of a chunk
constexpr int GH_OR_HALO = GH_OR_TILE + GH_ORIENT_MAX_K - 1;     // 24 input columns a row of the tile reads
constexpr int GH_OR_HS = 28;                    // halo row stride (floats): 8 rows of 16-byte loads hit distinct banks

static_assert(GH_OR_HS >= GH_OR_HALO && GH_OR_HS % 4 == 0, "halo rows must hold the window and stay 16-byte aligned");

// Workspace (256-byte aligned base): the float32 DoG, the float64 gray image and the two axis-0 passes (gh_orient_dog),
// then the re-laid bank and the per-warp tap rectangles (gh_orient_gabor).
struct GhOrientWS {
    float* dog32;
    double* gray;
    double* tlo;
    double* thi;
    float* wbank;
    int4* sup;

    static size_t dog_bytes(size_t npix) {
        return gh_align_up(npix * sizeof(float), 256) + 3 * gh_align_up(npix * sizeof(double), 256);
    }
    static size_t chunks(int N, int nf) { return (size_t)(N / nf) * ((nf + GH_OR_CHUNK - 1) / GH_OR_CHUNK); }
    static size_t bytes(size_t npix, int N, int K, int nf) {
        const size_t nb = chunks(N, nf);
        return dog_bytes(npix) + gh_align_up(nb * K * K * GH_OR_CHUNK * sizeof(float), 256) +
               gh_align_up(nb * 8 * sizeof(int4), 256);
    }
    static GhOrientWS carve(char* base, size_t npix, int N, int K, int nf) {
        GhOrientWS w;
        size_t off = 0;
        w.dog32 = (float*)(base + off); off += gh_align_up(npix * sizeof(float), 256);
        w.gray = (double*)(base + off); off += gh_align_up(npix * sizeof(double), 256);
        w.tlo = (double*)(base + off); off += gh_align_up(npix * sizeof(double), 256);
        w.thi = (double*)(base + off); off += gh_align_up(npix * sizeof(double), 256);
        w.wbank = (float*)(base + off);
        if (N > 0) off += gh_align_up(chunks(N, nf) * K * K * GH_OR_CHUNK * sizeof(float), 256);
        w.sup = (int4*)(base + off);
        return w;
    }
};

// ------------------------------------------------------------------------------------------- difference of Gaussians
__global__ void __launch_bounds__(256)
gh_orient_gray_kernel(int n, int C, const unsigned char* __restrict__ img, double* __restrict__ gray)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned char* p = img + (size_t)i * C;
    // numpy: 0.2989 * r + 0.5870 * g + 0.1140 * b, left to right, in float64
    gray[i] = __dadd_rn(__dadd_rn(__dmul_rn(0.2989, (double)p[0]), __dmul_rn(0.5870, (double)p[1])),
                        __dmul_rn(0.1140, (double)p[2]));
}

// scipy.ndimage.correlate1d on a symmetric odd filter (ni_filters.c, NI_Correlate1D): out = x[i] * w[r], then
// out += (x[i + jj] + x[i - jj]) * w[r + jj] for jj = -r .. -1, every operation rounded on its own; 'nearest' clamps the
// index to the line.
__device__ __forceinline__ double gh_orient_corr1d(const double* __restrict__ line, long long stride, int n, int i,
                                                   const double* __restrict__ w, int r)
{
    double acc = __dmul_rn(line[(long long)i * stride], __ldg(w + r));
    for (int jj = -r; jj < 0; jj++) {
        const int a = max(i + jj, 0), b = min(i - jj, n - 1);
        acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(line[(long long)a * stride], line[(long long)b * stride]), __ldg(w + r + jj)));
    }
    return acc;
}

__global__ void __launch_bounds__(256)
gh_orient_dog_axis0_kernel(int H, int W, const double* __restrict__ gray, const double* __restrict__ wl, int rl,
                           const double* __restrict__ wh, int rh, double* __restrict__ tlo, double* __restrict__ thi)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const int y = i / W, x = i - y * W;
    tlo[i] = gh_orient_corr1d(gray + x, W, H, y, wl, rl);
    thi[i] = gh_orient_corr1d(gray + x, W, H, y, wh, rh);
}

__global__ void __launch_bounds__(256)
gh_orient_dog_axis1_kernel(int H, int W, const double* __restrict__ tlo, const double* __restrict__ thi,
                           const double* __restrict__ wl, int rl, const double* __restrict__ wh, int rh,
                           double* __restrict__ dog, float* __restrict__ dog32)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const int y = i / W, x = i - y * W;
    const size_t row = (size_t)y * W;
    const double d = __dsub_rn(gh_orient_corr1d(tlo + row, 1, W, x, wl, rl), gh_orient_corr1d(thi + row, 1, W, x, wh, rh));
    dog[i] = d;
    dog32[i] = __double2float_rn(d);
}

// ---------------------------------------------------------------------------------------------------- Gabor bank
// One CTA per (group g, chunk c): wbank[b][tap][f] = bank[(c*64 + f) * G + g][tap] (0 past num_filters), and for warp w
// the rectangle (ky0, ky1, kx0, kx1) holding every non-zero tap of filters [8w, 8w + 8) of the chunk (ky1 = -1: none).
__global__ void __launch_bounds__(GH_OR_THREADS)
gh_orient_bank_kernel(int K, int nf, int G, int nch, const float* __restrict__ bank, float* __restrict__ wbank,
                      int4* __restrict__ sup)
{
    const int b = blockIdx.x, g = b / nch, c = b - g * nch;
    const int KK = K * K;
    float* dst = wbank + (size_t)b * KK * GH_OR_CHUNK;
    for (int e = threadIdx.x; e < KK * GH_OR_CHUNK; e += GH_OR_THREADS) {
        const int tap = e / GH_OR_CHUNK, f = e - tap * GH_OR_CHUNK, j = c * GH_OR_CHUNK + f;
        dst[e] = j < nf ? bank[((size_t)j * G + g) * KK + tap] : 0.f;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int y0 = INT_MAX, y1 = -1, x0 = INT_MAX, x1 = -1;
    for (int e = lane; e < 8 * KK; e += 32) {
        const int f = warp * 8 + e / KK, tap = e % KK, j = c * GH_OR_CHUNK + f;
        if (j < nf && bank[((size_t)j * G + g) * KK + tap] != 0.f) {
            const int ky = tap / K, kx = tap - ky * K;
            y0 = min(y0, ky); y1 = max(y1, ky); x0 = min(x0, kx); x1 = max(x1, kx);
        }
    }
    y0 = __reduce_min_sync(0xffffffffu, y0); y1 = __reduce_max_sync(0xffffffffu, y1);
    x0 = __reduce_min_sync(0xffffffffu, x0); x1 = __reduce_max_sync(0xffffffffu, x1);
    if (lane == 0) sup[(size_t)b * 8 + warp] = y1 < 0 ? make_int4(0, -1, 0, -1) : make_int4(y0, y1, x0, x1);
}

__device__ __forceinline__ void gh_orient_chunk_async(float* s, const float* __restrict__ g, int n4)
{
    for (int i = threadIdx.x; i < n4; i += GH_OR_THREADS) {
        const unsigned int sa = (unsigned int)__cvta_generic_to_shared(s + 4 * i);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(g + 4 * i));
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}

// Shared memory: the tile's zero-padded input window (8 + K - 1 rows, stride 28), two chunk buffers of K*K*64 weights
// (tap-major: the 8 filters of a warp are 32 consecutive bytes), and |response| of one group, F[j][64 pixels].
// Thread (warp w, lane l) computes pixels (row l & 7, columns 0..7) x filters 8w + 2(l >> 3) + {0, 1} of each chunk:
// 16 accumulators; per tap one broadcast 8-byte weight load and 16 FMAs on a register window of the row.
__global__ void __launch_bounds__(GH_OR_THREADS, 1)
gh_orient_gabor_kernel(int H, int W, int K, int nf, int G, int nch, const float* __restrict__ dog32,
                       const float* __restrict__ wbank, const int4* __restrict__ sup, const float* __restrict__ thetas,
                       long long* __restrict__ orients, float* __restrict__ var)
{
    extern __shared__ float4 gh_orient_smem[];
    float* halo = (float*)gh_orient_smem;
    const int KK = K * K;
    float* wbuf0 = halo + GH_OR_HALO * GH_OR_HS;
    float* wbuf1 = wbuf0 + KK * GH_OR_CHUNK;
    float* Fs = wbuf1 + KK * GH_OR_CHUNK;

    const int ntx = (W + GH_OR_TILE - 1) / GH_OR_TILE;
    const int tx0 = (blockIdx.x % ntx) * GH_OR_TILE, ty0 = (blockIdx.x / ntx) * GH_OR_TILE;
    const int pad = K / 2, rows = GH_OR_TILE + K - 1;
    const int tid = threadIdx.x;
    const int total = G * nch, n4 = KK * GH_OR_CHUNK / 4;

    gh_orient_chunk_async(wbuf0, wbank, n4);
    for (int e = tid; e < GH_OR_HALO * GH_OR_HS; e += GH_OR_THREADS) {
        const int hy = e / GH_OR_HS, hx = e - hy * GH_OR_HS;
        const int gy = ty0 + hy - pad, gx = tx0 + hx - pad;
        float v = 0.f;
        if (hy < rows && hx < GH_OR_TILE + K - 1 && gy >= 0 && gy < H && gx >= 0 && gx < W) v = dog32[(size_t)gy * W + gx];
        halo[e] = v;
    }

    const int warp = tid >> 5, lane = tid & 31;
    const int s = lane & 7, fl = warp * 8 + 2 * (lane >> 3);
    int best_idx = 0;
    float best_var = 0.f;
    for (int it = 0; it < total; it++) {
        if (it + 1 < total) {
            gh_orient_chunk_async((it & 1) ? wbuf0 : wbuf1, wbank + (size_t)(it + 1) * KK * GH_OR_CHUNK, n4);
            asm volatile("cp.async.wait_group 1;\n" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        }
        __syncthreads();
        const int g = it / nch, c = it - g * nch;
        const float* wb = (it & 1) ? wbuf1 : wbuf0;
        const int4 sp = sup[(size_t)it * 8 + warp];
        float acc0[GH_OR_TILE], acc1[GH_OR_TILE];
#pragma unroll
        for (int r = 0; r < GH_OR_TILE; r++) { acc0[r] = 0.f; acc1[r] = 0.f; }
        for (int ky = sp.x; ky <= sp.y; ky++) {
            const float4* rowp = (const float4*)(halo + (s + ky) * GH_OR_HS);
            float xs[GH_OR_HALO];
#pragma unroll
            for (int i = 0; i < GH_OR_HALO / 4; i++) {
                const float4 v = rowp[i];
                xs[4 * i] = v.x; xs[4 * i + 1] = v.y; xs[4 * i + 2] = v.z; xs[4 * i + 3] = v.w;
            }
            const float* wr = wb + ky * K * GH_OR_CHUNK + fl;
#pragma unroll
            for (int kx = 0; kx < GH_ORIENT_MAX_K; kx++) {
                if (kx < sp.z || kx > sp.w) continue;       // warp-uniform: taps outside the rectangle are all zero
                const float2 w = *(const float2*)(wr + kx * GH_OR_CHUNK);
#pragma unroll
                for (int r = 0; r < GH_OR_TILE; r++) {
                    acc0[r] = fmaf(w.x, xs[r + kx], acc0[r]);
                    acc1[r] = fmaf(w.y, xs[r + kx], acc1[r]);
                }
            }
        }
        const int j0 = c * GH_OR_CHUNK + fl;
        if (j0 < nf) {
            float4* o = (float4*)(Fs + (size_t)j0 * GH_OR_PIX + s * GH_OR_TILE);
            o[0] = make_float4(fabsf(acc0[0]), fabsf(acc0[1]), fabsf(acc0[2]), fabsf(acc0[3]));
            o[1] = make_float4(fabsf(acc0[4]), fabsf(acc0[5]), fabsf(acc0[6]), fabsf(acc0[7]));
        }
        if (j0 + 1 < nf) {
            float4* o = (float4*)(Fs + (size_t)(j0 + 1) * GH_OR_PIX + s * GH_OR_TILE);
            o[0] = make_float4(fabsf(acc1[0]), fabsf(acc1[1]), fabsf(acc1[2]), fabsf(acc1[3]));
            o[1] = make_float4(fabsf(acc1[4]), fabsf(acc1[5]), fabsf(acc1[6]), fabsf(acc1[7]));
        }
        if (c == nch - 1) {
            __syncthreads();
            if (tid < GH_OR_PIX) {
                int idx;
                float v;
                gh_orient_group(Fs + tid, GH_OR_PIX, nf, thetas, &idx, &v);
                gh_orient_keep(g, idx, v, best_idx, best_var);
            }
        }
        __syncthreads();     // the next chunk overwrites this buffer (and, after a group, F)
    }
    if (tid < GH_OR_PIX) {
        const int y = ty0 + tid / GH_OR_TILE, x = tx0 + tid % GH_OR_TILE;
        if (y < H && x < W) {
            orients[(size_t)y * W + x] = best_idx;
            var[(size_t)y * W + x] = best_var;
        }
    }
}

size_t gh_orient_smem_bytes(int K, int nf)
{
    return ((size_t)GH_OR_HALO * GH_OR_HS + 2 * (size_t)K * K * GH_OR_CHUNK + (size_t)nf * GH_OR_PIX) * sizeof(float);
}

int gh_orient_check_image(const char* who, int H, int W)
{
    if (H <= 0 || W <= 0 || (long long)H * W >= (1ll << 31))
        return gh_set_error(GH_E_INVALID_ARG, "%s: H and W must be positive with H*W < 2^31", who);
    return GH_OK;
}

int gh_orient_check_bank(const char* who, int N, int K, int nf)
{
    if (K < 1 || K > GH_ORIENT_MAX_K || (K & 1) == 0)
        return gh_set_error(GH_E_INVALID_ARG, "%s: K must be odd and in [1, %d]", who, GH_ORIENT_MAX_K);
    if (nf < 1 || nf > GH_ORIENT_MAX_FILTERS || N < nf || N > GH_ORIENT_MAX_N || N % nf != 0)
        return gh_set_error(GH_E_INVALID_ARG, "%s: need 1 <= num_filters <= %d and N a multiple of num_filters, N <= %d", who,
                            GH_ORIENT_MAX_FILTERS, GH_ORIENT_MAX_N);
    return GH_OK;
}

int gh_orient_check_ws(const char* who, const void* workspace, size_t bytes, size_t need)
{
    if (!workspace || ((size_t)workspace & 255))
        return gh_set_error(GH_E_INVALID_ARG, "%s: workspace must be a 256-byte aligned device pointer", who);
    if (bytes < need) return gh_set_error(GH_E_INVALID_ARG, "%s: workspace smaller than gh_orient_workspace_size", who);
    return GH_OK;
}

}  // namespace

extern "C" int gh_orient_workspace_size(int H, int W, int N, int K, int num_filters, size_t* bytes)
{
    gh_clear_error();
    int rc = gh_orient_check_image("gh_orient_workspace_size", H, W);
    if (rc == GH_OK) rc = gh_orient_check_bank("gh_orient_workspace_size", N, K, num_filters);
    if (rc != GH_OK) return rc;
    if (!bytes) return gh_set_error(GH_E_INVALID_ARG, "gh_orient_workspace_size: bytes is NULL");
    *bytes = GhOrientWS::bytes((size_t)H * W, N, K, num_filters);
    return GH_OK;
}

extern "C" int gh_orient_dog(int H, int W, int C, const unsigned char* image, const double* w_low, int r_low,
                             const double* w_high, int r_high, double* dog, void* workspace, size_t bytes,
                             gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_orient_check_image("gh_orient_dog", H, W);
    if (rc != GH_OK) return rc;
    if (C != 3 && C != 4) return gh_set_error(GH_E_INVALID_ARG, "gh_orient_dog: C must be 3 (RGB) or 4 (RGBA)");
    if (r_low < 0 || r_high < 0 || r_low > GH_ORIENT_MAX_RADIUS || r_high > GH_ORIENT_MAX_RADIUS)
        return gh_set_error(GH_E_INVALID_ARG, "gh_orient_dog: Gaussian radii must lie in [0, GH_ORIENT_MAX_RADIUS]");
    if (!image || !w_low || !w_high || !dog) return gh_set_error(GH_E_INVALID_ARG, "gh_orient_dog: missing image, weights or dog");
    if (((size_t)w_low & 7) || ((size_t)w_high & 7) || ((size_t)dog & 7))
        return gh_set_error(GH_E_INVALID_ARG, "gh_orient_dog: weights and dog must be 8-byte aligned double arrays");
    rc = gh_orient_check_ws("gh_orient_dog", workspace, bytes, GhOrientWS::dog_bytes((size_t)H * W));
    if (rc != GH_OK) return rc;
    const GhOrientWS ws = GhOrientWS::carve((char*)workspace, (size_t)H * W, 0, 1, 1);
    const int n = H * W, blocks = (n + 255) / 256;
    gh_orient_gray_kernel<<<blocks, 256, 0, stream>>>(n, C, image, ws.gray);
    gh_orient_dog_axis0_kernel<<<blocks, 256, 0, stream>>>(H, W, ws.gray, w_low, r_low, w_high, r_high, ws.tlo, ws.thi);
    gh_orient_dog_axis1_kernel<<<blocks, 256, 0, stream>>>(H, W, ws.tlo, ws.thi, w_low, r_low, w_high, r_high, dog, ws.dog32);
    return gh_launch_status("gh_orient_dog", 3);
}

extern "C" int gh_orient_gabor(int H, int W, const float* bank, int N, int K, int num_filters, const float* thetas,
                               long long* orients, float* var, void* workspace, size_t bytes, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    int rc = gh_orient_check_image("gh_orient_gabor", H, W);
    if (rc == GH_OK) rc = gh_orient_check_bank("gh_orient_gabor", N, K, num_filters);
    if (rc != GH_OK) return rc;
    if (!bank || !thetas || !orients || !var)
        return gh_set_error(GH_E_INVALID_ARG, "gh_orient_gabor: missing bank, thetas, orients or var");
    if (((size_t)bank & 3) || ((size_t)thetas & 3) || ((size_t)var & 3) || ((size_t)orients & 7))
        return gh_set_error(GH_E_INVALID_ARG, "gh_orient_gabor: bank, thetas and var must be 4-byte aligned, orients 8-byte aligned");
    rc = gh_orient_check_ws("gh_orient_gabor", workspace, bytes, GhOrientWS::bytes((size_t)H * W, N, K, num_filters));
    if (rc != GH_OK) return rc;
    const GhOrientWS ws = GhOrientWS::carve((char*)workspace, (size_t)H * W, N, K, num_filters);
    const int G = N / num_filters, nch = (num_filters + GH_OR_CHUNK - 1) / GH_OR_CHUNK;
    const size_t smem = gh_orient_smem_bytes(K, num_filters);
    const cudaError_t e = cudaFuncSetAttribute(gh_orient_gabor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return gh_cuda_status("gh_orient_gabor", "cudaFuncSetAttribute(shared memory)", e);
    gh_orient_bank_kernel<<<G * nch, GH_OR_THREADS, 0, stream>>>(K, num_filters, G, nch, bank, ws.wbank, ws.sup);
    const long long tiles = (long long)((W + GH_OR_TILE - 1) / GH_OR_TILE) * ((H + GH_OR_TILE - 1) / GH_OR_TILE);
    gh_orient_gabor_kernel<<<(unsigned int)tiles, GH_OR_THREADS, smem, stream>>>(H, W, K, num_filters, G, nch, ws.dog32,
                                                                               ws.wbank, ws.sup, thetas, orients, var);
    return gh_launch_status("gh_orient_gabor", 2);
}
