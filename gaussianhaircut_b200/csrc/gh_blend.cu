// Stage 3 / 4: per-tile front-to-back alpha compositing of the 10-channel feature vector
// (RGB, label, ones, dir2D(3), orientation confidence, depth) and its back-to-front backward.
//
// Per-pixel arithmetic and every skip/stop decision follow the reference kernels renderCUDA
// (cuda_rasterizer/forward.cu:287-400, backward.cu:403-561) bit for bit.  The work decomposition is
// new and built around the shape of strand-aligned Gaussians (long thin ellipses: of the 256 pixels
// of a tile a splat typically reaches alpha >= 1/255 on ~15):
//
//   forward  (gh_blend_forward_kernel, CTA = tile, 4 warps, a vertical pixel pair per lane, 6 CTAs per SM)
//   * lists of <= GH_INKERNEL_SORT_MAX (1792) records are depth-sorted by the CTA itself (gh_bucket_sort_tile)
//     before blending;
//   * the sorted list is staged one 384-record window at a time into shared memory with cp.async (LDGSTS),
//     single buffered: the other resident CTAs cover the gather;
//   * each staged Gaussian is scan-converted ONCE per tile: the exact-conservative x-span of
//     {alpha >= 1/255} on every pixel row gives 16-bit row masks, the two rows of a pixel pair are ORed,
//     4 shuffle transposes of 32 (Gaussian) x 32 (pair) bit matrices give one hit list per pixel pair,
//     and every lane walks only ITS pair's list -- a skipped Gaussian costs nothing, and one load of a
//     Gaussian from shared memory serves two pixels;
//   * each pixel of the pair keeps the reference's per-pixel arithmetic and decisions; a pixel that does not
//     blend a Gaussian of the pair's list keeps its state through selects.
//   backward (gh_blend_backward_kernel, CTA = tile, 4 warps, a vertical pixel pair per lane)
//   * one 384-record window staged at a time; Gaussians are scan-converted against the tile's 64 blocks
//     of 2x2 pixels and shuffle transposes leave one bit list per block;
//   * a block is owned by 2 lanes; the 16 blocks of a warp walk their own lists in lock-step (one warp
//     instruction works on 16 different Gaussians); blocks are assigned to warps by list length;
//   * the pixel pair is evaluated as float2 pairs (.x upper pixel, .y lower pixel; on sm_90 every half is
//     one scalar FP32 instruction); the six geometric gradients are built once per lane from three sums
//     over the pair, which share dx; the 16 gradient components are summed over the block's lanes and
//     leave as REDG.E.ADD.F32x4 into a 64-byte per-Gaussian record -- instead of 16 scalar atomicAdd
//     per (pixel, Gaussian) pair in the reference (backward.cu:527,549-558);
//   * dL/dalpha uses the scalar form of the reference's per-channel suffix recursion
//     (backward.cu:519-523):  sum_ch (c - accum_rec)[ch] dL[ch]  =  c.dL  -  A,   A' = a_last (c_last.dL) + (1-a_last) A.
#include "gh_common.cuh"
#include "gh_kernels.h"

#include <atomic>

#define GH_HALF_C (GH_NUM_CHANNELS / 2)

// ---- build-time tunables (defaults = the measured best; tools/bench_variants.py rebuilds with -D overrides)
#ifndef GH_FWD_CHUNK
#define GH_FWD_CHUNK 384         // forward staging window (records, a multiple of 32; 512 fits 5 CTAs per SM)
#endif
#ifndef GH_FWD_MIN_CTAS
#define GH_FWD_MIN_CTAS 6        // __launch_bounds__ second argument of the forward kernel (register cap: 80 at 6)
#endif
#ifndef GH_BWD_CHUNK
#define GH_BWD_CHUNK 384         // backward staging window (records)
#endif
#ifndef GH_BWD_MIN_CTAS
#define GH_BWD_MIN_CTAS 6        // __launch_bounds__ second argument of the backward kernel (register cap: 80 at 6)
#endif
// Ablations for timing experiments only (DESIGN.md section 9); a build with any of them set computes wrong results.
#ifndef GH_ABLATE_SORT
#define GH_ABLATE_SORT 0         // forward: skip the in-CTA tile sort
#endif
#ifndef GH_ABLATE_TRAVERSE
#define GH_ABLATE_TRAVERSE 0     // forward: skip the per-pair traversal (the blend itself)
#endif
#ifndef GH_ABLATE_REDG
#define GH_ABLATE_REDG 0         // backward: form the gradient sums but issue no reductions
#endif

namespace {

struct GhPixEval {
    float dx, dy, power, G, alpha;
    bool ok;   // passes the reference's `power > 0` and `alpha < 1/255` skips
};

__device__ __forceinline__ GhPixEval gh_eval(const float4 g0, const float4 g1, float pxf, float pyf) {
    GhPixEval e;
    e.dx = GH_SUB(g0.x, pxf);
    e.dy = GH_SUB(g0.y, pyf);
    e.power = gh_power(e.dx, e.dy, g0.z, g0.w, g1.x);
    e.G = 0.f; e.alpha = 0.f;
    e.ok = false;
    if (!(e.power > 0.0f)) {
        e.G = expf(e.power);
        e.alpha = fminf(0.99f, GH_MUL(g1.y, e.G));
        e.ok = !(e.alpha < 1.0f / 255.0f);
    }
    return e;
}

__device__ __forceinline__ void gh_cp_async16(void* smem, const void* gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void gh_cp_async8(void* smem, const void* gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void gh_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void gh_cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// Pairs of FP32 values (two pixel rows, two pixels, two channels) evaluated together.  Each half is one
// IEEE-rounded FMUL / FADD / FFMA: the _rn intrinsics keep the compiler from contracting or reordering
// them, so both passes (and the reference's scalar code) round identically.
__device__ __forceinline__ float2 gh_f2(float a) { return make_float2(a, a); }
__device__ __forceinline__ float2 gh_neg2(float2 a) { return make_float2(-a.x, -a.y); }
__device__ __forceinline__ float2 gh_mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 gh_add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 gh_sub2(float2 a, float2 b) { return gh_add2(a, gh_neg2(b)); }
__device__ __forceinline__ float2 gh_fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float gh_rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

#define GH_FWD_THREADS 128                       // CTA = tile, 4 warps, a vertical pixel pair per lane
#define GH_FWD_WORDS (GH_FWD_CHUNK / 32)         // list words per pair and window
static_assert(GH_FWD_CHUNK % 32 == 0 && GH_FWD_WORDS <= 32, "forward window: a multiple of 32 records, at most 1024");

// One staged window of N records in shared memory, for both blend kernels: geometry records and feature rows.
template <int N>
struct GhStage {
    float4 g0[N];
    float4 g1[N];
    float2 feat[N * GH_HALF_C];
};
// Dynamic shared memory of the forward: the staging buffers + the pair lists ([word][pair]) while blending, and before
// that the in-CTA sort's two key buffers + its scratch.
constexpr size_t kFwdStageBytes = sizeof(GhStage<GH_FWD_CHUNK>) + (size_t)GH_FWD_WORDS * GH_FWD_THREADS * sizeof(uint32_t);
constexpr size_t kFwdSortBytes = 16u * GH_INKERNEL_SORT_MAX + 4u * GH_SORT_SCRATCH_WORDS;
constexpr size_t kFwdSmemBytes = kFwdStageBytes > kFwdSortBytes ? kFwdStageBytes : kFwdSortBytes;

// issue the gather of one instance (geometry record + feature row) into slot `slot`
template <int N>
__device__ __forceinline__ void gh_stage_issue(GhStage<N>& st, int slot, uint32_t id,
                                               const GhGeo* __restrict__ geo, const float* __restrict__ features) {
    const float4* gp = reinterpret_cast<const float4*>(geo + id);
    gh_cp_async16(&st.g0[slot], gp);
    gh_cp_async16(&st.g1[slot], gp + 1);
    const float2* fp = reinterpret_cast<const float2*>(features + (size_t)id * GH_NUM_CHANNELS);
#pragma unroll
    for (int k = 0; k < GH_HALF_C; k++) gh_cp_async8(&st.feat[slot * GH_HALF_C + k], fp + k);
}

// Level Q of the exact-conservative {alpha >= 1/255} test of a Gaussian against the tile with origin (tx0, ty0): a
// pixel at offset d = (dx, dy) from the mean can reach alpha >= 1/255 only where a dx^2 + 2 b dx dy + c dy^2 <= Q.
// Exactly that is Q = 2 thr (power = -q / 2, alpha = op exp(power)); the slack, 1e-3 plus 2e-5 of the quadratic's
// largest magnitude over the tile, covers __logf in thr and the rounding of power.
__device__ __forceinline__ float gh_span_level(const float4 g0, const float4 g1, float tx0, float ty0) {
    const float gx = g0.x, gy = g0.y, a = g0.z, b = g0.w, c = g1.x, thr = g1.z;
    const float mxd = fmaxf(fabsf(gx - tx0), fabsf(gx - (tx0 + 15.f)));
    const float myd = fmaxf(fabsf(gy - ty0), fabsf(gy - (ty0 + 15.f)));
    const float slack = 1e-3f + 2e-5f * (a * mxd * mxd + c * myd * myd + 2.f * fabsf(b) * mxd * myd);
    return 2.f * (thr + slack);
}

// Per-PAIR instance lists of one staged window (forward pass).  Batch `word` = Gaussians [32 word, 32 word + 32) of
// the window, one per lane: on every pixel row the exact-conservative x-span of {alpha >= 1/255} (gh_span_level, same
// quadratic as gh_block_mask_2x2) becomes a 16-bit column mask, and the two rows of a pixel pair are ORed into one
// pair-row mask.  Warp w of the blend owns pair-rows 2w and 2w + 1 (pair p = 32 w + lane: column lane & 15, pair-row 2w + lane / 16),
// so one 32-bit word per (Gaussian, blend warp) covers its 32 pairs.  Each of these 32 (Gaussian) x 32 (pair) bit
// matrices is transposed inside the warp with 5 shuffle steps, so lane P ends with "which of the batch's 32
// Gaussians reach pair P of warp w" and stores it: no atomics, no clearing pass.  pairbits is [word][pair] -> a warp
// reads consecutive banks.
__device__ __forceinline__ uint32_t gh_transpose32(uint32_t x, int lane) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const uint32_t m = (s == 16) ? 0x0000ffffu : (s == 8) ? 0x00ff00ffu : (s == 4) ? 0x0f0f0f0fu
                         : (s == 2) ? 0x33333333u : 0x55555555u;
        const uint32_t y = __shfl_xor_sync(0xffffffffu, x, s);
        x = (lane & s) ? (((y >> s) & m) | (x & ~m)) : ((x & m) | ((y & m) << s));
    }
    return x;
}

__device__ __forceinline__ void gh_build_pair_lists(const GhStage<GH_FWD_CHUNK>& st, uint32_t* pairbits, int cnt,
                                                    int word, int lane, float tx0, float ty0) {
    const int j = word * 32 + lane;
    uint32_t pairmask[8];            // pair-row t = pixel rows 2t, 2t + 1
#pragma unroll
    for (int t = 0; t < 8; t++) pairmask[t] = 0u;
    float gx = 0.f, gy = 0.f, b = 0.f, ia = 0.f, aQ = -1.f, bbac = 0.f;
    int r0 = 16, r1 = -1;            // rows of the tile this Gaussian can reach
    bool all_pixels = false;
    if (j < cnt) {
        const float4 g0 = st.g0[j], g1 = st.g1[j];
        gx = g0.x; gy = g0.y; b = g0.w;
        const float a = g0.z, c = g1.x, pd = g1.w;
        const float Q = gh_span_level(g0, g1, tx0, ty0);
        if (pd == 0.f || Q != Q) {
            all_pixels = true; r0 = 0; r1 = 15;                     // no bound available: every pixel
        } else if (Q >= 0.f) {
            ia = __frcp_rn(a);
            aQ = a * Q;
            bbac = b * b - a * c;                                   // < 0 for a PD conic
            // rows with a real span: dy^2 < aQ / (ac - b^2)
            const float ry = sqrtf(aQ / (-bbac)) + 0.01f;
            r0 = 0; r1 = 15;
            if (ry == ry) { r0 = max(0, __float2int_ru(gy - ry - ty0)); r1 = min(15, __float2int_rd(gy + ry - ty0)); }
        }
    }
    // warp-uniform row window: the 32 Gaussians of a batch are neighbours in depth, not in space, but
    // strand Gaussians are small, so most rows are empty for the whole warp
    int wr0 = r0, wr1 = r1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        wr0 = min(wr0, __shfl_xor_sync(0xffffffffu, wr0, o));
        wr1 = max(wr1, __shfl_xor_sync(0xffffffffu, wr1, o));
    }
    // the two rows of a pair as one float2 step; a row without a real span has disc <= 0 and is masked out below
    const float2 bbac2 = gh_f2(bbac), aQ2 = gh_f2(aQ), b2 = gh_f2(b), ia2 = gh_f2(ia), gx2 = gh_f2(gx);
    const float2 off2 = gh_f2(-0.01f), ntx2 = gh_f2(-tx0);
#pragma unroll
    for (int t = 0; t < 8; t++) {
        if (2 * t + 1 < wr0 || 2 * t > wr1) continue;               // uniform
        const float2 dy = make_float2(gy - (ty0 + (float)(2 * t)), gy - (ty0 + (float)(2 * t + 1)));
        // a dx^2 + 2 b dy dx + (c dy^2 - Q) <= 0,  dx = gx - px
        const float2 disc = gh_fma2(gh_mul2(dy, dy), bbac2, aQ2);
        const float2 sq = gh_mul2(disc, make_float2(rsqrtf(disc.x), rsqrtf(disc.y)));
        const float2 hb = gh_mul2(b2, dy);
        const float2 lo = gh_add2(gh_add2(gh_fma2(gh_sub2(hb, sq), ia2, gx2), off2), ntx2);
        const float2 hi = gh_add2(gh_add2(gh_fma2(gh_add2(hb, sq), ia2, gx2), gh_neg2(off2)), ntx2);
        const int p0a = max(0, __float2int_ru(lo.x)), p1a = min(15, __float2int_rd(hi.x));
        const int p0b = max(0, __float2int_ru(lo.y)), p1b = min(15, __float2int_rd(hi.y));
        const uint32_t ma = (disc.x > 0.f && p0a <= p1a) ? (((2u << (p1a - p0a)) - 1u) << p0a) : 0u;
        const uint32_t mb = (disc.y > 0.f && p0b <= p1b) ? (((2u << (p1b - p0b)) - 1u) << p0b) : 0u;
        pairmask[t] = all_pixels ? 0xffffu : (ma | mb);             // rows outside [r0, r1] have disc <= 0
    }
#pragma unroll
    for (int w = 0; w < GH_FWD_THREADS / 32; w++) {
        const uint32_t m = pairmask[2 * w] | (pairmask[2 * w + 1] << 16);   // my coverage of blend warp w's pairs
        uint32_t col = 0u;
        if (__any_sync(0xffffffffu, m != 0u)) col = gh_transpose32(m, lane);
        pairbits[word * GH_FWD_THREADS + w * 32 + lane] = col;              // pair 32w+lane: bits = Gaussians
    }
}

// ------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(GH_FWD_THREADS, GH_FWD_MIN_CTAS)
gh_blend_forward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_perm, uint64_t* inst,
                        const GhGeo* __restrict__ geo, const float* __restrict__ features,
                        int W, int H, int gx, const float* __restrict__ bg,
                        float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                        float* __restrict__ out,
                        float4* __restrict__ zero_records, size_t zero_n)   // NULL, or the P * 4 float4 of acc16
{
    // Forward needs no cross-pixel communication, so every lane walks the list of ITS OWN pixel pair (the union of
    // the two pixels' lists): a lane only ever touches Gaussians whose alpha >= 1/255 footprint (conservatively)
    // reaches one of its two pixels, whatever the other lanes of the warp are doing.
    extern __shared__ __align__(16) unsigned char gh_fwd_smem[];
    GhStage<GH_FWD_CHUNK>& st = *reinterpret_cast<GhStage<GH_FWD_CHUNK>*>(gh_fwd_smem);
    uint32_t* pairbits = reinterpret_cast<uint32_t*>(gh_fwd_smem + sizeof(st));   // [word][pair] (GH_FWD_WORDS x 128)

    gh_pdl_wait();                                    // the lists, ranges and tile order come from emit and the scan
    gh_pdl_trigger();

    const int tile = (int)tile_perm[blockIdx.x];      // heaviest tiles first
    const int tx = tile % gx, ty = tile / gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // a warp owns four pixel rows: lanes 0..15 rows 4w, 4w+1, lanes 16..31 rows 4w+2, 4w+3 (pixel pair = one column)
    const int px = tx * GH_BLOCK_X + (lane & 15);
    const int py0 = ty * GH_BLOCK_Y + 4 * warp + 2 * (lane >> 4);
    const bool inside0 = (px < W) && (py0 < H), inside1 = (px < W) && (py0 + 1 < H);
    const float pxf = (float)px, pyf0 = (float)py0, pyf1 = (float)(py0 + 1);
    const float tx0 = (float)(tx * GH_BLOCK_X), ty0 = (float)(ty * GH_BLOCK_Y);

    const uint2 rg = ranges[tile];
    const int n = (int)(rg.y - rg.x);
    const int nchunks = (n + GH_FWD_CHUNK - 1) / GH_FWD_CHUNK;

    // state of the pixel pair: .x = pixel (px, py0), .y = pixel (px, py0 + 1)
    float2 T = make_float2(1.0f, 1.0f);
    float2 C[GH_NUM_CHANNELS];
#pragma unroll
    for (int ch = 0; ch < GH_NUM_CHANNELS; ch++) C[ch] = make_float2(0.f, 0.f);
    uint32_t last0 = 0, last1 = 0;
    bool done0 = !inside0, done1 = !inside1;
    bool warp_done = (__ballot_sync(0xffffffffu, done0 && done1) == 0xffffffffu);

    // Sort this tile's bucket by (depth bits, Gaussian index) right here when it fits the shared memory
    // (<= GH_INKERNEL_SORT_MAX records): the sort is latency/barrier bound, the blend is issue bound, and as
    // one kernel the two overlap across the CTAs of an SM.  The sorted bucket is written back for the
    // backward pass.  Longer lists were sorted by gh_tile_split_long_kernel + gh_segment_sort_kernel
    // (gh_binning.cu) before this launch.
    if (!GH_ABLATE_SORT && n >= 2 && n <= (int)GH_INKERNEL_SORT_MAX) {
        uint64_t* sbase = reinterpret_cast<uint64_t*>(gh_fwd_smem);                    // GH_INKERNEL_SORT_MAX keys
        uint64_t* spong = sbase + GH_INKERNEL_SORT_MAX;                                  // the same again
        uint32_t* sscratch = reinterpret_cast<uint32_t*>(spong + GH_INKERNEL_SORT_MAX);  // GH_SORT_SCRATCH_WORDS
        uint64_t* gl = inst + rg.x;
        // The bucket is one contiguous run of 8-byte records: the TMA engine copies it into shared memory
        // (cp.async.bulk, one request, completion on an mbarrier) instead of a load/store loop.  Bulk copies
        // move 16-byte granules, so the run is widened to even record indices; `skeys` skips the extra
        // leading record.  The rare run that would not fit after widening takes the loop.
        const uint32_t odd = rg.x & 1u;
        const uint32_t nrec = ((uint32_t)n + odd + 1u) & ~1u;
        uint64_t* skeys = sbase;                  // the loop path below uses the whole buffer
        if (nrec <= GH_INKERNEL_SORT_MAX) {
            skeys = sbase + odd;
            __shared__ __align__(8) uint64_t s_mbar;
            const uint32_t mbar = (uint32_t)__cvta_generic_to_shared(&s_mbar);
            if (tid == 0) {
                asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar) : "memory");
                asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            }
            __syncthreads();
            if (tid == 0) {
                const uint32_t bytes = nrec * 8u;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"((uint32_t)__cvta_generic_to_shared(sbase)), "l"(gl - odd), "r"(bytes), "r"(mbar) : "memory");
            }
            uint32_t landed = 0;
            for (uint32_t it = 0; it < (1u << 24) && !landed; it++)
                asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n selp.u32 %0, 1, 0, p;\n}"
                             : "=r"(landed) : "r"(mbar) : "memory");
            if (!landed) __trap();            // the copy engine never reported completion
        } else {
            for (int i = tid; i < n; i += GH_FWD_THREADS) skeys[i] = gl[i];
            __syncthreads();
        }
        if (n <= 64) gh_bitonic_sort(skeys, (uint32_t)n, tid, GH_FWD_THREADS);
        else gh_bucket_sort_tile<GH_FWD_THREADS>(skeys, spong, sscratch, n, tid);
        for (int i = tid; i < n; i += GH_FWD_THREADS) gl[i] = skeys[i];
        __syncthreads();
    }

    // staging: thread t gathers slots t, t + 128, ... of a window; the indices of the next window wait in registers
    constexpr int PER_THREAD = (GH_FWD_CHUNK + GH_FWD_THREADS - 1) / GH_FWD_THREADS;
    uint32_t next_id[PER_THREAD];
#pragma unroll
    for (int h = 0; h < PER_THREAD; h++) {
        const int slot = tid + h * GH_FWD_THREADS;
        next_id[h] = (slot < GH_FWD_CHUNK && slot < n) ? (uint32_t)inst[(size_t)rg.x + slot] : 0u;
    }
    // gather window `c` from next_id, then fetch the indices of window c + 1
    auto stage_window = [&](int c) {
        const int wbase = c * GH_FWD_CHUNK;
#pragma unroll
        for (int h = 0; h < PER_THREAD; h++) {
            const int slot = tid + h * GH_FWD_THREADS;
            if (slot < GH_FWD_CHUNK && wbase + slot < n) gh_stage_issue(st, slot, next_id[h], geo, features);
        }
        gh_cp_async_commit();
#pragma unroll
        for (int h = 0; h < PER_THREAD; h++) {
            const int slot = tid + h * GH_FWD_THREADS, nx = wbase + GH_FWD_CHUNK + slot;
            if (slot < GH_FWD_CHUNK && nx < n) next_id[h] = (uint32_t)inst[(size_t)rg.x + nx];
        }
    };

    for (int c = 0; c < nchunks; c++) {
        const int base = c * GH_FWD_CHUNK;
        const int cnt = min(GH_FWD_CHUNK, n - base);
        const int nwords = (cnt + 31) >> 5;
        // everyone is done with the previous window; block-wide early exit like the reference's
        // __syncthreads_count(done) == BLOCK_SIZE
        if (__syncthreads_and(warp_done)) break;
        stage_window(c);
        gh_cp_async_wait_all();
        __syncthreads();
        // each of the 4 warps scan-converts every fourth batch of 32 Gaussians
        for (int word = warp; word < nwords; word += GH_FWD_THREADS / 32)
            gh_build_pair_lists(st, pairbits, cnt, word, lane, tx0, ty0);
        __syncthreads();

        if (!(done0 && done1) && !GH_ABLATE_TRAVERSE) {
            // which of my pair's list words are non-empty
            uint32_t nz = 0u;
#pragma unroll
            for (int k = 0; k < GH_FWD_WORDS; k++)
                if (k < nwords) nz |= (pairbits[k * GH_FWD_THREADS + tid] != 0u) ? (1u << k) : 0u;
            int wi = 0;
            uint32_t cur = 0u;
            while (true) {
                if (cur == 0u) {
                    if (nz == 0u) break;
                    wi = __ffs(nz) - 1;
                    nz &= nz - 1;
                    cur = pairbits[wi * GH_FWD_THREADS + tid];
                }
                const int bpos = __ffs(cur) - 1;
                cur &= cur - 1;
                const int jj = wi * 32 + bpos;
                const float4 g0 = st.g0[jj], g1 = st.g1[jj];
                // each pixel takes the reference's per-pixel path (forward.cu:356-394): gh_eval, the early stop on
                // test_T, then the blend.  A pixel that is done, or that skips this Gaussian, keeps its state bit
                // for bit (selects, no multiplication by zero).
                const GhPixEval e0 = gh_eval(g0, g1, pxf, pyf0), e1 = gh_eval(g0, g1, pxf, pyf1);
                const float2 test_T = make_float2(GH_MUL(T.x, GH_SUB(1.0f, e0.alpha)), GH_MUL(T.y, GH_SUB(1.0f, e1.alpha)));
                const bool ok0 = !done0 && e0.ok, ok1 = !done1 && e1.ok;
                const bool stop0 = ok0 && test_T.x < 0.0001f, stop1 = ok1 && test_T.y < 0.0001f;
                const bool blend0 = ok0 && !stop0, blend1 = ok1 && !stop1;
                done0 = done0 || stop0;
                done1 = done1 || stop1;
                if (blend0 || blend1) {
                    // C[ch] = fma(T, alpha * f[ch], C[ch]) (forward.cu:379-380 as ptxas fuses it)
                    const uint32_t pos = (uint32_t)(base + jj + 1);
#pragma unroll
                    for (int k = 0; k < GH_HALF_C; k++) {
                        const float2 f = st.feat[jj * GH_HALF_C + k];
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const float fc = h ? f.y : f.x;
                            float2& Cc = C[2 * k + h];
                            const float c0 = GH_FMA(T.x, GH_MUL(e0.alpha, fc), Cc.x);
                            const float c1 = GH_FMA(T.y, GH_MUL(e1.alpha, fc), Cc.y);
                            Cc = make_float2(blend0 ? c0 : Cc.x, blend1 ? c1 : Cc.y);
                        }
                    }
                    T = make_float2(blend0 ? test_T.x : T.x, blend1 ? test_T.y : T.y);
                    last0 = blend0 ? pos : last0;
                    last1 = blend1 ? pos : last1;
                }
                if (done0 && done1) break;
            }
        }
        warp_done = (__ballot_sync(0xffffffffu, done0 && done1) == 0xffffffffu);
    }
    gh_cp_async_wait_all();

    const size_t plane = (size_t)H * W;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        if (!(r ? inside1 : inside0)) continue;
        const size_t pix = (size_t)(py0 + r) * W + px;
        const float Tr = r ? T.y : T.x;
        final_T[pix] = Tr;
        n_contrib[pix] = r ? last1 : last0;
#pragma unroll
        for (int ch = 0; ch < GH_NUM_CHANNELS; ch++)
            out[ch * plane + pix] = GH_FMA(Tr, __ldg(bg + ch), r ? C[ch].y : C[ch].x);
    }

    // Clear the backward's accumulation records, so that the blend backward needs no clearing pass of its own.  The
    // first quarter of the CTAs -- the heaviest tiles, launched first -- take one contiguous slice each: their
    // traversal is bound by latency and leaves the memory pipe idle, whereas the light and empty tiles that run last
    // are bound by their image stores (zeroing in every CTA cost ~9 us of blend forward on the bench step, in the
    // prologue or at the end alike).  At the end, after the CTA's own stores: CTAs finish at different times, so the
    // clearing spreads over the kernel.
    const unsigned nzero = max(1u, gridDim.x / 4);
    if (zero_records != nullptr && blockIdx.x < nzero) {
        const size_t per = (zero_n + nzero - 1) / nzero;
        const size_t end = min(zero_n, per * (blockIdx.x + 1));
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        for (size_t i = per * blockIdx.x + tid; i < end; i += GH_FWD_THREADS) zero_records[i] = z;
    }
}

// ------------------------------------------------------------------------------------------ backward
// The backward's blocks: 2x2 pixels, 8 across the tile (block index = 8 by + bx), each owned by 2 lanes.
constexpr int kBwdBlocks = 64;

// Backward staging: ONE window of GH_BWD_CHUNK instances (single-buffered; the other resident CTAs of
// the SM cover the gather latency), their Gaussian indices and one list per block.  The 16 blocks of a
// warp walk their lists in lock-step, so a warp spends max(list length over its blocks) steps per window.
struct GhStageB : GhStage<GH_BWD_CHUNK> {
    uint32_t id[GH_BWD_CHUNK];
    uint32_t bits[kBwdBlocks][GH_BWD_CHUNK / 32 + 1];   // [block][word]; +1 pad against bank conflicts
};

// Which of the tile's 64 blocks can this Gaussian reach with alpha >= 1/255?  Bit = by * 8 + bx;
// .x = block rows 0..3, .y = rows 4..7.  Exact-conservative: on each pixel row the set {q(d) <= Q}
// (gh_span_level) is an x-interval obtained from the quadratic; the interval is widened by 0.01 px and
// rounded outwards to whole pixels.  Returns all ones when the conic is not positive definite (no bound
// available).  Skipping a Gaussian in a block whose bit is clear cannot change any pixel of that block:
// each of them would take the reference's `alpha < 1/255 -> continue` (forward.cu:370, backward.cu:503).
// Two pixel rows per instruction; a row without a real span has disc <= 0 -> s = NaN -> fminf / fmaxf
// ignore it.
__device__ __forceinline__ uint2 gh_block_mask_2x2(const float4 g0, const float4 g1, float tx0, float ty0) {
    const float gx = g0.x, gy = g0.y, a = g0.z, b = g0.w, c = g1.x, pd = g1.w;
    if (pd == 0.f) return make_uint2(0xffffffffu, 0xffffffffu);
    const float Q = gh_span_level(g0, g1, tx0, ty0);
    if (!(Q >= 0.f)) return (Q != Q) ? make_uint2(0xffffffffu, 0xffffffffu) : make_uint2(0u, 0u);
    const float2 ia = gh_f2(__frcp_rn(a)), aQ = gh_f2(a * Q), bbac = gh_f2(b * b - a * c), gx2 = gh_f2(gx), b2 = gh_f2(b);
    float2 dy = make_float2(gy - ty0, gy - (ty0 + 1.f));     // rows 2 by, 2 by + 1
    uint32_t m[2] = {0u, 0u};
    // not unrolled across the two halves: the build runs while the blend loop's state is live in registers
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
        uint32_t mh = 0u;
#pragma unroll
        for (int by = 0; by < 4; by++) {
            // a dx^2 + 2 b dy dx + (c dy^2 - Q) <= 0,  dx = gx - px
            const float2 disc = gh_fma2(gh_mul2(dy, dy), bbac, aQ);
            const float2 s = gh_mul2(disc, make_float2(rsqrtf(disc.x), rsqrtf(disc.y)));   // NaN unless disc > 0
            const float2 hb = gh_mul2(b2, dy);
            const float2 lo2 = gh_fma2(gh_sub2(hb, s), ia, gx2), hi2 = gh_fma2(gh_add2(hb, s), ia, gx2);
            const float xlo = fminf(fminf(1e30f, lo2.x), lo2.y), xhi = fmaxf(fmaxf(-1e30f, hi2.x), hi2.y);
            // tile-local integer pixel columns inside [xlo - .01, xhi + .01]
            const float lo = (xlo - 0.01f) - tx0, hi = (xhi + 0.01f) - tx0;
            const int p0 = max(0, __float2int_ru(lo)), p1 = min(15, __float2int_rd(hi));
            if (p0 <= p1) {
                const int b0 = p0 >> 1, b1 = p1 >> 1;
                mh |= (((2u << (b1 - b0)) - 1u) << b0) << (8 * by);
            }
            dy = gh_add2(dy, gh_f2(-2.f));
        }
        if (half == 0) m[0] = mh; else m[1] = mh;
    }
    return make_uint2(m[0], m[1]);
}

// batch `word` = instances [32 word, 32 word + 32) of the window, one per lane; a 5-step shuffle
// transpose turns the 32 block masks into one list word per block (lane = block).  The word is cut at
// the block's deepest blended list position `glast` here, once, rather than in the traversal loop.
__device__ __forceinline__ uint32_t gh_valid_bits(uint32_t glast, int first_pos) {
    const int lim = (int)glast - first_pos;
    return lim >= 32 ? 0xffffffffu : (lim <= 0 ? 0u : ((1u << lim) - 1u));
}

// glast_lo / glast_hi: deepest blended list position of blocks `lane` and 32 + `lane` (after the transpose, lane b
// holds the words of blocks b and 32 + b).  Callers read them from shared memory at every build rather than hold
// them in registers through the blend loop.
__device__ __forceinline__ void gh_build_lists_b(GhStageB& st, int cnt, int word, int lane, float tx0, float ty0,
                                                 int base, uint32_t glast_lo, uint32_t glast_hi) {
    const int j = word * 32 + lane;
    uint2 m = make_uint2(0u, 0u);
    if (j < cnt) m = gh_block_mask_2x2(st.g0[j], st.g1[j], tx0, ty0);
    uint32_t lo = 0, hi = 0;
    if (__any_sync(0xffffffffu, m.x != 0u)) lo = gh_transpose32(m.x, lane);
    if (__any_sync(0xffffffffu, m.y != 0u)) hi = gh_transpose32(m.y, lane);
    st.bits[lane][word] = lo & gh_valid_bits(glast_lo, base + word * 32);
    st.bits[32 + lane][word] = hi & gh_valid_bits(glast_hi, base + word * 32);
}

// CTA = tile = 4 warps.  A lane owns a vertical pixel pair (x, y0), (x, y0+1); 2 lanes own a 2x2 block;
// the 16 blocks of a warp walk their own lists in lock-step, i.e. every warp instruction works on SIXTEEN
// different Gaussians.  The two pixels of a lane are summed in registers, then the 16 gradient components
// over the block's 2 lanes (gh_group2_reduce16), leaving two REDG.E.ADD.F32x4 per lane.
#define GH_BWD_THREADS 128

// Each lane sends the half of the 16 components its partner keeps through 8 SHFL.BFLY and adds the partner's half
// to its own (8 FADD); no shared memory.  Every sum is own + partner's value.  The even lane keeps components 0..3
// and 8..11, the odd lane 4..7 and 12..15, so each of the pair's two REDG.E.ADD.F32x4 instructions updates one
// 32-byte sector of the 64-byte record (with halves 0..7 / 8..15, which touch both sectors, the kernel took 25 %
// longer: DESIGN.md section 9).
__device__ __forceinline__ void gh_group2_reduce16(const float (&v)[16], int lane, float4& out0, float4& out1) {
    const bool odd = (lane & 1) != 0;
    float k[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int c = (i & 3) + 8 * (i >> 2);      // component the even lane keeps; the odd lane keeps c + 4
        const float send = odd ? v[c] : v[c + 4], keep = odd ? v[c + 4] : v[c];
        k[i] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
    }
    out0 = make_float4(k[0], k[1], k[2], k[3]);
    out1 = make_float4(k[4], k[5], k[6], k[7]);
}

// State of the lane's pixel pair; .x = pixel (x, y0), .y = pixel (x, y0 + 1).
struct GhBwdPair {
    float2 T, A, last_alpha, last_cdot;
    float2 ntf_bg;                 // -T_final * (bg . dL_dpix)
    float2 npy;                    // -(pixel y)
    uint32_t last0, last1;
    float2 dL0[GH_HALF_C], dL1[GH_HALF_C];   // dL/dpixel of pixel 0 / pixel 1, channel pairs (2k, 2k+1)
};

// The pixel pair's share of one Gaussian, branch-free: every lane runs the same instruction stream and
// a pixel that does not blend this Gaussian (behind its last contributor, power > 0, alpha < 1/255 --
// the reference's three `continue`s, backward.cu:490-505) has alpha = G = 0, contributes exact zeros
// and keeps its state.  power / alpha are bit-identical to the forward pass (same operation order,
// every half rounded like FMUL / FFMA), so both passes agree on which pixels blend.  Downstream of those
// decisions only gradients are formed, and their sums are free to be reassociated.  v = the 16 gradient
// components summed over the two pixels; nddelx_dx / nddely_dy = -W/2, -H/2.
__device__ __forceinline__ bool gh_bwd_pair(GhBwdPair& p, const float4 g0, const float4 g1, const float2* feat,
                                            float pxf, uint32_t pos, float nddelx_dx, float nddely_dy, float (&v)[16]) {
    const float dx = GH_SUB(g0.x, pxf);
    const float2 dx2 = gh_f2(dx);
    const float2 dy = gh_add2(gh_f2(g0.y), p.npy);
    // gh_power: fma(fma(dx, dx*ca, dy*(dy*cc)), -0.5, -(dy*(dx*cb)))
    const float t1 = GH_MUL(dx, g0.z), dxcb = GH_MUL(dx, g0.w);
    const float2 t3 = gh_mul2(dy, gh_mul2(dy, gh_f2(g1.x)));
    const float2 sq = gh_fma2(dx2, gh_f2(t1), t3);
    const float2 power = gh_fma2(sq, gh_f2(-0.5f), gh_mul2(dy, gh_f2(-dxcb)));
    const float Gx0 = expf((power.x > 0.0f) ? 0.0f : power.x);   // expf(power) whenever the reference evaluates it
    const float Gx1 = expf((power.y > 0.0f) ? 0.0f : power.y);
    const float2 ao = gh_mul2(gh_f2(g1.y), make_float2(Gx0, Gx1));
    const float alpha0 = fminf(0.99f, ao.x), alpha1 = fminf(0.99f, ao.y);
    const bool ok0 = (pos < p.last0) & !(power.x > 0.0f) & !(alpha0 < 1.0f / 255.0f);
    const bool ok1 = (pos < p.last1) & !(power.y > 0.0f) & !(alpha1 < 1.0f / 255.0f);
    const float2 am = make_float2(ok0 ? alpha0 : 0.f, ok1 ? alpha1 : 0.f);
    const float2 G = make_float2(ok0 ? Gx0 : 0.f, ok1 ? Gx1 : 0.f);
    // T_{before this Gaussian} = T / (1 - alpha); gradients only need ~1 ulp here: MUFU.RCP, 1 - alpha
    // is in [0.01, 1] and rcp(1) == 1 exactly
    const float2 om = gh_sub2(gh_f2(1.0f), am);
    const float2 r = make_float2(gh_rcp_approx(om.x), gh_rcp_approx(om.y));
    p.T = gh_mul2(p.T, r);
    const float2 w = gh_mul2(am, p.T);                          // d(out)/d(color)
    const float2 w0 = gh_f2(w.x), w1 = gh_f2(w.y);
    float2 c0, c1;
#pragma unroll
    for (int k = 0; k < GH_HALF_C; k++) {
        const float2 f = feat[k];
        c0 = (k == 0) ? gh_mul2(f, p.dL0[0]) : gh_fma2(f, p.dL0[k], c0);
        c1 = (k == 0) ? gh_mul2(f, p.dL1[0]) : gh_fma2(f, p.dL1[k], c1);
        const float2 vc = gh_fma2(w1, p.dL1[k], gh_mul2(w0, p.dL0[k]));
        v[2 * k] = vc.x; v[2 * k + 1] = vc.y;
    }
    const float2 cdot = make_float2(c0.x + c0.y, c1.x + c1.y);
    // suffix recursion on the dot product (backward.cu:519-523), A' = a_last c_last + (1 - a_last) A written
    // as A + a_last (c_last - A); state advances only when blended
    const float2 A_new = gh_fma2(p.last_alpha, gh_sub2(p.last_cdot, p.A), p.A);
    // alpha also scales how much background shows through (backward.cu:535-538).  Not masked: every use
    // below is multiplied by G, which is 0 for a pixel that does not blend.
    const float2 dL_dalpha = gh_fma2(gh_sub2(cdot, A_new), p.T, gh_mul2(p.ntf_bg, r));
    // State update WITHOUT selects: a pixel that does not blend stores last_alpha = 0, so the next step computes
    // A_new = fma(0, last_cdot - A, A) = A exactly (both are finite) -- the recursion skips it just as the
    // reference's `continue` does, and A_new of this step is what the next blended step would have computed.
    p.A = A_new;
    p.last_cdot = cdot;
    p.last_alpha = am;
    // Geometry.  With q = G dL/dalpha per pixel and dL/dG = opacity dL/dalpha (backward.cu:539-558):
    //   dL/dmean2D.x = -(a dx sum(op q) + b sum(op q dy)) W/2     dL/dconic.a = -dx^2/2 sum(op q)
    //   dL/dmean2D.y = -(c sum(op q dy) + b dx sum(op q)) H/2     dL/dconic.b = -dx/2 sum(op q dy)
    //   dL/dopacity  = sum(q)                                    dL/dconic.c = -1/2 sum(op q dy^2)
    // The two pixels of the pair share dx, so only the three sums over the pair depend on the pixel.
    const float2 q = gh_mul2(G, dL_dalpha), qdy = gh_mul2(q, dy);
    const float S0 = q.x + q.y, S1 = qdy.x + qdy.y, S2 = fmaf(qdy.y, dy.y, qdy.x * dy.x);
    const float U0 = g1.y * S0, U1 = g1.y * S1;
    const float hdx = -0.5f * dx;
    v[10] = fmaf(t1, U0, g0.w * U1) * nddelx_dx;
    v[11] = fmaf(g1.x, U1, dxcb * U0) * nddely_dy;
    v[12] = (hdx * dx) * U0;
    v[13] = hdx * U1;
    v[14] = (-0.5f * g1.y) * S2;
    v[15] = S0;
    return ok0 | ok1;
}

// ---- deterministic instantiation (DET = true): no atomics.  The tile's partial sum for each instance of its list
// leaves as one 64-byte row at a Gaussian-major slot (GhDetWS); gh_det_gather_kernel sums the rows of each
// Gaussian in a fixed order afterwards.
struct GhDetArgs {
    const int* radii;          // the radii emit used: with geo.x, geo.y they give the tile rectangle
    const uint32_t* off;       // [P + 1] first row of each Gaussian
    float4* rows;              // [R][4]
    int gy;
};

// Row of instance (Gaussian id, tile (tx, ty)): off[id] + the tile's row-major rank inside the Gaussian's tile
// rectangle, from the same gh_get_rect call on the same inputs as emit (gh_binning.cu)
__device__ __forceinline__ float4* gh_det_row(const GhDetArgs& d, float mx, float my, uint32_t id, int tx, int ty, int gx) {
    int minx, miny, maxx, maxy;
    gh_get_rect(mx, my, d.radii[id], gx, d.gy, minx, miny, maxx, maxy);
    const uint32_t k = (uint32_t)((ty - miny) * (maxx - minx) + (tx - minx));
    return d.rows + 4 * ((size_t)d.off[id] + k);
}

// Per-warp partial records of one 32-record list word, [warp][record][quad], after the staging buffers
constexpr size_t kBwdDetPartBytes = (size_t)(GH_BWD_THREADS / 32) * 32 * 4 * sizeof(float4);

template <bool DET>
__global__ void __launch_bounds__(GH_BWD_THREADS, GH_BWD_MIN_CTAS)
gh_blend_backward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_perm, const uint64_t* __restrict__ inst,
                         const GhGeo* __restrict__ geo, const float* __restrict__ features,
                         int W, int H, int gx, const float* __restrict__ bg,
                         const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                         const float* __restrict__ dL_dpix,
                         float* __restrict__ acc16,   // [P][16]: colors 0..9, mean2D x,y, conic x,y,w, opacity
                         GhDetArgs det)               // DET only
{
    extern __shared__ __align__(16) unsigned char gh_bwd_smem[];
    GhStageB& st = *reinterpret_cast<GhStageB*>(gh_bwd_smem);
    __shared__ uint32_t s_warp_last[GH_BWD_THREADS / 32];
    __shared__ uint32_t s_glast[kBwdBlocks];              // per block: deepest list position any of its pixels blended
    __shared__ uint8_t s_perm[GH_BWD_THREADS / 32][kBwdBlocks];   // per warp (redundant copies): rank -> block

    gh_pdl_wait();                                    // every input but the caller's comes from the forward
    gh_pdl_trigger();
    const int tile = (int)tile_perm[blockIdx.x];      // heaviest tiles first
    const int tx = tile % gx, ty = tile / gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float tx0 = (float)(tx * GH_BLOCK_X), ty0 = (float)(ty * GH_BLOCK_Y);
    const size_t plane = (size_t)H * W;
    const uint2 rg = ranges[tile];

    // ---- how far do the blocks / the tile reach into the list?  (natural block order here)
    {
        const int nb = 16 * warp + lane / 2;
        const int nx = tx * GH_BLOCK_X + 2 * (nb % 8) + (lane % 2);
        const int ny = ty * GH_BLOCK_Y + 2 * (nb / 8);
        uint32_t gl = 0;
        if (nx < W && ny < H) gl = n_contrib[(size_t)ny * W + nx];
        if (nx < W && ny + 1 < H) gl = max(gl, n_contrib[(size_t)(ny + 1) * W + nx]);
        gl = max(gl, __shfl_xor_sync(0xffffffffu, gl, 1));
        if ((lane % 2) == 0) s_glast[nb] = gl;
        uint32_t wl = gl;
#pragma unroll
        for (int o = 2; o < 32; o <<= 1) wl = max(wl, __shfl_xor_sync(0xffffffffu, wl, o));
        if (lane == 0) s_warp_last[warp] = wl;
    }
    __syncthreads();
    uint32_t tile_last = 0;
#pragma unroll
    for (int w = 0; w < GH_BWD_THREADS / 32; w++) tile_last = max(tile_last, s_warp_last[w]);
    const int n = (int)tile_last;             // nothing beyond is blended by any pixel of this tile
    const int nchunks = (n + GH_BWD_CHUNK - 1) / GH_BWD_CHUNK;
    if constexpr (DET) {                      // instances past tile_last: zero rows
        const int len = (int)(rg.y - rg.x);
        for (int j = n + tid; j < len; j += GH_BWD_THREADS) {
            const uint32_t id = (uint32_t)inst[(size_t)rg.x + j];
            const float2 m = *reinterpret_cast<const float2*>(geo + id);
            float4* row = gh_det_row(det, m.x, m.y, id, tx, ty, gx);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            row[0] = z; row[1] = z; row[2] = z; row[3] = z;
        }
    }
    if (nchunks == 0) return;
    // staging slots per thread; the last one may be partial when the window is not a multiple of 128
    constexpr int PER_THREAD = (GH_BWD_CHUNK + GH_BWD_THREADS - 1) / GH_BWD_THREADS;

    // ---- stage the last window (windows are visited last to first) and build its lists
    uint32_t next_id[PER_THREAD];
    {
        const int base = (nchunks - 1) * GH_BWD_CHUNK;
        const int cnt = n - base;
#pragma unroll
        for (int h = 0; h < PER_THREAD; h++) {
            const int slot = tid + h * GH_BWD_THREADS;
            if (slot < cnt) {
                const uint32_t id = (uint32_t)inst[(size_t)rg.x + base + slot];
                gh_stage_issue(st, slot, id, geo, features);
                st.id[slot] = id;
            }
        }
        gh_cp_async_commit();
        if (nchunks > 1) {
#pragma unroll
            for (int h = 0; h < PER_THREAD; h++)
                if (tid + h * GH_BWD_THREADS < GH_BWD_CHUNK)
                    next_id[h] = (uint32_t)inst[(size_t)rg.x + base - GH_BWD_CHUNK + tid + h * GH_BWD_THREADS];
        }
        gh_cp_async_wait_all();
        __syncthreads();
        for (int word = warp; word * 32 < cnt; word += GH_BWD_THREADS / 32)
            gh_build_lists_b(st, cnt, word, lane, tx0, ty0, base, s_glast[lane], s_glast[32 + lane]);
        __syncthreads();
    }

    // ---- block -> (warp, lane pair) assignment.  The blocks of a warp advance in lock-step, so a warp pays for
    // its LONGEST list: blocks are ranked by the length of their list in the window just built (lane b counts blocks
    // b and 32 + b; every warp computes the same ranking for itself) and each warp takes 16 neighbours of that
    // ranking.  Any assignment gives the same gradients up to the order of the float atomics.
    int blk;
    if constexpr (DET) {
        blk = 16 * warp + lane / 2;           // natural order: a warp's 16 blocks are neighbours, their lists overlap
    } else {
        const int nw = (n - (nchunks - 1) * GH_BWD_CHUNK + 31) >> 5;
        uint32_t len0 = 0, len1 = 0;
        for (int w = 0; w < nw; w++) {
            len0 += __popc(st.bits[lane][w]);
            len1 += __popc(st.bits[32 + lane][w]);
        }
        const uint32_t key0 = (len0 << 6) | (uint32_t)lane, key1 = (len1 << 6) | (uint32_t)(32 + lane);
        int rank0 = 0, rank1 = 0;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const uint32_t a = __shfl_sync(0xffffffffu, key0, k);
            const uint32_t b = __shfl_sync(0xffffffffu, key1, k);
            rank0 += ((a < key0) ? 1 : 0) + ((b < key0) ? 1 : 0);
            rank1 += ((a < key1) ? 1 : 0) + ((b < key1) ? 1 : 0);
        }
        s_perm[warp][rank0] = (uint8_t)lane;
        s_perm[warp][rank1] = (uint8_t)(32 + lane);
        __syncwarp();
        blk = s_perm[warp][16 * warp + lane / 2];
    }
    const int px = tx * GH_BLOCK_X + 2 * (blk % 8) + (lane % 2);
    const int py0 = ty * GH_BLOCK_Y + 2 * (blk / 8);
    const float pxf = (float)px;

    GhBwdPair pr;
    {
        float tf[2], bgd[2];
        uint32_t lastv[2];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const int py = py0 + r;
            const bool inside = (px < W) && (py < H);
            const size_t pi = (size_t)py * W + px;
            tf[r] = inside ? final_T[pi] : 0.f;
            lastv[r] = inside ? n_contrib[pi] : 0u;     // pixel blends list positions 1..last
            float d[GH_NUM_CHANNELS];
            bgd[r] = 0.f;
#pragma unroll
            for (int ch = 0; ch < GH_NUM_CHANNELS; ch++) {
                d[ch] = inside ? dL_dpix[ch * plane + pi] : 0.f;
                bgd[r] += __ldg(bg + ch) * d[ch];
            }
#pragma unroll
            for (int k = 0; k < GH_HALF_C; k++) {
                if (r == 0) pr.dL0[k] = make_float2(d[2 * k], d[2 * k + 1]);
                else pr.dL1[k] = make_float2(d[2 * k], d[2 * k + 1]);
            }
        }
        pr.T = make_float2(tf[0], tf[1]);
        pr.ntf_bg = make_float2(-tf[0] * bgd[0], -tf[1] * bgd[1]);
        pr.npy = make_float2(-(float)py0, -(float)(py0 + 1));
        pr.A = gh_f2(0.f); pr.last_alpha = gh_f2(0.f); pr.last_cdot = gh_f2(0.f);
        pr.last0 = lastv[0]; pr.last1 = lastv[1];
    }
    // pixel-coordinate -> NDC chain rule factors (backward.cu:464-465), negated for gh_bwd_pair
    const float nddelx_dx = -0.5f * W, nddely_dy = -0.5f * H;

    uint32_t wlast = s_glast[blk];
#pragma unroll
    for (int o = 2; o < 32; o <<= 1) wlast = max(wlast, __shfl_xor_sync(0xffffffffu, wlast, o));

    for (int c = nchunks - 1; c >= 0; c--) {
        const int base = c * GH_BWD_CHUNK;
        const int cnt = min(GH_BWD_CHUNK, n - base);
        if (c != nchunks - 1) {
            __syncthreads();                       // everyone is done with the previous window
#pragma unroll
            for (int h = 0; h < PER_THREAD; h++) {
                const int slot = tid + h * GH_BWD_THREADS;
                if (slot < GH_BWD_CHUNK) {
                    gh_stage_issue(st, slot, next_id[h], geo, features);
                    st.id[slot] = next_id[h];
                }
            }
            gh_cp_async_commit();
            if (c > 0) {
#pragma unroll
                for (int h = 0; h < PER_THREAD; h++)
                    if (tid + h * GH_BWD_THREADS < GH_BWD_CHUNK)
                        next_id[h] = (uint32_t)inst[(size_t)rg.x + base - GH_BWD_CHUNK + tid + h * GH_BWD_THREADS];
            }
            gh_cp_async_wait_all();
            __syncthreads();
            // per-block lists: each of the 4 warps scan-converts every fourth batch of 32 Gaussians
            for (int word = warp; word * 32 < cnt; word += GH_BWD_THREADS / 32)
                gh_build_lists_b(st, cnt, word, lane, tx0, ty0, base, s_glast[lane], s_glast[32 + lane]);
            __syncthreads();
        }
        if constexpr (DET) {
            // Word by word, back to front: the warp walks the UNION of its 16 blocks' hit words, so at each step all
            // blocks evaluate the same Gaussian (a block that does not list it runs with pos = UINT_MAX: exact zeros,
            // state kept).  Its 16 components are summed over the block's 2 lanes, then over the 16 blocks by a fixed
            // butterfly, and stored as the warp's partial; after a barrier the 4 warps are summed in warp order and
            // the tile's partial leaves as one row per instance.  Every sum has a fixed order.
            const bool walk = (uint32_t)base < wlast;
            float4* wpart = reinterpret_cast<float4*>(gh_bwd_smem + sizeof(GhStageB));   // [warp][record][quad]
            float4* mine_part = wpart + warp * 32 * 4;
            for (int wi = ((cnt + 31) >> 5) - 1; wi >= 0; wi--) {
#pragma unroll
                for (int i = 0; i < 4; i++) mine_part[lane + 32 * i] = make_float4(0.f, 0.f, 0.f, 0.f);
                const uint32_t mine = walk ? st.bits[blk][wi] : 0u;
                uint32_t uni = __reduce_or_sync(0xffffffffu, mine);
                __syncwarp();
                while (uni != 0u) {
                    const int bpos = 31 - __clz(uni);
                    uni &= ~(1u << bpos);
                    const int jj = wi * 32 + bpos;
                    const float4 g0 = st.g0[jj], g1 = st.g1[jj];
                    const uint32_t pos = ((mine >> bpos) & 1u) ? (uint32_t)(base + jj) : 0xffffffffu;
                    float v[16];
                    const bool contrib = gh_bwd_pair(pr, g0, g1, &st.feat[jj * GH_HALF_C], pxf, pos, nddelx_dx, nddely_dy, v);
                    if (!__any_sync(0xffffffffu, contrib)) continue;     // the record stays zero
                    float4 s0, s1;
                    gh_group2_reduce16(v, lane, s0, s1);
#pragma unroll
                    for (int o = 2; o < 32; o <<= 1) {
                        s0.x += __shfl_xor_sync(0xffffffffu, s0.x, o); s0.y += __shfl_xor_sync(0xffffffffu, s0.y, o);
                        s0.z += __shfl_xor_sync(0xffffffffu, s0.z, o); s0.w += __shfl_xor_sync(0xffffffffu, s0.w, o);
                        s1.x += __shfl_xor_sync(0xffffffffu, s1.x, o); s1.y += __shfl_xor_sync(0xffffffffu, s1.y, o);
                        s1.z += __shfl_xor_sync(0xffffffffu, s1.z, o); s1.w += __shfl_xor_sync(0xffffffffu, s1.w, o);
                    }
                    if (lane < 2) {                  // components 0..3, 8..11 (lane 0) / 4..7, 12..15 (lane 1)
                        mine_part[bpos * 4 + lane] = s0;
                        mine_part[bpos * 4 + 2 + lane] = s1;
                    }
                }
                __syncthreads();
                {
                    const int r = tid >> 2, q = tid & 3, jj = wi * 32 + r;
                    if (jj < cnt) {
                        float4 a = wpart[r * 4 + q];
#pragma unroll
                        for (int w = 1; w < GH_BWD_THREADS / 32; w++) {
                            const float4 b = wpart[(w * 32 + r) * 4 + q];
                            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
                        }
                        const float4 g0 = st.g0[jj];
                        gh_det_row(det, g0.x, g0.y, st.id[jj], tx, ty, gx)[q] = a;
                    }
                }
                __syncthreads();
            }
            continue;
        }
        if ((uint32_t)base >= wlast) continue;

        int wi = (cnt + 31) >> 5;
        uint32_t cur = 0;
        while (true) {
            while (cur == 0 && wi > 0) cur = st.bits[blk][--wi];
            const bool act = (cur != 0);
            if (!__any_sync(0xffffffffu, act)) break;

            // blocks whose list is exhausted run the same code on slot 0 with pos = UINT_MAX (-> all zeros)
            const int bpos = act ? 31 - __clz(cur) : 0;   // back to front
            cur &= ~(1u << bpos);
            const int jj = act ? wi * 32 + bpos : 0;
            const uint32_t id = st.id[jj];
            const float4 g0 = st.g0[jj], g1 = st.g1[jj];
            const float2* feat = &st.feat[jj * GH_HALF_C];
            const uint32_t pos = act ? (uint32_t)(base + jj) : 0xffffffffu;
            float v[16];
            const bool contrib = gh_bwd_pair(pr, g0, g1, feat, pxf, pos, nddelx_dx, nddely_dy, v);
            const uint32_t cm = __ballot_sync(0xffffffffu, contrib);
            if (cm == 0u) continue;
            float4 s0, s1;
            gh_group2_reduce16(v, lane, s0, s1);
            // a block issues its reductions when either of its two lanes contributed; GH_ABLATE_REDG: the sums are
            // still formed, the reductions are not issued
            if (GH_ABLATE_REDG ? (s0.x == -1.5e-38f) : ((cm >> (lane & 30)) & 3u)) {
                float4* dst = reinterpret_cast<float4*>(acc16 + (size_t)id * 16) + (lane & 1);
                atomicAdd(dst, s0);       // REDG.E.ADD.F32x4: components 0..3 / 4..7
                atomicAdd(dst + 2, s1);   //                              8..11 / 12..15
            }
        }
    }
    gh_cp_async_wait_all();
}

// ---------------------------------------------------------------------------- gradient unpack
// acc16 -> the reference binding's layouts (rasterize_points.cu:160-168): dL_dcolor (P,10),
// dL_dmean2D (P,3) [z never written by the reference: 0], dL_dconic (P,2,2) [.z unused: 0], dL_dopacity (P,1)
__global__ void __launch_bounds__(256)
gh_unpack_grads_kernel(int P, const float* __restrict__ acc16, float* __restrict__ dL_dmean2D,
                       float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor,
                       float* __restrict__ dL_dmean3D, float* __restrict__ dL_dcov3D,
                       float* __restrict__ dL_dscale, float* __restrict__ dL_drot)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    gh_pdl_wait();                                    // acc16 comes from the blend backward
    gh_pdl_trigger();
    const float4* a = reinterpret_cast<const float4*>(acc16 + (size_t)idx * 16);
    const float4 a0 = a[0], a1 = a[1], a2 = a[2], a3 = a[3];
    float2* dc = reinterpret_cast<float2*>(dL_dcolor + (size_t)idx * GH_NUM_CHANNELS);
    dc[0] = make_float2(a0.x, a0.y); dc[1] = make_float2(a0.z, a0.w);
    dc[2] = make_float2(a1.x, a1.y); dc[3] = make_float2(a1.z, a1.w);
    dc[4] = make_float2(a2.x, a2.y);
    dL_dmean2D[3 * idx + 0] = a2.z; dL_dmean2D[3 * idx + 1] = a2.w; dL_dmean2D[3 * idx + 2] = 0.f;
    reinterpret_cast<float4*>(dL_dconic)[idx] = make_float4(a3.x, a3.y, 0.f, a3.z);
    dL_dopacity[idx] = a3.w;
    // conic supplied by the caller: nothing flows through the geometry (reference backward.cu:371,398,588)
    if (dL_dmean3D) { dL_dmean3D[3 * idx + 0] = 0.f; dL_dmean3D[3 * idx + 1] = 0.f; dL_dmean3D[3 * idx + 2] = 0.f; }
    if (dL_dcov3D) {
#pragma unroll
        for (int k = 0; k < 6; k++) dL_dcov3D[6 * idx + k] = 0.f;
    }
    if (dL_dscale) { dL_dscale[3 * idx + 0] = 0.f; dL_dscale[3 * idx + 1] = 0.f; dL_dscale[3 * idx + 2] = 0.f; }
    if (dL_drot) reinterpret_cast<float4*>(dL_drot)[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---------------------------------------------------------------------------- deterministic backward: rows
// Offsets of the Gaussian-major rows: off = exclusive prefix sum of the tile-rectangle areas (emit's rectangles:
// 0 for radius <= 0), in three launches -- per-CTA sums, one CTA scanning those, per-CTA scans plus their offset.
__device__ __forceinline__ uint32_t gh_det_area(int i, int P, const GhGeo* __restrict__ geo, const int* __restrict__ radii,
                                                int gx, int gy) {
    if (i >= P) return 0u;
    const int r = radii[i];
    if (r <= 0) return 0u;
    const float2 m = *reinterpret_cast<const float2*>(geo + i);
    int minx, miny, maxx, maxy;
    gh_get_rect(m.x, m.y, r, gx, gy, minx, miny, maxx, maxy);
    return (uint32_t)((maxx - minx) * (maxy - miny));
}

// exclusive scan of one value per thread over a 256-thread CTA; returns the CTA total through `total`
__device__ __forceinline__ uint32_t gh_cta_scan256(uint32_t v, uint32_t* s_warp, uint32_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t nb = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += nb; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) { const uint32_t s = s_warp[w]; before += (w < warp) ? s : 0u; total += s; }
    __syncthreads();
    return before + x - v;
}

__global__ void __launch_bounds__(256)
gh_det_area_sums_kernel(int P, const GhGeo* __restrict__ geo, const int* __restrict__ radii, int gx, int gy,
                        uint32_t* __restrict__ part)
{
    __shared__ uint32_t s_warp[8];
    const int i0 = blockIdx.x * GH_DET_SCAN_ITEMS + threadIdx.x * 4;
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) s += gh_det_area(i0 + k, P, geo, radii, gx, gy);
    uint32_t total;
    gh_cta_scan256(s, s_warp, total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256)
gh_det_part_scan_kernel(int nb, int P, uint32_t* __restrict__ part, uint32_t* __restrict__ off)
{
    __shared__ uint32_t s_warp[8];
    uint32_t carry = 0;
    for (int b0 = 0; b0 < nb; b0 += 256) {
        const int b = b0 + (int)threadIdx.x;
        const uint32_t v = (b < nb) ? part[b] : 0u;
        uint32_t total;
        const uint32_t ex = gh_cta_scan256(v, s_warp, total);
        if (b < nb) part[b] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) off[P] = carry;       // = R
}

__global__ void __launch_bounds__(256)
gh_det_offsets_kernel(int P, const GhGeo* __restrict__ geo, const int* __restrict__ radii, int gx, int gy,
                      const uint32_t* __restrict__ part, uint32_t* __restrict__ off)
{
    __shared__ uint32_t s_warp[8];
    const int i0 = blockIdx.x * GH_DET_SCAN_ITEMS + threadIdx.x * 4;
    uint32_t a[4], s = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { a[k] = gh_det_area(i0 + k, P, geo, radii, gx, gy); s += a[k]; }
    uint32_t total;
    uint32_t run = part[blockIdx.x] + gh_cta_scan256(s, s_warp, total);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (i0 + k < P) off[i0 + k] = run;
        run += a[k];
    }
}

// acc16[i] = sum of rows off[i] .. off[i+1] in row order (4 threads per Gaussian, one float4 quad each); assigns every
// record, so no clearing pass is needed
__global__ void __launch_bounds__(256)
gh_det_gather_kernel(int P, const uint32_t* __restrict__ off, const float4* __restrict__ rows, float4* __restrict__ acc16)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t i = t >> 2;
    const int q = (int)(t & 3);
    if (i >= (size_t)P) return;
    const uint32_t r0 = off[i], r1 = off[i + 1];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t r = r0; r < r1; r++) {
        const float4 b = rows[4 * (size_t)r + q];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    acc16[4 * i + q] = a;
}

// The shared-memory attributes of a blend kernel, set once per device (bit `dev` of `devices`; devices past 63 set them
// on every launch): the forward's launch sits on the host's path from the read-back of R to the GPU's next work, where
// each runtime call is time the GPU may spend waiting.
template <typename Kernel>
void gh_blend_smem_once(Kernel kernel, int smem, std::atomic<unsigned long long>& devices)
{
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
    if (devices.load(std::memory_order_relaxed) & bit) return;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
        cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100) == cudaSuccess)
        devices.fetch_or(bit);
}
std::atomic<unsigned long long> g_fwd_smem_set{0}, g_bwd_smem_set{0}, g_bwd_det_smem_set{0};

}  // namespace

void gh_launch_blend_forward(int W, int H, int gx, int gy, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                             const float* features, const float* bg, float* out_color,
                             int P, bool zero_records, cudaStream_t stream)
{
    // 6 CTAs of 128 threads per SM: 34 KB of dynamic shared memory each (the in-CTA sort's buffers, the largest use)
    // out of the largest carve-out
    const int smem = (int)kFwdSmemBytes;
    gh_blend_smem_once(gh_blend_forward_kernel, smem, g_fwd_smem_set);
    gh_launch_pdl(gh_blend_forward_kernel, gx * gy, GH_FWD_THREADS, smem, stream,
                  img.ranges, img.tile_perm, bin.inst, geom.geo, features, W, H, gx, bg, img.final_T, img.n_contrib,
                  out_color, zero_records ? reinterpret_cast<float4*>(geom.acc16) : nullptr, (size_t)P * 4);
}

void gh_launch_blend_backward(int W, int H, int gx, int gy, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                              const float* features, const float* bg, const float* dL_dpix,
                              cudaStream_t stream)
{
    const int smem = (int)sizeof(GhStageB);
    gh_blend_smem_once(gh_blend_backward_kernel<false>, smem, g_bwd_smem_set);
    gh_launch_pdl(gh_blend_backward_kernel<false>, gx * gy, GH_BWD_THREADS, smem, stream,
                  img.ranges, img.tile_perm, bin.inst, geom.geo, features, W, H, gx, bg, img.final_T, img.n_contrib,
                  dL_dpix, geom.acc16, GhDetArgs{});
}

int gh_launch_det_offsets(int P, int gx, int gy, const int* radii, GhGeomWS geom, GhDetWS det, cudaStream_t stream)
{
    const int nb = (int)GhDetWS::scan_blocks((size_t)P);
    gh_det_area_sums_kernel<<<nb, 256, 0, stream>>>(P, geom.geo, radii, gx, gy, det.part);
    gh_det_part_scan_kernel<<<1, 256, 0, stream>>>(nb, P, det.part, det.off);
    gh_det_offsets_kernel<<<nb, 256, 0, stream>>>(P, geom.geo, radii, gx, gy, det.part, det.off);
    return 3;
}

void gh_launch_blend_backward_det(int W, int H, int gx, int gy, const int* radii, GhGeomWS geom, GhImgWS img, GhBinWS bin,
                                  GhDetWS det, const float* features, const float* bg, const float* dL_dpix,
                                  cudaStream_t stream)
{
    const int smem = (int)(sizeof(GhStageB) + kBwdDetPartBytes);
    gh_blend_smem_once(gh_blend_backward_kernel<true>, smem, g_bwd_det_smem_set);
    const GhDetArgs d{radii, det.off, reinterpret_cast<float4*>(det.rows), gy};
    gh_blend_backward_kernel<true><<<gx * gy, GH_BWD_THREADS, smem, stream>>>(img.ranges, img.tile_perm, bin.inst, geom.geo, features,
                                                         W, H, gx, bg, img.final_T, img.n_contrib, dL_dpix,
                                                         nullptr, d);
}

void gh_launch_det_gather(int P, GhGeomWS geom, GhDetWS det, cudaStream_t stream)
{
    const long long threads = 4ll * P;
    gh_det_gather_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(
        P, det.off, reinterpret_cast<const float4*>(det.rows), reinterpret_cast<float4*>(geom.acc16));
}

void gh_launch_unpack_grads(int P, GhGeomWS geom, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                            float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot,
                            cudaStream_t stream)
{
    gh_launch_pdl(gh_unpack_grads_kernel, (P + 255) / 256, 256, 0, stream,
                  P, geom.acc16, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot);
}
