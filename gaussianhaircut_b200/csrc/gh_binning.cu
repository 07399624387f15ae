// Stage 2: binning.  Produces, per 16x16 tile, the list of Gaussian instances overlapping it,
// ordered by the reference's 64-bit key  (tile_id << 32) | float_bits(depth)  with ties broken by
// ascending Gaussian index -- exactly the order the reference obtains from duplicateWithKeys +
// a stable cub::DeviceRadixSort::SortPairs over bits [0, 32+bit) + identifyTileRanges
// (rasterizer_impl.cu:70-138, 293-321).
//
// New design (no multi-pass device-wide radix sort): the tile id is an exact bucket, so
//   1. stage 1 already histogrammed instances per tile;
//   2. one block scans the histogram -> tile ranges (= identifyTileRanges' output) and R;
//   3. each Gaussian scatters (depth_bits << 32 | idx) into its tiles' buckets (atomic cursor);
//   4. each bucket is sorted in shared memory on the composite 64-bit (depth, idx) key, which
//      reproduces the stable order because a Gaussian appears at most once per tile.
// HBM traffic is 8 B write + 8 B read + 8 B write per instance instead of ~156 B for 6 radix passes.
#include <cooperative_groups.h>
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

namespace {

// ---------------------------------------------------------------- tile scan (one cluster of 8 CTAs)
// Exclusive scan of the per-tile histogram -> bucket cursors + tile ranges, the totals, and the launch order of
// the blend kernels.  The problem is tiny (T = 8160 tiles at 1080p) and sits on the critical path between two
// kernels, so what matters is latency and the store bandwidth of the SMs that take part: ONE thread-block cluster
// of 8 CTAs (8 SMs) shares the work, exchanging CTA totals, bucket histograms and the maximum through distributed
// shared memory instead of a second launch.  Every tile count is loaded once per pass with two 128-bit loads per
// thread and all later phases work from registers.
#define GH_SCAN_CTAS 8
#define GH_SCAN_THREADS 256
#define GH_SCAN_ROUND (GH_SCAN_CTAS * GH_SCAN_THREADS * 8)      // tiles per cluster round

__device__ __forceinline__ void gh_load_counts8(const uint32_t* __restrict__ tile_count, int i0, int T, uint32_t (&c)[8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) c[k] = 0u;
    if (i0 + 8 <= T) {     // 32-byte aligned: two 128-bit loads
        const uint4 a = reinterpret_cast<const uint4*>(tile_count + i0)[0], b = reinterpret_cast<const uint4*>(tile_count + i0)[1];
        c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = a.w; c[4] = b.x; c[5] = b.y; c[6] = b.z; c[7] = b.w;
    } else {
        for (int k = 0; k < 8; k++) if (i0 + k < T) c[k] = tile_count[i0 + k];
    }
}

__device__ __forceinline__ int gh_len_bucket(uint32_t count) { return (int)(127u - min(127u, count >> 4)); }

__global__ void __cluster_dims__(GH_SCAN_CTAS, 1, 1) __launch_bounds__(GH_SCAN_THREADS)
gh_tile_scan_kernel(int T, const uint32_t* __restrict__ tile_count, uint32_t* __restrict__ tile_cursor,
                    uint2* __restrict__ ranges, uint32_t* __restrict__ tile_perm, GhCtrl* __restrict__ ctrl)
{
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    constexpr int NW = GH_SCAN_THREADS / 32;
    __shared__ uint32_t warp_sums[NW];
    __shared__ uint32_t s_cta_total[2];         // this CTA's sum of the current round (double-buffered by round parity)
    __shared__ uint32_t s_cta_max;
    // Launch order of the blend kernels: a counting sort of the tiles by list length, longest first
    // (LPT scheduling: the ~14 waves of tile CTAs end together instead of waiting for a late heavy tile; the
    // empty tiles, ~40% at the benchmark view, run last and only write background).  128 buckets of 16 records.
    __shared__ uint32_t s_hist[128];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const unsigned rank = cluster.block_rank();
    if (tid < 128) s_hist[tid] = 0u;
    gh_pdl_wait();                              // tile_count is the preprocess kernel's histogram
    gh_pdl_trigger();
    uint32_t tmax = 0, carry = 0;
    __syncthreads();
    int round = 0;
    for (int base = 0; base < T; base += GH_SCAN_ROUND, round++) {
        const int i0 = base + ((int)rank * GH_SCAN_THREADS + tid) * 8;
        uint32_t c[8];
        gh_load_counts8(tile_count, i0, T, c);
        uint32_t sum = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { sum += c[k]; tmax = max(tmax, c[k]); }
        uint32_t v = sum;   // inclusive warp scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t nb = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += nb; }
        if (lane == 31) warp_sums[wid] = v;
        // histogram of list-length buckets.  Neighbouring tiles mostly share a bucket (the empty ones, ~40%, all
        // do): a thread adds each RUN of equal buckets among its 8 tiles with one shared-memory atomic
        {
            int bkt[8];
#pragma unroll
            for (int k = 0; k < 8; k++) bkt[k] = (i0 + k < T) ? gh_len_bucket(c[k]) : -1;
            uint32_t len = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                len++;
                const bool last = (k == 7) || (bkt[k + 1 < 8 ? k + 1 : 7] != bkt[k]);
                if (last) { if (bkt[k] >= 0) atomicAdd(&s_hist[bkt[k]], len); len = 0; }
            }
        }
        __syncthreads();
        uint32_t before = 0, cta_sum = 0;          // sum of the warps before mine / of the CTA
#pragma unroll
        for (int w = 0; w < NW; w++) { const uint32_t ws = warp_sums[w]; before += (w < wid) ? ws : 0u; cta_sum += ws; }
        if (tid == 0) s_cta_total[round & 1] = cta_sum;
        cluster.sync();                            // totals of all 8 CTAs visible (also orders the warp_sums reuse)
        uint32_t cta_before = 0, round_sum = 0;
#pragma unroll
        for (unsigned r = 0; r < GH_SCAN_CTAS; r++) {
            const uint32_t t = cluster.map_shared_rank(s_cta_total, r)[round & 1];
            cta_before += (r < rank) ? t : 0u;
            round_sum += t;
        }
        uint32_t run = carry + cta_before + before + (v - sum);
        carry += round_sum;
        uint32_t cur8[8];
        uint2 rg8[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            cur8[k] = run;
            // empty tiles keep (0,0) like the reference's memset + identifyTileRanges
            rg8[k] = (c[k] > 0) ? make_uint2(run, run + c[k]) : make_uint2(0u, 0u);
            run += c[k];
        }
        if (i0 + 8 <= T) {
            uint4* cp = reinterpret_cast<uint4*>(tile_cursor + i0);
            cp[0] = make_uint4(cur8[0], cur8[1], cur8[2], cur8[3]);
            cp[1] = make_uint4(cur8[4], cur8[5], cur8[6], cur8[7]);
            uint4* rp = reinterpret_cast<uint4*>(ranges + i0);
#pragma unroll
            for (int k = 0; k < 4; k++) rp[k] = make_uint4(rg8[2 * k].x, rg8[2 * k].y, rg8[2 * k + 1].x, rg8[2 * k + 1].y);
        } else {
            for (int k = 0; k < 8; k++) if (i0 + k < T) { tile_cursor[i0 + k] = cur8[k]; ranges[i0 + k] = rg8[k]; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
    if (lane == 0) warp_sums[wid] = tmax;          // (every thread is past the last round's cluster.sync)
    __syncthreads();
    if (tid == 0) {
        uint32_t m = 0;
        for (int w = 0; w < NW; w++) m = max(m, warp_sums[w]);
        s_cta_max = m;
    }
    cluster.sync();                                // histograms and maxima of all CTAs complete
    if (rank == 0 && tid == 0) {
        uint32_t m = 0;
        for (unsigned r = 0; r < GH_SCAN_CTAS; r++) m = max(m, *cluster.map_shared_rank(&s_cta_max, r));
        ctrl->num_rendered = carry;
        ctrl->max_tile_len = m;
    }
    // first slot of (bucket, this CTA) in the permutation: buckets in descending-length order, CTAs by rank inside
    uint32_t mine_before = 0, bucket_total = 0;
    if (tid < 128) {
#pragma unroll
        for (unsigned r = 0; r < GH_SCAN_CTAS; r++) {
            const uint32_t h = cluster.map_shared_rank(s_hist, r)[tid];
            mine_before += (r < rank) ? h : 0u;
            bucket_total += h;
        }
    }
    cluster.sync();                                // everyone has read the histograms: they become cursors now
    if (tid < 128) {                               // exclusive scan of the 128 bucket totals (4 warps)
        uint32_t v = bucket_total;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t nb = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += nb; }
        if (lane == 31) warp_sums[wid] = v;
        s_hist[tid] = v - bucket_total + mine_before;
    }
    __syncthreads();
    if (tid < 128) {
        uint32_t before = 0;
#pragma unroll
        for (int w = 0; w < 4; w++) before += (w < wid) ? warp_sums[w] : 0u;
        s_hist[tid] += before;
    }
    __syncthreads();
    for (int base = 0; base < T; base += GH_SCAN_ROUND) {
        const int i0 = base + ((int)rank * GH_SCAN_THREADS + tid) * 8;
        uint32_t c[8];
        gh_load_counts8(tile_count, i0, T, c);       // L1 / L2 hit
        int bkt[8];
        uint32_t rl[8], pos[8];
#pragma unroll
        for (int k = 0; k < 8; k++) bkt[k] = (i0 + k < T) ? gh_len_bucket(c[k]) : -1;
        rl[7] = 1;
#pragma unroll
        for (int k = 6; k >= 0; k--) rl[k] = (bkt[k] == bkt[k + 1]) ? rl[k + 1] + 1 : 1;   // length of the run starting at k
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const bool first = (k == 0) || (bkt[k > 0 ? k - 1 : 0] != bkt[k]);
            pos[k] = 0;
            if (first && bkt[k] >= 0) pos[k] = atomicAdd(&s_hist[bkt[k]], rl[k]);     // independent reservations
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (k > 0 && bkt[k - (k > 0 ? 1 : 0)] == bkt[k]) pos[k] = pos[k - (k > 0 ? 1 : 0)] + 1;
            if (bkt[k] >= 0) tile_perm[pos[k]] = (uint32_t)(i0 + k);
        }
    }
}

// ---------------------------------------------------------------- emit
// Consecutive Gaussians of a strand fall into the same tiles, so the lanes of a warp mostly ask for
// slots of the same few buckets: lanes that want the same tile in the same loop step are grouped
// with match.any and their leader reserves all their slots with ONE atomic.
// `capacity`: records the instance buffer holds.  The forward's first phase may launch emit before the host has read R
// back (the binning buffer of gh_forward_preprocess): when R = ctrl->num_rendered exceeds the capacity, no thread writes anything and the
// tile cursors stay as the scan left them, so the host can launch emit again into a buffer of the exact size.
__global__ void __launch_bounds__(256)
gh_emit_kernel(int P, const int* __restrict__ radii, const GhGeo* __restrict__ geo,
               const float* __restrict__ depth, uint32_t* __restrict__ tile_cursor,
               uint64_t* __restrict__ inst, int gx, int gy, const GhCtrl* __restrict__ ctrl, uint32_t capacity)
{
    gh_pdl_wait();                                 // every input comes from the preprocess kernel and the scan
    gh_pdl_trigger();
    if (ctrl->num_rendered > capacity) return;     // uniform over the grid
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int minx = 0, miny = 0, maxx = 0, maxy = 0;
    uint64_t rec = 0;
    if (idx < P) {
        const int r = radii[idx];
        if (r > 0) {
            const float4 g0 = reinterpret_cast<const float4*>(geo + idx)[0];
            gh_get_rect(g0.x, g0.y, r, gx, gy, minx, miny, maxx, maxy);
            rec = ((uint64_t)__float_as_uint(depth[idx]) << 32) | (uint32_t)idx;
        }
    }
    // the warp walks the flattened list of its (Gaussian, tile) instances, GH_EMIT_U x 32 items per round: the slot
    // reservations of a round are independent atomics, so their L2 round trips overlap instead of adding up
    const GhWarpRects wr = gh_warp_rects(minx, miny, maxx, maxy, lane);
    const uint32_t rec_hi = (uint32_t)(rec >> 32);
    const uint32_t idx0 = (uint32_t)(idx - lane);
    constexpr int GH_EMIT_U = 2;
    for (int j0 = 0; j0 < wr.total; j0 += 32 * GH_EMIT_U) {
        int tile[GH_EMIT_U];
        uint32_t peers[GH_EMIT_U], base[GH_EMIT_U], key_hi[GH_EMIT_U], key_lo[GH_EMIT_U];
#pragma unroll
        for (int u = 0; u < GH_EMIT_U; u++) {
            int owner;
            tile[u] = gh_warp_rect_item(wr, j0 + 32 * u + lane, gx, owner);
            key_hi[u] = __shfl_sync(0xffffffffu, rec_hi, owner);
            key_lo[u] = idx0 + (uint32_t)owner;
        }
#pragma unroll
        for (int u = 0; u < GH_EMIT_U; u++) peers[u] = __match_any_sync(0xffffffffu, tile[u]);
#pragma unroll
        for (int u = 0; u < GH_EMIT_U; u++) {
            base[u] = 0;
            if (tile[u] >= 0 && lane == __ffs(peers[u]) - 1)
                base[u] = atomicAdd(&tile_cursor[tile[u]], (uint32_t)__popc(peers[u]));
        }
#pragma unroll
        for (int u = 0; u < GH_EMIT_U; u++) {
            const uint32_t b = __shfl_sync(0xffffffffu, base[u], __ffs(peers[u]) - 1);
            if (tile[u] >= 0)
                inst[b + __popc(peers[u] & ((1u << lane) - 1u))] = ((uint64_t)key_hi[u] << 32) | key_lo[u];
        }
    }
}

// ---------------------------------------------------------------- per-tile sort (network in gh_common.cuh)
// Long lists (more than GH_INKERNEL_SORT_MAX records in a tile; the forward CTA sorts shorter ones
// itself) are sorted in linear time by two kernels:
//   split: one 256-thread CTA per long tile finds the depth range of the list, splits it (MSD, order
//          preserving) into segments of ~768 records by linearly quantised depth, scatters the records
//          into the scratch buffer segment by segment and appends (start, length) descriptors;
//   sort:  one CTA per segment sorts it in shared memory (gh_bucket_sort_tile) into its final place.
// A segment that still exceeds the shared buffer (heavily clustered depths) uses the in-place network.
#define GH_LONG_MAX_SUPER 1024
__global__ void __launch_bounds__(256)
gh_tile_split_long_kernel(const uint2* __restrict__ ranges, const uint64_t* __restrict__ inst, uint64_t* __restrict__ tmp,
                          uint2* __restrict__ seg, GhCtrl* ctrl, uint32_t lo)
{
    __shared__ uint32_t s_cnt[GH_LONG_MAX_SUPER];
    __shared__ uint32_t s_red[16];
    __shared__ uint32_t s_segbase;
    const uint2 rg = ranges[blockIdx.x];
    const uint32_t n = rg.y - rg.x;
    if (n <= lo) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t* src = inst + rg.x;
    uint64_t* dst = tmp + rg.x;
    uint32_t dmin = 0xffffffffu, dmax = 0u;
    for (uint32_t i = tid; i < n; i += 256) { const uint32_t d = (uint32_t)(src[i] >> 32); dmin = min(dmin, d); dmax = max(dmax, d); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
        dmax = max(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
    }
    if (lane == 0) { s_red[warp] = dmin; s_red[8 + warp] = dmax; }
    const uint32_t nsuper = min((uint32_t)GH_LONG_MAX_SUPER, (n + 767u) / 768u);
    for (uint32_t i = tid; i < nsuper; i += 256) s_cnt[i] = 0u;
    if (tid == 0) s_segbase = atomicAdd(&ctrl->nseg, nsuper);
    __syncthreads();
#pragma unroll
    for (int w = 0; w < 8; w++) { dmin = min(dmin, s_red[w]); dmax = max(dmax, s_red[8 + w]); }
    const float inv = (float)nsuper / ((float)(dmax - dmin) + 1.0f);
    for (uint32_t i = tid; i < n; i += 256) {
        const uint32_t d = (uint32_t)(src[i] >> 32);
        atomicAdd(&s_cnt[min(nsuper - 1u, (uint32_t)((float)(d - dmin) * inv))], 1u);
    }
    __syncthreads();
    {   // exclusive scan of nsuper counts: thread t owns 4 consecutive counters
        uint32_t c[4], sum = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { const uint32_t j = tid * 4 + k; c[k] = j < nsuper ? s_cnt[j] : 0u; sum += c[k]; }
        uint32_t v = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t nb = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += nb; }
        __syncthreads();
        if (lane == 31) s_red[warp] = v;
        __syncthreads();
        uint32_t run = v - sum;
#pragma unroll
        for (int w = 0; w < 8; w++) run += (w < warp) ? s_red[w] : 0u;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t j = tid * 4 + k;
            if (j < nsuper) {
                s_cnt[j] = run;
                seg[s_segbase + j] = make_uint2(rg.x + run, c[k]);
            }
            run += c[k];
        }
    }
    __syncthreads();
    for (uint32_t i = tid; i < n; i += 256) {
        const uint64_t key = src[i];
        const uint32_t d = (uint32_t)(key >> 32);
        dst[atomicAdd(&s_cnt[min(nsuper - 1u, (uint32_t)((float)(d - dmin) * inv))], 1u)] = key;
    }
}

__global__ void __launch_bounds__(256)
gh_segment_sort_kernel(const uint2* __restrict__ seg, const GhCtrl* __restrict__ ctrl, uint64_t* inst, uint64_t* tmp)
{
    __shared__ __align__(16) uint64_t sA[GH_INKERNEL_SORT_MAX];
    __shared__ __align__(16) uint64_t sB[GH_INKERNEL_SORT_MAX];
    __shared__ __align__(16) uint32_t s_small[GH_SORT_SCRATCH_WORDS];
    if (blockIdx.x >= ctrl->nseg) return;
    const uint2 sg = seg[blockIdx.x];
    const uint32_t b0 = sg.x, m = sg.y;
    if (m == 0) return;
    const int tid = threadIdx.x;
    if (m <= GH_INKERNEL_SORT_MAX) {
        for (uint32_t i = tid; i < m; i += 256) sA[i] = tmp[b0 + i];
        __syncthreads();
        if (m <= 64) gh_bitonic_sort(sA, m, tid, 256);
        else gh_bucket_sort_tile<256>(sA, sB, s_small, (int)m, tid);
        for (uint32_t i = tid; i < m; i += 256) inst[b0 + i] = sA[i];
    } else {
        gh_bitonic_sort(tmp + b0, m, tid, 256);
        for (uint32_t i = tid; i < m; i += 256) inst[b0 + i] = tmp[b0 + i];
    }
}

// ---------------------------------------------------------------- capacity guard (capturable forward)
// Runs between the tile scan and emit.  R fits: nothing to do (every CTA leaves after one load of ctrl).  R exceeds the
// capacity of the binning buffer: emit writes nothing (its own test), and this kernel empties the frame -- every tile
// range (0, 0), every radius 0 -- so that the sort, both blend kernels, the deterministic row offsets and the
// densification statistics all see a frame with no instance: background image, zero records, zero gradients.
__global__ void __launch_bounds__(256)
gh_capacity_guard_kernel(int P, int* __restrict__ radii, int T, uint2* __restrict__ ranges, const GhCtrl* __restrict__ ctrl,
                         uint32_t capacity, unsigned int* __restrict__ status, unsigned int* __restrict__ r_out)
{
    const uint32_t R = ctrl->num_rendered;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (r_out) *r_out = R;
        if (R > capacity) atomicOr(status, GH_STATUS_BINNING_OVERFLOW);
    }
    if (R <= capacity) return;
    const int stride = gridDim.x * blockDim.x;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += stride) ranges[i] = make_uint2(0u, 0u);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += stride) radii[i] = 0;
}

}  // namespace

void gh_launch_tile_scan(int T, GhImgWS img, cudaStream_t stream)
{
    gh_launch_pdl(gh_tile_scan_kernel, GH_SCAN_CTAS, GH_SCAN_THREADS, 0, stream,
                  T, img.tile_count, img.tile_cursor, img.ranges, img.tile_perm, img.ctrl);
}

void gh_launch_emit(int P, const int* radii, GhGeomWS geom, GhImgWS img, GhBinWS bin, unsigned int capacity,
                    int gx, int gy, cudaStream_t stream)
{
    gh_launch_pdl(gh_emit_kernel, (P + 255) / 256, 256, 0, stream,
                  P, radii, geom.geo, geom.depth, img.tile_cursor, bin.inst, gx, gy, img.ctrl, capacity);
}

int gh_launch_tile_sort(int T, unsigned int max_tile_len, long long R, GhImgWS img, GhBinWS bin, cudaStream_t stream)
{
    // tiles with at most GH_INKERNEL_SORT_MAX instances are sorted by the forward blend CTA itself
    // (gh_blend.cu); only longer lists need these kernels
    if (max_tile_len <= GH_INKERNEL_SORT_MAX) return 0;
    gh_tile_split_long_kernel<<<T, 256, 0, stream>>>(img.ranges, bin.inst, bin.tmp, bin.seg, img.ctrl, GH_INKERNEL_SORT_MAX);
    const unsigned int nseg_max = (unsigned int)GhBinWS::max_segments((size_t)R);   // >= sum over long tiles of ceil(n/768)
    gh_segment_sort_kernel<<<nseg_max, 256, 0, stream>>>(bin.seg, img.ctrl, bin.inst, bin.tmp);
    return 2;
}

void gh_launch_capacity_guard(int P, int* radii, int T, GhImgWS img, unsigned int capacity, unsigned int* status,
                              unsigned int* num_rendered_out, cudaStream_t stream)
{
    gh_capacity_guard_kernel<<<2 * 132, 256, 0, stream>>>(P, radii, T, img.ranges, img.ctrl, capacity, status, num_rendered_out);
}

int gh_launch_tile_sort_capturable(int T, unsigned int capacity, GhImgWS img, GhBinWS bin, cudaStream_t stream)
{
    // max_tile_len is only known on the device: the split always runs (a CTA whose list is short leaves at once), and the
    // segment sort gets the grid of the largest R that fits (R <= capacity, hence nseg <= max_segments(capacity))
    gh_tile_split_long_kernel<<<T, 256, 0, stream>>>(img.ranges, bin.inst, bin.tmp, bin.seg, img.ctrl, GH_INKERNEL_SORT_MAX);
    const unsigned int nseg_max = (unsigned int)GhBinWS::max_segments((size_t)capacity);
    gh_segment_sort_kernel<<<nseg_max, 256, 0, stream>>>(bin.seg, img.ctrl, bin.inst, bin.tmp);
    return 2;
}
