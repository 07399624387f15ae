// Gradient all-reduce over NVLink peer memory (SURVEY.md 8e: views are sharded one per GPU and the
// per-Gaussian gradients are summed once per step).
//
// One kernel per rank on the step's stream, no NCCL on the data path.  Every rank's gradient arena lives
// in symmetric memory (same allocation on every GPU, all of them mapped into every process), so a rank
// can load from and store to its peers' arenas directly through NVSwitch:
//     entry barrier   "my gradients are complete" flags, release/acquire at system scope
//     two-shot sum    rank r owns slice r of the arena: it reads slice r of every peer (world-1 remote
//                     loads in flight per element), adds, and writes the sum into slice r of EVERY arena
//                     (or, when the allocation has an NVLS multicast mapping, one multimem.ld_reduce and
//                     one multimem.st per 16 bytes: the switch does the reduction and the broadcast)
//     exit barrier    "my stores have landed everywhere" flags; the kernel ends when all peers said so,
//                     so whatever follows on the stream (the optimizer) sees the reduced gradients
// Per GPU and direction the links carry 2 (world-1)/world of the arena (peers reading my copy + my stores
// to them), the same as a ring all-reduce, but in one launch with every pair of GPUs talking at once; the
// multimem path sends each reduced slice only once.
//
// Failure handling: every spin is bounded by WALL-CLOCK time (%globaltimer; default 30 s, GH_ALLREDUCE_TIMEOUT_MS).
// If a peer does not arrive, CTA 0 raises the sticky error word local[2], publishes the epoch as failed
// (local[3]) and every CTA SKIPS the reduction -- nobody sums a peer's unfinished arena.  A CTA whose own
// wait for CTA 0 times out raises the error word as well and skips.  The error word can be handed to
// gh_adam_step as `skip_flag`, so that the optimizer step that follows on the stream does not consume an
// undefined result.  The NaN guard of the optimizer can ride on the reduction: every rank reports whether
// its slice of the SUM holds a NaN, the reports are exchanged with the exit barrier, and `nan_out` ends up
// identical on all ranks.
#include "gh_common.cuh"
#include "gh_kernels.h"
#include "../../include/gh_rasterizer.h"

#include <cstdlib>

namespace {

#define GH_AR_MAX_THREADS 512
#define GH_AR_MAX_WORLD 16

struct GhArPeers {
    float* buf[GH_AR_MAX_WORLD];
    unsigned int* flag[GH_AR_MAX_WORLD];     // per rank: uint[3 * world] = entry flags, exit flags, NaN reports
};

__device__ __forceinline__ void gh_st_release_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void gh_st_relaxed_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int gh_ld_acquire_sys(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned int gh_ld_acquire_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long gh_globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// wait until *p >= epoch (epochs only grow; compare with wrap-around), at most timeout_ns
template <bool SYS>
__device__ __forceinline__ bool gh_spin(const unsigned int* p, unsigned int epoch, unsigned long long timeout_ns) {
    const unsigned long long t0 = gh_globaltimer_ns();
    for (unsigned int it = 0;; it++) {
        const unsigned int v = SYS ? gh_ld_acquire_sys(p) : gh_ld_acquire_gpu(p);
        if ((int)(v - epoch) >= 0) return true;
        if ((it & 63u) == 63u && gh_globaltimer_ns() - t0 > timeout_ns) return false;
        __nanosleep(20);
    }
}

__device__ __forceinline__ bool gh_nan4(const float4 v) { return (v.x != v.x) | (v.y != v.y) | (v.z != v.z) | (v.w != v.w); }

// local[0]: "go" word (entry barrier passed), local[1]: exit arrival counter, local[2]: sticky error word,
// local[3]: last failed epoch, local[4]: NaN seen in my slice during this call
// WORLD_T > 0: world size known at compile time (2, 4, 8) for the peer load/store path: U = 8 / WORLD_T
// elements per thread per round so that 8 remote 16-byte loads are in flight per thread.
// MC_U: 16-byte multimem requests in flight per thread on the NVLS path.
template <int WORLD_T, int MC_U>
__global__ void __launch_bounds__(GH_AR_MAX_THREADS)
gh_allreduce_p2p_kernel(GhArPeers peers, float* __restrict__ mc, int rank, int world_rt, size_t off4, size_t n4,
                        unsigned int epoch, unsigned int* __restrict__ local, unsigned int* __restrict__ nan_out,
                        unsigned long long timeout_ns)
{
    const int world = WORLD_T > 0 ? WORLD_T : world_rt;
    const int tid = threadIdx.x, nt = blockDim.x;
    __shared__ unsigned int s_fail;
    if (tid == 0) s_fail = 0u;
    __syncthreads();
    // ---------------------------------------------------------------- entry barrier
    if (blockIdx.x == 0) {
        if (tid < world) {
            gh_st_release_sys(peers.flag[tid] + rank, epoch);                  // tell peer `tid`: my gradients are final
            if (!gh_spin<true>(peers.flag[rank] + tid, epoch, timeout_ns)) { atomicExch(local + 2, 1u); atomicOr(&s_fail, 1u); }
        }
        __syncthreads();
        if (tid == 0) {
            if (s_fail) atomicExch(local + 3, epoch);      // this epoch failed: the other CTAs must not reduce
            __threadfence();
            atomicExch(local + 0, epoch);
        }
    } else if (tid == 0) {
        // CTA 0 decides; wait a little longer than it does, so that its verdict (not my own timeout) is what I see
        if (!gh_spin<false>(local + 0, epoch, 2ull * timeout_ns + 1000000000ull)) { atomicExch(local + 2, 1u); s_fail = 1u; }
        else if (gh_ld_acquire_gpu(local + 3) == epoch) s_fail = 1u;
    }
    __syncthreads();
    const bool failed = (s_fail != 0u);

    // ---------------------------------------------------------------- my slice: sum over ranks, write everywhere
    bool bad = false;
    if (!failed) {
        const size_t lo = off4 + n4 * (size_t)rank / (size_t)world, hi = off4 + n4 * (size_t)(rank + 1) / (size_t)world;
        const size_t stride = (size_t)gridDim.x * nt;
        if (mc != nullptr) {
            // NVLS: the switch reduces the `world` copies on the load and replicates the store
            float4* m4 = reinterpret_cast<float4*>(mc);
            for (size_t i0 = lo + (size_t)blockIdx.x * nt + tid; i0 < hi; i0 += MC_U * stride) {
                float4 v[MC_U];
#pragma unroll
                for (int u = 0; u < MC_U; u++) {
                    const size_t i = i0 + u * stride;
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (i < hi)
                        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                                     : "=f"(v[u].x), "=f"(v[u].y), "=f"(v[u].z), "=f"(v[u].w) : "l"(m4 + i) : "memory");
                }
#pragma unroll
                for (int u = 0; u < MC_U; u++) {
                    const size_t i = i0 + u * stride;
                    bad |= gh_nan4(v[u]);
                    if (i < hi)
                        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                                     ::"l"(m4 + i), "f"(v[u].x), "f"(v[u].y), "f"(v[u].z), "f"(v[u].w) : "memory");
                }
            }
        } else if (WORLD_T > 0) {
            constexpr int U = WORLD_T > 0 ? (8 / WORLD_T > 0 ? 8 / WORLD_T : 1) : 1;
            for (size_t i0 = lo + (size_t)blockIdx.x * nt + tid; i0 < hi; i0 += U * stride) {
                float4 part[U][WORLD_T > 0 ? WORLD_T : 1];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const size_t i = i0 + u * stride;
#pragma unroll
                    for (int p = 0; p < WORLD_T; p++)
                        part[u][p] = (i < hi) ? __ldcg(reinterpret_cast<const float4*>(peers.buf[p]) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const size_t i = i0 + u * stride;
                    float4 acc = part[u][0];
#pragma unroll
                    for (int p = 1; p < WORLD_T; p++) { acc.x += part[u][p].x; acc.y += part[u][p].y; acc.z += part[u][p].z; acc.w += part[u][p].w; }   // rank order: same bits everywhere
                    bad |= gh_nan4(acc);
                    if (i < hi) {
#pragma unroll
                        for (int p = 0; p < WORLD_T; p++) __stcg(reinterpret_cast<float4*>(peers.buf[p]) + i, acc);
                    }
                }
            }
        } else {
            for (size_t i = lo + (size_t)blockIdx.x * nt + tid; i < hi; i += stride) {
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int p = 0; p < world; p++) {
                    const float4 v = __ldcg(reinterpret_cast<const float4*>(peers.buf[p]) + i);
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                }
                bad |= gh_nan4(acc);
                for (int p = 0; p < world; p++) __stcg(reinterpret_cast<float4*>(peers.buf[p]) + i, acc);
            }
        }
    }

    // ---------------------------------------------------------------- exit barrier
    __threadfence_system();                       // my stores are visible system-wide before I report
    const int any_bad = __syncthreads_or(bad ? 1 : 0);
    __shared__ bool s_last;
    if (tid == 0) {
        if (any_bad) atomicOr(local + 4, 1u);
        __threadfence();
        s_last = (atomicAdd(local + 1, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __shared__ unsigned int s_nan;
    if (tid == 0) {
        __threadfence();
        s_nan = atomicExch(local + 4, 0u);        // every CTA of this launch has reported by now
        local[1] = 0u;
        __threadfence_system();
    }
    __syncthreads();
    unsigned int peer_nan = 0u;
    if (tid < world && !failed) {
        if (s_nan) gh_st_relaxed_sys(peers.flag[tid] + 2 * world + rank, epoch);     // ordered before the release below
        gh_st_release_sys(peers.flag[tid] + world + rank, epoch);
        if (!gh_spin<true>(peers.flag[rank] + world + tid, epoch, timeout_ns)) atomicExch(local + 2, 1u);
        else peer_nan = (gh_ld_acquire_sys(peers.flag[rank] + 2 * world + tid) == epoch) ? 1u : 0u;
    }
    const int nan_any = __syncthreads_or((int)peer_nan);
    if (tid == 0 && nan_out != nullptr) *nan_out = nan_any ? 1u : 0u;
}

int gh_env_int(const char* name, int dflt, int lo, int hi) {
    const char* s = std::getenv(name);
    if (!s || !*s) return dflt;
    const long v = std::strtol(s, nullptr, 10);
    return (int)(v < lo ? lo : (v > hi ? hi : v));
}

}  // namespace

extern "C" int gh_allreduce_p2p(const unsigned long long* peer_bufs, const unsigned long long* peer_flags,
                                unsigned long long multicast_buf, int rank, int world,
                                size_t offset_floats, size_t n_floats, unsigned int epoch,
                                unsigned int* local_sync, unsigned int* nan_out, gh_stream_t stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    gh_clear_error();
    if (!peer_bufs || !peer_flags || !local_sync || world < 1 || world > GH_AR_MAX_WORLD || rank < 0 || rank >= world ||
        (offset_floats & 3) || (n_floats & 3) || epoch == 0)
        return gh_set_error(GH_E_INVALID_ARG, "gh_allreduce_p2p: bad rank/world/epoch, missing pointer, or a range that is not a multiple of 4 floats");
    if (n_floats == 0) return GH_OK;
    GhArPeers peers;
    for (int p = 0; p < GH_AR_MAX_WORLD; p++) {
        peers.buf[p] = p < world ? reinterpret_cast<float*>(peer_bufs[p]) : nullptr;
        peers.flag[p] = p < world ? reinterpret_cast<unsigned int*>(peer_flags[p]) : nullptr;
        if (p < world && (!peers.buf[p] || !peers.flag[p] || (peer_bufs[p] & 15)))
            return gh_set_error(GH_E_INVALID_ARG, "gh_allreduce_p2p: NULL or misaligned peer mapping");
    }
    float* mc = reinterpret_cast<float*>(multicast_buf);
    // every CTA waits for the entry barrier, so all of them must be resident: sms x (CTAs that fit per SM, capped)
    // defaults (tunable through the environment, swept by tools/allreduce_case.py --sweep; not yet re-swept on H100
    // machines): the NVLS path with FEW requests in flight (128 threads, 1 CTA per SM, 2 x 16 B per thread); the peer
    // load/store path with one full CTA per SM
    const int threads = gh_env_int("GH_ALLREDUCE_THREADS", mc ? 128 : 512, 32, GH_AR_MAX_THREADS) & ~31;
    const int mc_u = gh_env_int("GH_ALLREDUCE_UNROLL", 2, 1, 16);
    const int want_cps = gh_env_int("GH_ALLREDUCE_CTAS_PER_SM", 1, 1, 8);
    const int max_ctas = gh_env_int("GH_ALLREDUCE_MAX_CTAS", 1 << 20, 1, 1 << 20);
    const unsigned long long timeout_ns = 1000000ull * (unsigned long long)gh_env_int("GH_ALLREDUCE_TIMEOUT_MS", 30000, 1, 3600000);
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return gh_cuda_status("gh_allreduce_p2p", "query the device", e);
    const size_t n4 = n_floats / 4, per_rank = (n4 + world - 1) / world;

#define GH_AR_LAUNCH(WT, MU)                                                                                       \
    do {                                                                                                           \
        int occ = 1;                                                                                               \
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gh_allreduce_p2p_kernel<WT, MU>, threads, 0) !=    \
            cudaSuccess || occ < 1) occ = 1;                                                                       \
        const int cps = occ < want_cps ? occ : want_cps;                                                           \
        size_t want = (per_rank + threads - 1) / threads;                                                          \
        const size_t cap0 = (size_t)sms * cps;                                                                     \
        const size_t cap = cap0 < (size_t)max_ctas ? cap0 : (size_t)max_ctas;                                      \
        const int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));                                          \
        gh_allreduce_p2p_kernel<WT, MU><<<grid, threads, 0, stream>>>(peers, mc, rank, world, offset_floats / 4,   \
                                                                      n4, epoch, local_sync, nan_out, timeout_ns); \
    } while (0)
    if (mc != nullptr) {
        if (mc_u >= 16) GH_AR_LAUNCH(0, 16);
        else if (mc_u >= 8) GH_AR_LAUNCH(0, 8);
        else if (mc_u >= 4) GH_AR_LAUNCH(0, 4);
        else if (mc_u >= 2) GH_AR_LAUNCH(0, 2);
        else GH_AR_LAUNCH(0, 1);
    } else if (world == 2) GH_AR_LAUNCH(2, 1);
    else if (world == 4) GH_AR_LAUNCH(4, 1);
    else if (world == 8) GH_AR_LAUNCH(8, 1);
    else GH_AR_LAUNCH(0, 1);
#undef GH_AR_LAUNCH
    return gh_launch_status("gh_allreduce_p2p", 1);
}
