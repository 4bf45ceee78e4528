// pnp_device.cuh -- device-side plumbing shared by the sm_90a kernels of the EPro-PnP hot path: launch / shared-memory
// macros (which also let the file build under the test-only CPU SIMT emulator), mbarrier + 1-D TMA bulk-copy wrappers,
// special-function functors, the kernel argument block, warp / block reductions, the packed point store with its TMA
// loader, and the Huber cost sweep over the resident points.  Included by pnp_kernels.cu only.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>

#include "pnp_math.cuh"

// Kernel launches and the dynamic shared-memory declaration are spelled through two macros so that the kernels also
// build, unchanged, under the test-only SIMT emulator (tests/simt_emul, g++ -DEPNP_SIMT_EMUL) that lets the CPU suite
// execute their control flow.  In the nvcc build they expand to the plain CUDA forms.
#if defined(EPNP_SIMT_EMUL)
#define EPNP_LAUNCH(kern, grid, block, smem, stream, ...) simt::launch(grid, block, smem, [&] { kern(__VA_ARGS__); })
#define EPNP_DYN_SMEM(type, name, align) type* name = reinterpret_cast<type*>(simt::state().dyn_smem)
#else
#define EPNP_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#define EPNP_DYN_SMEM(type, name, align) extern __shared__ __align__(align) type name[]
#endif

namespace {
using namespace pnp;

constexpr int NT = 128;                 // threads per CTA of the CTA-per-object kernels
constexpr int NW = NT / 32;
constexpr int CH = 128;                 // correspondences per TMA chunk (2 slots x 3.5 KB)
constexpr int STAGE_FLOATS = CH * 7;    // x3d (3) + x2d (2) + w2d (2)
constexpr int MAX_ITER = 8;             // AMIS iterations supported (reference default 4)
constexpr int PROP_FLOATS = 19;         // proposals dump: mu3, Lt6, Lr10
constexpr size_t SMEM_LIMIT = 227 * 1024;

// Phase timers (profiling build: -DEPNP_PHASE_TIMERS; tools/phase_profile.py).  The serial thread `st` of every AMIS CTA
// adds the clock64() cycles it spent in each phase; the production build compiles them away.
enum Phase { PH_LOAD = 0, PH_DRAW_SWEEP, PH_LOGP_OLD, PH_WEIGHTS, PH_REFIT_SUMS, PH_REFIT_FINISH, PH_OUTPUT, PH_COUNT };
#ifdef EPNP_PHASE_TIMERS
#define PH_DECL long long ph_t = clock64()
#define PH_MARK(a_, which)                                                                     \
    do {                                                                                       \
        if ((int)threadIdx.x == st && (a_).prof) {                              \
            const long long now_ = clock64();                                                  \
            atomicAdd((a_).prof + (which), (unsigned long long)(now_ - ph_t));                 \
            ph_t = now_;                                                                       \
        }                                                                                      \
    } while (0)
#else
#define PH_DECL
#define PH_MARK(a_, which)
#endif

// Cluster audit, a build option of the test-only emulator (-DEPNP_SPLIT_AUDIT): the split kernels count, per cluster
// rank, the output elements each rank stores and the elements of its AMIS state (costs, log-densities, samples) that
// differ from rank 0's.  The shipped build compiles the macros away.
#if defined(EPNP_SIMT_EMUL) && defined(SIMT_EMUL_HAS_CLUSTERS) && defined(EPNP_SPLIT_AUDIT)
#define SPLIT_AUDIT_STORES(n) (simt::audit().stores[simt::cluster_rank()] += (n))
#define SPLIT_AUDIT_MISMATCH() (++simt::audit().mismatches[simt::cluster_rank()])
#else
#define SPLIT_AUDIT_STORES(n)
#define SPLIT_AUDIT_MISMATCH()
#endif

// ------------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + 1-D TMA bulk copy; special-function units
#if defined(EPNP_SIMT_EMUL)
// emulator: an mbarrier word is {completed phases (low 32 bits), bytes still expected (high 32 bits)}; a bulk copy
// is a memcpy that retires its bytes and completes the phase when none are left; waiting on a parity yields to the
// other fibers until that phase has completed.  Exact libm stands in for the approximate special-function units.
inline void mbar_init(uint64_t* bar, uint32_t) { *bar = 0; }
inline void fence_barrier_init() {}
inline void fence_proxy_async() {}
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { *bar += (uint64_t)bytes << 32; }
inline void mbar_wait(uint64_t* bar, uint32_t parity) { while (((uint32_t)*bar & 1u) == parity) simt::yield(); }
inline void tma_load_1d(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
    std::memcpy(dst_smem, src, bytes);
    *bar -= (uint64_t)bytes << 32;
    if ((*bar >> 32) == 0) *bar = (uint32_t)*bar + 1u;
}
inline void named_barrier(int id, int count) { simt::named_barrier(id, count); }
#if defined(SIMT_EMUL_HAS_CLUSTERS)
// thread-block clusters: the cluster emulator (tests/simt_cluster) runs a cluster's CTAs as one set of fibers
inline int cluster_rank() { return simt::cluster_rank(); }
inline void cluster_sync() { simt::cluster_sync(); }
inline float dsmem_ld(const float* p, int rank) { return *simt::map_shared_rank(p, rank); }
#else
// the single-CTA emulator (tests/simt_emul) has no clusters: the split kernels compile, their launches are refused
// (launch_cluster_per_object), so these never run
inline int cluster_rank() { return 0; }
inline void cluster_sync() { std::abort(); }
inline float dsmem_ld(const float*, int) { std::abort(); }
#endif
struct FastRcp { float operator()(float x) const { return 1.0f / x; } };
struct FastSqrt { float operator()(float x) const { return sqrtf(x); } };
struct FastRsqrt { float operator()(float x) const { return 1.0f / sqrtf(x); } };
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// barrier `id` (1..15; 0 is __syncthreads) among `count` threads (a multiple of 32) of the CTA
__device__ __forceinline__ void named_barrier(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Thread-block clusters (sm_90): the CTA's rank in its cluster; a barrier of every thread of every CTA in the cluster
// whose release / acquire orders shared-memory writes before it against distributed-shared-memory reads after it; a
// read of the float at the same shared-memory offset as `p` in the CTA of rank `rank` (mapa + ld.shared::cluster).
__device__ __forceinline__ int cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return (int)r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
__device__ __forceinline__ float dsmem_ld(const float* p, int rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(p)), "r"(rank));
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
    return v;
}

struct FastRcp {
    __device__ __forceinline__ float operator()(float x) const { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
};
struct FastSqrt {
    __device__ __forceinline__ float operator()(float x) const { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
};
struct FastRsqrt {
    __device__ __forceinline__ float operator()(float x) const { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
};
#endif

// ------------------------------------------------------------------------------------------------
struct KArgs {
    const float *x3d, *x2d, *w2d, *cam, *lb, *ub, *delta;
    const float *pose_init;                 // LM entry
    const float *pose_opt_in, *pose_cov_in; // AMIS entry (the LM kernel's outputs in the fused call)
    const float *noise_n3, *noise_chi2, *noise_rot;
    const float *poses;                     // cost-only entry: (S, B, D)
    float *pose_opt, *pose_cov, *cost, *pose_plus, *cost_init;
    float *pose_samples, *logw, *proposals;
    float *cost_out;                        // cost-only entry: (S, B)
    int B, N, S_eval, use_tma, num_sms;
    int cov_stride;                         // floats between two objects' covariances (dof^2, or M*D when the fused
                                            // call parks them in the not-yet-written sample buffer)
    uint32_t obj_offset;
    uint64_t seed;
    unsigned long long* prof;               // phase timers (profiling build only), else unused
    Params p;
};

// ------------------------------------------------------------------------------------------------
// Packed point store of the CTA-per-object kernels.  Pair j = points (2j, 2j+1) occupies 16 floats:
//   [0..3] X0 X1 Y0 Y1   [4..7] Z0 Z1 -u0 -u1   [8..11] -v0 -v1 wu0 wu1   [12..15] wv0 wv1 0 0
// the operand layout of the packed fp32x2 sweep (4 x LDS.128 per pair, warp-broadcast).
__device__ __forceinline__ void store_point(float* pts, int n, float X, float Y, float Z, float u, float v, float wu, float wv) {
    float* p = pts + (n >> 1) * 16 + (n & 1);
    p[0] = X; p[2] = Y; p[4] = Z; p[6] = -u; p[8] = -v; p[10] = wu; p[12] = wv;
}
// odd N: the second half of the last pair is a zero-weight copy of the last point (contributes exactly 0);
// written by the SAME thread that stores point N-1, so no other thread's data is read
__device__ __forceinline__ void store_point_padded(float* pts, int n, int N, float X, float Y, float Z, float u, float v,
                                                   float wu, float wv) {
    store_point(pts, n, X, Y, Z, u, v, wu, wv);
    if ((N & 1) && n == N - 1) store_point(pts, n + 1, X, Y, Z, u, v, 0.f, 0.f);
}

// Correspondence loader of the CTA-per-object kernels (one object per CTA, blockIdx.x = object): the object's
// {x3d, x2d, w2d} come from HBM exactly once, in CHUNK-point chunks through a 2-slot TMA ring (cp.async.bulk completing on
// an mbarrier), and are re-packed into the pair records; plain loads when the pointers / N break the 16-byte rules.
// CHUNK = 128 (2 x 3.5 KB of ring, hidden inside the sample buffer); 512 for the 512-thread CTAs of long point sets.
template <int CHUNK = CH>
struct LoaderT {
    static constexpr int SLOT_FLOATS = CHUNK * 7;
    const KArgs& a;
    uint64_t* bar;
    float* stage;
    int nch;

    __device__ LoaderT(const KArgs& a_, uint64_t* bar_, float* stage_) : a(a_), bar(bar_), stage(stage_) {
        nch = (a.N + CHUNK - 1) / CHUNK;
    }
    __device__ void issue(int obj, int k) {          // one thread
        const int npts = min(CHUNK, a.N - k * CHUNK);
        const size_t first = (size_t)obj * a.N + (size_t)k * CHUNK;
        float* dst = stage + (k & 1) * SLOT_FLOATS;
        uint64_t* b = bar + (k & 1);
        mbar_expect_tx(b, (uint32_t)npts * 28u);
        tma_load_1d(dst, a.x3d + first * 3, (uint32_t)npts * 12u, b);
        tma_load_1d(dst + CHUNK * 3, a.x2d + first * 2, (uint32_t)npts * 8u, b);
        tma_load_1d(dst + CHUNK * 5, a.w2d + first * 2, (uint32_t)npts * 8u, b);
    }
    // Bring object `obj` into the packed point array (T = threads of the CTA).  Ends with a barrier of the threads that
    // took part.  skip_warp < 0: all T threads take part (barriers = __syncthreads).  skip_warp = w: warp w does NOT call
    // this function (it is busy with the object's serial set-up); the other T - 32 threads synchronise on named barrier
    // 1, and the caller joins everybody with a __syncthreads afterwards.
    template <int T = NT> __device__ void load_object(int obj, float* pts, int skip_warp = -1) {
        const int tid = threadIdx.x;
        const bool partial = skip_warp >= 0;
        const int nthr = partial ? T - 32 : T;
        const int rank = (partial && tid >= 32 * (skip_warp + 1)) ? tid - 32 : tid;      // index among the participants
        auto sync = [&]() { if (partial) named_barrier(1, T - 32); else __syncthreads(); };
        if (a.use_tma) {
            if (rank == 0) {
                mbar_init(bar + 0, 1);
                mbar_init(bar + 1, 1);
                fence_barrier_init();
                issue(obj, 0);
                if (nch > 1) issue(obj, 1);
            }
            sync();
            for (int k = 0; k < nch; ++k) {
                const float* st = stage + (k & 1) * SLOT_FLOATS;
                mbar_wait(bar + (k & 1), (uint32_t)((k >> 1) & 1));
                const int npts = min(CHUNK, a.N - k * CHUNK);
                for (int n = rank; n < npts; n += nthr) {
                    const float2 uv = reinterpret_cast<const float2*>(st + CHUNK * 3)[n];
                    const float2 w = reinterpret_cast<const float2*>(st + CHUNK * 5)[n];
                    store_point_padded(pts, k * CHUNK + n, a.N, st[3 * n], st[3 * n + 1], st[3 * n + 2], uv.x, uv.y, w.x, w.y);
                }
                sync();                     // slot drained (and, after the last chunk, pts complete)
                if (rank == 0 && k + 2 < nch) { fence_proxy_async(); issue(obj, k + 2); }
            }
        } else {
            const float* g3 = a.x3d + (size_t)obj * a.N * 3;
            const float* g2 = a.x2d + (size_t)obj * a.N * 2;
            const float* gw = a.w2d + (size_t)obj * a.N * 2;
            for (int n = rank; n < a.N; n += nthr)
                store_point_padded(pts, n, a.N, __ldg(g3 + 3 * n), __ldg(g3 + 3 * n + 1), __ldg(g3 + 3 * n + 2),
                                   __ldg(g2 + 2 * n), __ldg(g2 + 2 * n + 1), __ldg(gw + 2 * n), __ldg(gw + 2 * n + 1));
            sync();
        }
    }

    // load_object for the points [p0, p1) of object `obj` only (a CTA of a cluster-split kernel): they become pair records
    // 0, 1, ... of `pts`, an odd count padded like an odd N.  p0 is a multiple of 8 points, so with N % 4 == 0 every bulk
    // copy starts on 16 bytes and moves a multiple of 16 bytes, as load_object's do.  Same participants and barriers.
    __device__ void issue_range(int obj, int k, int p0, int p1) {
        const int npts = min(CHUNK, p1 - p0 - k * CHUNK);
        const size_t first = (size_t)obj * a.N + (size_t)p0 + (size_t)k * CHUNK;
        float* dst = stage + (k & 1) * SLOT_FLOATS;
        uint64_t* b = bar + (k & 1);
        mbar_expect_tx(b, (uint32_t)npts * 28u);
        tma_load_1d(dst, a.x3d + first * 3, (uint32_t)npts * 12u, b);
        tma_load_1d(dst + CHUNK * 3, a.x2d + first * 2, (uint32_t)npts * 8u, b);
        tma_load_1d(dst + CHUNK * 5, a.w2d + first * 2, (uint32_t)npts * 8u, b);
    }
    template <int T> __device__ void load_range(int obj, float* pts, int p0, int p1, int skip_warp = -1) {
        const int tid = threadIdx.x;
        const bool partial = skip_warp >= 0;
        const int nthr = partial ? T - 32 : T;
        const int rank = (partial && tid >= 32 * (skip_warp + 1)) ? tid - 32 : tid;
        auto sync = [&]() { if (partial) named_barrier(1, T - 32); else __syncthreads(); };
        const int cnt = p1 - p0, nchr = (cnt + CHUNK - 1) / CHUNK;
        if (a.use_tma) {
            if (rank == 0) {
                mbar_init(bar + 0, 1);
                mbar_init(bar + 1, 1);
                fence_barrier_init();
                if (nchr > 0) issue_range(obj, 0, p0, p1);
                if (nchr > 1) issue_range(obj, 1, p0, p1);
            }
            sync();
            for (int k = 0; k < nchr; ++k) {
                const float* st = stage + (k & 1) * SLOT_FLOATS;
                mbar_wait(bar + (k & 1), (uint32_t)((k >> 1) & 1));
                const int npts = min(CHUNK, cnt - k * CHUNK);
                for (int n = rank; n < npts; n += nthr) {
                    const float2 uv = reinterpret_cast<const float2*>(st + CHUNK * 3)[n];
                    const float2 w = reinterpret_cast<const float2*>(st + CHUNK * 5)[n];
                    store_point_padded(pts, k * CHUNK + n, cnt, st[3 * n], st[3 * n + 1], st[3 * n + 2], uv.x, uv.y, w.x, w.y);
                }
                sync();
                if (rank == 0 && k + 2 < nchr) { fence_proxy_async(); issue_range(obj, k + 2, p0, p1); }
            }
        } else {
            const float* g3 = a.x3d + ((size_t)obj * a.N + p0) * 3;
            const float* g2 = a.x2d + ((size_t)obj * a.N + p0) * 2;
            const float* gw = a.w2d + ((size_t)obj * a.N + p0) * 2;
            for (int n = rank; n < cnt; n += nthr)
                store_point_padded(pts, n, cnt, __ldg(g3 + 3 * n), __ldg(g3 + 3 * n + 1), __ldg(g3 + 3 * n + 2),
                                   __ldg(g2 + 2 * n), __ldg(g2 + 2 * n + 1), __ldg(gw + 2 * n), __ldg(gw + 2 * n + 1));
            sync();
        }
    }
};
typedef LoaderT<CH> Loader;

__device__ __forceinline__ Cam load_cam(const KArgs& a, int obj) {
    Cam c;
#pragma unroll
    for (int i = 0; i < 9; ++i) c.k[i] = __ldg(a.cam + (size_t)obj * 9 + i);
    c.z_min = a.p.z_min;
    c.bounded = (a.lb != nullptr && a.ub != nullptr) ? 1 : 0;
    if (c.bounded) {
        c.lbx = __ldg(a.lb + 2 * obj); c.lby = __ldg(a.lb + 2 * obj + 1);
        c.ubx = __ldg(a.ub + 2 * obj); c.uby = __ldg(a.ub + 2 * obj + 1);
    } else {
        c.lbx = c.lby = -CUDART_INF_F; c.ubx = c.uby = CUDART_INF_F;
    }
    return c;
}

// The once-per-iteration serial work of an AMIS CTA (first proposal, refit finish) runs on lane 0 of ONE warp.
// Co-resident CTAs of an SM are typically blockIdx, blockIdx + #SM, ...; rotating the serial warp with
// blockIdx / #SM puts their serial chains on different SM sub-partitions (warp w -> SMSP w % 4).
template <int T = NT> __device__ __forceinline__ int serial_thread(const KArgs& a) {
    return 32 * (int)((blockIdx.x / (unsigned)max(a.num_sms, 1)) & (T / 32 - 1));
}

// ------------------------------------------------------------------------------------------------
// Reductions
// 32 values per lane -> lane j holds the warp total of v[j]   (31 shuffles instead of 5 per value)
__device__ __forceinline__ float warp_transpose_sum(float (&v)[32]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int half = 16; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int k = 0; k < half; ++k) {
            const float keep = up ? v[k + half] : v[k];
            const float send = up ? v[k] : v[k + half];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    return v[0];
}

// W values per lane (W = 8, 16 or 32) -> lane l holds the warp total of v[l >> (5 - log2 W)]: log2(W) transposed
// butterfly stages (W - 1 shuffles) + plain butterfly adds for the rest.
template <int W> __device__ __forceinline__ float warp_transpose_sum_w(float (&v)[W]) {
    static_assert(W == 8 || W == 16 || W == 32, "W must be 8, 16 or 32");
    const int lane = threadIdx.x & 31;
    int m = 16;
#pragma unroll
    for (int half = W / 2; half >= 1; half >>= 1, m >>= 1) {
        const bool up = (lane & m) != 0;
#pragma unroll
        for (int k = 0; k < half; ++k) {
            const float keep = up ? v[k + half] : v[k];
            const float send = up ? v[k] : v[k + half];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
    }
    float r = v[0];
#pragma unroll
    for (int o = 16 / W; o >= 1; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    return r;
}

// Block-wide sums of K values per thread (T threads, a multiple of 128); every thread gets the totals.  `red` holds two
// halves of (T / 32) * 32 floats: call sites alternate `half` so one __syncthreads per reduction is enough (a thread
// can be at most one reduction ahead of the slowest reader, and then it writes the other half).  The per-warp totals
// are added in warp order, four at a time -- the same association for every T.
template <int T> __device__ __forceinline__ float sum_warp_partials(const float* r, int k) {
    float tot = (r[k] + r[32 + k]) + (r[64 + k] + r[96 + k]);
#pragma unroll
    for (int w = 4; w < T / 32; w += 4) tot += (r[w * 32 + k] + r[(w + 1) * 32 + k]) + (r[(w + 2) * 32 + k] + r[(w + 3) * 32 + k]);
    return tot;
}
template <int K, int T = NT> __device__ __forceinline__ void block_sum(float (&v)[K], float* red, int half) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* r = red + half * (T / 32 * 32);
    static_assert(K <= 32 && T % 128 == 0, "block_sum: at most 32 values, whole groups of four warps");
    if constexpr (K > 2) {
        constexpr int W = K <= 8 ? 8 : (K <= 16 ? 16 : 32);
        float w[W];
#pragma unroll
        for (int k = 0; k < W; ++k) w[k] = k < K ? v[k] : 0.f;
        const float tot = warp_transpose_sum_w<W>(w);
        constexpr int SH = W == 8 ? 2 : (W == 16 ? 1 : 0);
        if ((lane & ((1 << SH) - 1)) == 0 && (lane >> SH) < K) r[warp * 32 + (lane >> SH)] = tot;
    } else {
#pragma unroll
        for (int k = 0; k < K; ++k) {
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < K; ++k) r[warp * 32 + k] = v[k];
        }
    }
    __syncthreads();
    if constexpr (K > 4) {
        // lane k of every warp adds the per-warp totals of value k (T / 32 loads); K shuffles hand every lane all K
        // totals -- instead of K * T / 32 loads per thread
        const float mine = lane < K ? sum_warp_partials<T>(r, lane) : 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = __shfl_sync(0xffffffffu, mine, k);
    } else {
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = sum_warp_partials<T>(r, k);
    }
}

template <int T = NT> __device__ __forceinline__ float block_max(float v, float* red, int half) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* r = red + half * (T / 32 * 32);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) r[warp * 32] = v;
    __syncthreads();
    float m = fmaxf(fmaxf(r[0], r[32]), fmaxf(r[64], r[96]));
#pragma unroll
    for (int w = 4; w < T / 32; ++w) m = fmaxf(m, r[w * 32]);
    return m;
}

// ------------------------------------------------------------------------------------------------
// Huber cost of one pose over every resident point: thread-private sweep, every lane reads the same pair record
// (shared-memory broadcast, 4 x LDS.128 per 2 points) and evaluates two points side by side in fp32x2 pairs
// (two scalar FFMA / FMUL per V2 op on sm_90a).  P2[k] = (P[k], P[k]) is the pre-multiplied projection K[R|t] duplicated into both
// halves.  Per point pair: 17 packed FP ops + 4 MUFU (rcp, sqrt); Huber as m (s - m / 2), m = min(s, delta) -- both
// branches in one expression, no select -- accumulated by its last multiply-add.  Same arithmetic per half as pnp::point_cost.
__device__ __forceinline__ float2 splat(float x) { return make_float2(x, x); }

// ZCLAMP = false drops the depth clamp: only for a pose whose every point is known to lie beyond z_min (depth_clears),
// where fmaxf(zh, z_min) == zh and the result is the same.
template <bool BOUNDED, bool ZCLAMP = true>
__device__ __forceinline__ float2 pair_cost(const float2 (&P2)[12], const Cam& cam, float delta, float2 acc,
                                            const float4 q0, const float4 q1, const float4 q2, const float4 q3) {
    const float2 X = make_float2(q0.x, q0.y), Y = make_float2(q0.z, q0.w), Z = make_float2(q1.x, q1.y);
    const float2 nu = make_float2(q1.z, q1.w), nv = make_float2(q2.x, q2.y);
    const float2 wu = make_float2(q2.z, q2.w), wv = make_float2(q3.x, q3.y);
    const float2 xh = v2fma(P2[0], X, v2fma(P2[1], Y, v2fma(P2[2], Z, P2[3])));
    const float2 yh = v2fma(P2[4], X, v2fma(P2[5], Y, v2fma(P2[6], Z, P2[7])));
    const float2 zh = v2fma(P2[8], X, v2fma(P2[9], Y, v2fma(P2[10], Z, P2[11])));
    const float2 iz = ZCLAMP ? make_float2(FastRcp()(fmaxf(zh.x, cam.z_min)), FastRcp()(fmaxf(zh.y, cam.z_min)))
                             : make_float2(FastRcp()(zh.x), FastRcp()(zh.y));
    float2 tx, ty;
    if (BOUNDED) {
        float2 px = v2mul(xh, iz), py = v2mul(yh, iz);
        px.x = fminf(fmaxf(px.x, cam.lbx), cam.ubx); px.y = fminf(fmaxf(px.y, cam.lbx), cam.ubx);
        py.x = fminf(fmaxf(py.x, cam.lby), cam.uby); py.y = fminf(fmaxf(py.y, cam.lby), cam.uby);
        tx = v2add(px, nu); ty = v2add(py, nv);
    } else {
        tx = v2fma(xh, iz, nu); ty = v2fma(yh, iz, nv);
    }
    const float2 rx = v2mul(tx, wu), ry = v2mul(ty, wv);
    const float2 s2 = v2fma(rx, rx, v2mul(ry, ry));
    const float2 s = make_float2(FastSqrt()(s2.x), FastSqrt()(s2.y));
    const float2 m = make_float2(fminf(s.x, delta), fminf(s.y, delta));
    return v2fma(m, v2fma(m, splat(-0.5f), s), acc);
}

// pair records [j0, j1)
template <bool BOUNDED, bool ZCLAMP = true>
__device__ __forceinline__ float sweep_cost(const float4* pts4, int j0, int j1, const float* P, const Cam& cam, float delta) {
    // point pairs in flight per thread: enough independent chains to cover the FMA and MUFU latencies at five
    // resident CTAs per SM without raising the register count past what those five CTAs allow
    constexpr int U = 4;
    float2 P2[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) P2[k] = splat(P[k]);
    float2 c[U];
#pragma unroll
    for (int u = 0; u < U; ++u) c[u] = splat(0.f);
    const int npair = j1;
    int j = j0;
    for (; j + U <= npair; j += U) {
        const float4* q = pts4 + 4 * j;
#pragma unroll
        for (int u = 0; u < U; ++u) c[u] = pair_cost<BOUNDED, ZCLAMP>(P2, cam, delta, c[u], q[4 * u], q[4 * u + 1], q[4 * u + 2], q[4 * u + 3]);
    }
    for (; j < npair; ++j) {
        const float4* q = pts4 + 4 * j;
        c[0] = pair_cost<BOUNDED, ZCLAMP>(P2, cam, delta, c[0], q[0], q[1], q[2], q[3]);
    }
    float2 t = c[0];
#pragma unroll
    for (int u = 1; u < U; ++u) t = v2add(t, c[u]);
    return t.x + t.y;
}

// cost of `pose` over the pair records [j0, j1)
template <int DOF>
__device__ __forceinline__ float pose_cost_pairs(const float* pts, int j0, int j1, const float* pose, const Cam& cam, float delta) {
    float R[9], P[12];
    pose_to_rot<DOF>(pose, R);
    make_proj(cam.k, R, pose, P);
    const float4* pts4 = reinterpret_cast<const float4*>(pts);
    return cam.bounded ? sweep_cost<true>(pts4, j0, j1, P, cam, delta) : sweep_cost<false>(pts4, j0, j1, P, cam, delta);
}
template <int DOF>
__device__ __forceinline__ float pose_cost(const float* pts, int N, const float* pose, const Cam& cam, float delta) {
    return pose_cost_pairs<DOF>(pts, 0, (N + 1) >> 1, pose, cam, delta);
}

// Axis-aligned bounding box of an object's resident points: box[0..2] = min X, Y, Z, box[3..5] = max X, Y, Z.  An axis
// with a non-finite coordinate gets (-inf, +inf), so depth_clears fails for every pose.  Block-wide (T threads), the
// per-warp partials pass through `red`; `box` is shared memory and complete when the function returns.
template <int T>
__device__ __forceinline__ void point_box(const float* pts, int N, float* red, float* box) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float v[6];                             // min X, min Y, min Z, -max X, -max Y, -max Z
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = CUDART_INF_F;
    const float4* pts4 = reinterpret_cast<const float4*>(pts);
    for (int j = threadIdx.x; j < (N + 1) >> 1; j += T) {
        const float4 a = pts4[4 * j], b = pts4[4 * j + 1];      // X0 X1 Y0 Y1, Z0 Z1 ..
        const float c[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const int ax = k >> 1;
            if (isfinite(c[k])) { v[ax] = fminf(v[ax], c[k]); v[3 + ax] = fminf(v[3 + ax], -c[k]); }
            else v[ax] = v[3 + ax] = -CUDART_INF_F;
        }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k)
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) v[k] = fminf(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) red[warp * 32 + k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        const int k = threadIdx.x;
        float m = red[k];
#pragma unroll
        for (int w = 1; w < T / 32; ++w) m = fminf(m, red[w * 32 + k]);
        box[k] = k < 3 ? m : -m;
    }
    __syncthreads();
}

// Whether zh = P[8] X + P[9] Y + P[10] Z + P[11] exceeds z_min for every point of `box`, however the sweep rounds it: the
// box's lowest zh, less a margin far above the rounding error of both that bound and the sweep's three-FFMA chain (each a
// few units in the last place of |P[8]| |X| + |P[9]| |Y| + |P[10]| |Z| + |P[11]|).  NaN anywhere makes it false.
__device__ __forceinline__ bool depth_clears(const float* P, const float* box, float z_min) {
    float lo = P[11], mag = fabsf(P[11]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo += fminf(P[8 + k] * box[k], P[8 + k] * box[3 + k]);
        mag += fabsf(P[8 + k]) * fmaxf(fabsf(box[k]), fabsf(box[3 + k]));
    }
    return lo - (1e-5f * mag + 1e-30f) > z_min;
}

// pose_cost_pairs for an object whose points lie in `box`.  Where no point of the pose can reach the depth clamp and the
// camera has no bounds, the sweep runs without the clamp; the lanes sweeping together vote, so a warp runs one loop.
template <int DOF>
__device__ __forceinline__ float pose_cost_pairs(const float* pts, int j0, int j1, const float* pose, const Cam& cam, float delta,
                                                 const float* box) {
    float R[9], P[12];
    pose_to_rot<DOF>(pose, R);
    make_proj(cam.k, R, pose, P);
    const float4* pts4 = reinterpret_cast<const float4*>(pts);
    if (__all_sync(__activemask(), !cam.bounded && depth_clears(P, box, cam.z_min)))
        return sweep_cost<false, false>(pts4, j0, j1, P, cam, delta);
    return cam.bounded ? sweep_cost<true>(pts4, j0, j1, P, cam, delta) : sweep_cost<false>(pts4, j0, j1, P, cam, delta);
}

}  // namespace
