// TEST-ONLY stand-in for <cuda_runtime.h>, the SIMT emulator of tests/simt_emul/cuda_runtime.h extended to thread-block
// clusters (tests/simt_cluster_native.py builds pnp_kernels.cu against it for tests/test_split_simt_cpu.py; the rest of
// the CPU suite keeps the single-CTA emulator).  It lets g++ compile epro-pnp_b200/csrc/pnp_kernels.cu UNCHANGED
// (-DEPNP_SIMT_EMUL, this directory first on the include path, tests/simt_emul next for math_constants.h) into a host
// library whose kernels execute under a small SIMT emulator: the threads of a CTA are user-level fibers (ucontext) of one
// OS thread, scheduled round-robin and switched only at barriers / warp shuffles, CTAs run one after another.  A thread-block cluster
// (cudaLaunchKernelEx with a cluster dimension C) runs as the C CTAs' fibers under one scheduler: each CTA has its own
// shared memory, __syncthreads and named barriers, the cluster barrier waits for every fiber of the C CTAs, and a
// distributed-shared-memory read lands in the target rank's buffer at the same offset.
//
// What this buys the CPU suite (-m "not gpu"): the REAL kernel source -- staging and pair-record packing, the
// block reductions, the LM state machine, the AMIS loop and its shared-memory bookkeeping, the C ABI's argument
// handling -- runs against the golden vectors without a GPU.  Missing barriers are probed by re-running with the fibers scheduled in descending and in
// randomly permuted order (simt_set_schedule): results must be bit-identical.  What it cannot show: memory-model /
// async-proxy ordering, real TMA latency (bulk copies complete synchronously here), the approximate
// special-function units (exact libm here), performance.
// It is not a product path: the shipped library is nvcc-built and has no CPU fallback.
#pragma once
#include <ucontext.h>

// what pnp_device.cuh tests for: this emulator runs thread-block clusters
#define SIMT_EMUL_HAS_CLUSTERS 1

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __align__(n) alignas(n)
#define __shared__ static              // CTAs run one at a time and their threads share the address space
#define __restrict__

using std::max;
using std::min;

struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a) : x(a) {} dim3(int a) : x((unsigned)a) {} };

namespace simt {

constexpr int kMaxThreads = 1024;                      // per CTA
constexpr int kMaxCtas = 8;                            // per cluster
constexpr int kMaxFibers = kMaxThreads * kMaxCtas;
constexpr size_t kStackBytes = 512 * 1024;

struct Fiber {
    ucontext_t ctx;
    char* stack = nullptr;
    bool done = false;
};

// The fibers of one cluster (a plain launch is a cluster of one CTA): fiber cur = cta * nthreads + thread.
struct BlockState {
    ucontext_t sched;
    std::vector<Fiber> fibers;
    const std::function<void()>* body = nullptr;
    int nthreads = 0, ncta = 1, cur = 0, live = 0;      // threads per CTA, CTAs, current fiber, live fibers
    int cta_live[kMaxCtas];
    int bar_count[kMaxCtas];
    unsigned bar_gen[kMaxCtas];
    int named_count[kMaxCtas][16];
    unsigned named_gen[kMaxCtas][16];
    int cl_count = 0;                                   // cluster barrier
    unsigned cl_gen = 0;
    int warp_live[kMaxFibers / 32];
    int warp_count[kMaxFibers / 32];
    unsigned warp_gen[kMaxFibers / 32];
    uint32_t slot[kMaxFibers];
    unsigned char* dyn_smem = nullptr;                  // the current fiber's CTA's dynamic shared memory
    unsigned char* cta_smem[kMaxCtas];
    size_t smem_bytes = 0;
    int cta() const { return cur / nthreads; }
};

inline BlockState& state() { static BlockState s; return s; }
inline uint3& tidx() { static uint3 v{0, 0, 0}; return v; }
inline uint3& bidx() { static uint3 v{0, 0, 0}; return v; }
inline dim3& bdim() { static dim3 v; return v; }
inline dim3& gdim() { static dim3 v; return v; }

inline int& schedule_mode() { static int m = 0; return m; }
inline uint64_t& schedule_seed() { static uint64_t v = 1; return v; }

inline void yield() {
    BlockState& s = state();
    swapcontext(&s.fibers[s.cur].ctx, &s.sched);
}

inline void syncthreads() {
    BlockState& s = state();
    const int c = s.cta();
    const unsigned gen = s.bar_gen[c];
    if (++s.bar_count[c] >= s.cta_live[c]) { s.bar_count[c] = 0; ++s.bar_gen[c]; return; }
    while (s.bar_gen[c] == gen) yield();
}

// bar.sync id, count: `count` threads of the CTA meet on barrier `id` (the kernels only use it with fixed sets)
inline void named_barrier(int id, int count) {
    BlockState& s = state();
    int& cnt = s.named_count[s.cta()][id];
    unsigned& gen = s.named_gen[s.cta()][id];
    const unsigned g = gen;
    if (++cnt >= count) { cnt = 0; ++gen; return; }
    while (gen == g) yield();
}

// barrier.cluster.arrive + wait: every thread of every CTA of the cluster
inline void cluster_sync() {
    BlockState& s = state();
    const unsigned gen = s.cl_gen;
    if (++s.cl_count >= s.live) { s.cl_count = 0; ++s.cl_gen; return; }
    while (s.cl_gen == gen) yield();
}
inline int cluster_rank() { return state().cta(); }

// mapa: the address at p's offset in the dynamic shared memory of the cluster's CTA `rank`
inline const float* map_shared_rank(const float* p, int rank) {
    BlockState& s = state();
    const std::ptrdiff_t off = reinterpret_cast<const unsigned char*>(p) - s.cta_smem[s.cta()];
    if (rank < 0 || rank >= s.ncta || off < 0 || (size_t)off + sizeof(float) > s.smem_bytes) {
        std::fprintf(stderr, "simt_emul: distributed shared memory read of rank %d at offset %td outside [0, %zu) of %d CTAs\n",
                     rank, off, s.smem_bytes, s.ncta);
        std::abort();
    }
    return reinterpret_cast<const float*>(s.cta_smem[rank] + off);
}

inline void syncwarp() {
    BlockState& s = state();
    const int w = s.cur >> 5;
    const unsigned gen = s.warp_gen[w];
    if (++s.warp_count[w] >= s.warp_live[w]) { s.warp_count[w] = 0; ++s.warp_gen[w]; return; }
    while (s.warp_gen[w] == gen) yield();
}

inline uint32_t shfl_xor_bits(uint32_t v, int lane_mask) {
    BlockState& s = state();
    const int me = s.cur;
    s.slot[me] = v;
    syncwarp();
    const uint32_t r = s.slot[(me & ~31) | ((me ^ lane_mask) & 31)];
    syncwarp();
    return r;
}

inline void fiber_main() {
    BlockState& s = state();
    (*s.body)();
    Fiber& f = s.fibers[s.cur];
    f.done = true;
    const int c = s.cta();
    --s.live;
    --s.cta_live[c];
    --s.warp_live[s.cur >> 5];
    // a thread that leaves must not strand the others on a barrier it no longer takes part in
    if (s.cta_live[c] > 0 && s.bar_count[c] >= s.cta_live[c]) { s.bar_count[c] = 0; ++s.bar_gen[c]; }
    if (s.live > 0 && s.cl_count >= s.live) { s.cl_count = 0; ++s.cl_gen; }
    const int w = s.cur >> 5;
    if (s.warp_live[w] > 0 && s.warp_count[w] >= s.warp_live[w]) { s.warp_count[w] = 0; ++s.warp_gen[w]; }
    swapcontext(&f.ctx, &s.sched);
}

// The ncta CTAs of blocks first_block .. first_block + ncta - 1 (one cluster); smem[c] is CTA c's shared memory.
inline void run_cluster(int ncta, int nthreads, unsigned first_block, unsigned char* const* smem,
                        const std::function<void()>& body) {
    BlockState& s = state();
    if (ncta < 1 || ncta > kMaxCtas || nthreads > kMaxThreads || (ncta > 1 && nthreads % 32 != 0)) {
        std::fprintf(stderr, "simt_emul: unsupported launch shape (%d CTAs of %d threads)\n", ncta, nthreads);
        std::abort();
    }
    s.body = &body;
    s.nthreads = nthreads;
    s.ncta = ncta;
    const int nfib = ncta * nthreads;
    s.live = nfib;
    s.cl_count = 0;
    for (int c = 0; c < ncta; ++c) {
        s.cta_live[c] = nthreads;
        s.bar_count[c] = 0;
        s.cta_smem[c] = smem[c];
        for (int i = 0; i < 16; ++i) s.named_count[c][i] = 0;
    }
    if ((int)s.fibers.size() < nfib) s.fibers.resize(nfib);
    for (int w = 0; w < (nfib + 31) / 32; ++w) {
        s.warp_live[w] = std::min(32, nfib - 32 * w);
        s.warp_count[w] = 0;
    }
    for (int t = 0; t < nfib; ++t) {
        Fiber& f = s.fibers[t];
        if (!f.stack) f.stack = (char*)std::malloc(kStackBytes);
        f.done = false;
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = f.stack;
        f.ctx.uc_stack.ss_size = kStackBytes;
        f.ctx.uc_link = &s.sched;
        makecontext(&f.ctx, (void (*)())fiber_main, 0);
    }
    // Scheduling order of the fibers between synchronisation points: 0 = ascending thread index, 1 = descending,
    // 2 = a fresh pseudo-random permutation every round.  Results must not depend on it: a kernel whose output
    // changes with the order has an unsynchronised inter-thread dependency (what racecheck reports on hardware).
    std::vector<int> order(nfib);
    for (int t = 0; t < nfib; ++t) order[t] = (schedule_mode() == 1) ? nfib - 1 - t : t;
    uint64_t rng = schedule_seed() * 6364136223846793005ull + 1442695040888963407ull;
    long spins = 0;
    while (s.live > 0) {
        if (schedule_mode() == 2) {
            for (int t = nfib - 1; t > 0; --t) {
                rng = rng * 6364136223846793005ull + 1442695040888963407ull;
                std::swap(order[t], order[(int)((rng >> 33) % (uint64_t)(t + 1))]);
            }
        }
        for (int i = 0; i < nfib; ++i) {
            const int t = order[i];
            if (s.fibers[t].done) continue;
            s.cur = t;
            tidx() = uint3{(unsigned)(t % nthreads), 0, 0};
            bidx() = uint3{first_block + (unsigned)(t / nthreads), 0, 0};
            s.dyn_smem = smem[t / nthreads];
            swapcontext(&s.sched, &s.fibers[t].ctx);
        }
        if (++spins > 50000000L) { std::fprintf(stderr, "simt_emul: block never finished (deadlocked barrier?)\n"); std::abort(); }
    }
}

// grid.x / cluster clusters of `cluster` CTAs each, one cluster after another
template <class F>
inline void launch_cluster(dim3 grid, dim3 block, size_t smem_bytes, unsigned cluster, F&& kernel_call) {
    BlockState& s = state();
    const std::function<void()> body = kernel_call;
    if (cluster < 1 || cluster > (unsigned)kMaxCtas || grid.x % cluster != 0) {
        std::fprintf(stderr, "simt_emul: grid of %u CTAs in clusters of %u\n", grid.x, cluster);
        std::abort();
    }
    constexpr size_t kGuard = 16384;                  // canary behind the requested bytes: writes past the launch's
    unsigned char* smem[kMaxCtas];                    // dynamic shared memory size must not go unnoticed
    for (unsigned c = 0; c < cluster; ++c)
        smem[c] = (unsigned char*)std::aligned_alloc(1024, ((smem_bytes + kGuard + 1023) / 1024 + 1) * 1024);
    s.smem_bytes = smem_bytes;
    gdim() = grid;
    bdim() = block;
    for (unsigned b = 0; b < grid.x; b += cluster) {
        for (unsigned c = 0; c < cluster; ++c) {
            std::memset(smem[c], 0xCD, smem_bytes);   // poison: a read of never-written shared memory shows up
            std::memset(smem[c] + smem_bytes, 0xEE, kGuard);
        }
        run_cluster((int)cluster, (int)block.x, b, smem, body);
        for (unsigned c = 0; c < cluster; ++c)
            for (size_t i = 0; i < kGuard; ++i)
                if (smem[c][smem_bytes + i] != 0xEE) {
                    std::fprintf(stderr, "simt_emul: write %zu bytes past the %zu bytes of dynamic shared memory (CTA %u)\n",
                                 i, smem_bytes, b + c);
                    std::abort();
                }
    }
    s.dyn_smem = nullptr;
    for (unsigned c = 0; c < cluster; ++c) std::free(smem[c]);
}

template <class F>
inline void launch(dim3 grid, dim3 block, size_t smem_bytes, F&& kernel_call) {
    launch_cluster(grid, block, smem_bytes, 1, kernel_call);
}

}  // namespace simt

#define threadIdx (simt::tidx())
#define blockIdx (simt::bidx())
// identifiers, not expressions: cudaLaunchConfig_t below has members of these names
inline dim3& simt_block_dim = simt::bdim();
inline dim3& simt_grid_dim = simt::gdim();
#define blockDim simt_block_dim
#define gridDim simt_grid_dim

inline void __syncthreads() { simt::syncthreads(); }
inline void __syncwarp(unsigned = 0xffffffffu) { simt::syncwarp(); }
inline float __shfl_xor_sync(unsigned, float v, int m) {
    uint32_t b; std::memcpy(&b, &v, 4);
    b = simt::shfl_xor_bits(b, m);
    float r; std::memcpy(&r, &b, 4);
    return r;
}
inline float __shfl_sync(unsigned, float v, int src_lane) {
    simt::BlockState& s = simt::state();
    const int me = s.cur;
    uint32_t b; std::memcpy(&b, &v, 4);
    s.slot[me] = b;
    simt::syncwarp();
    const uint32_t r = s.slot[(me & ~31) | (src_lane & 31)];
    simt::syncwarp();
    float out; std::memcpy(&out, &r, 4);
    return out;
}
// the only use of __activemask() in the kernels is as the mask of a vote whose outcome selects between two
// equivalent code paths per thread; a per-thread answer is a legal outcome of that vote
constexpr unsigned kEmulActiveMask = 0xA5A5A5A5u;
inline unsigned __activemask() { return kEmulActiveMask; }
inline int __all_sync(unsigned mask, int pred) {
    if (mask == kEmulActiveMask) return pred != 0;
    if (mask == 0xffffffffu) {              // full-warp vote: every lane of the warp takes part
        simt::BlockState& s = simt::state();
        const int me = s.cur, base = me & ~31;
        s.slot[me] = pred != 0;
        simt::syncwarp();
        int all = 1;
        for (int l = 0; l < 32 && base + l < s.ncta * s.nthreads; ++l) all &= (int)s.slot[base + l];
        simt::syncwarp();
        return all;
    }
    std::fprintf(stderr, "simt_emul: __all_sync with an explicit mask is not emulated\n"); std::abort();
}
inline uint32_t __float_as_uint(float x) { uint32_t u; std::memcpy(&u, &x, 4); return u; }
inline float __uint_as_float(uint32_t u) { float x; std::memcpy(&x, &u, 4); return x; }

namespace simt {
// mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 as a warp collective (PTX ISA fragment layout, g = lane / 4,
// t = lane % 4):  A a0 (g, t) a1 (g+8, t) a2 (g, t+4) a3 (g+8, t+4);  B b0 (k = t, n = g) b1 (k = t+4, n = g);
// D d0 (g, 2t) d1 (g, 2t+1) d2 (g+8, 2t) d3 (g+8, 2t+1).  Inputs are truncated to TF32, accumulation is fp32.
inline float tf32(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
inline void mma_m16n8k8_tf32(float (&d)[4], const float (&a)[4], float b0, float b1) {
    static float xa[kMaxFibers][4], xb[kMaxFibers][2];
    BlockState& s = state();
    const int me = s.cur, base = me & ~31, lane = me & 31, g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; ++i) xa[me][i] = tf32(a[i]);
    xb[me][0] = tf32(b0); xb[me][1] = tf32(b1);
    syncwarp();
    for (int i = 0; i < 4; ++i) {
        const int row = g + ((i & 2) ? 8 : 0), col = 2 * t + (i & 1);
        float acc = d[i];
        for (int k = 0; k < 8; ++k) {
            const float av = xa[base + (row & 7) * 4 + (k & 3)][(row >= 8 ? 1 : 0) + (k >= 4 ? 2 : 0)];
            const float bv = xb[base + col * 4 + (k & 3)][k >= 4 ? 1 : 0];
            acc = fmaf(av, bv, acc);
        }
        d[i] = acc;
    }
    syncwarp();
}
}  // namespace simt

template <class T> inline T __ldg(const T* p) { return *p; }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p = o + v; return o; }
inline float atomicAdd(float* p, float v) { const float o = *p; *p = o + v; return o; }
inline long long clock64() { return 0; }

// ---- runtime API subset used by the C ABI's host code -------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0 };
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum { cudaDevAttrMultiProcessorCount = 16 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2 };
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) {          // SM count; SIMT_EMUL_SMS shrinks the "device"
    const char* e = std::getenv("SIMT_EMUL_SMS");
    *v = (e && std::atoi(e) > 0) ? std::atoi(e) : 132;
    return cudaSuccess;
}
template <class F> inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 4; return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (void*)1; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (void*)1; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t n, cudaMemcpyKind, cudaStream_t) { std::memcpy(dst, src, n); return cudaSuccess; }

// extensible launch with a cluster dimension: the clusters run under simt::launch_cluster; SIMT_EMUL_CLUSTERS sets what
// cudaOccupancyMaxActiveClusters reports (0: a device that cannot co-schedule the cluster)
enum cudaLaunchAttributeID { cudaLaunchAttributeClusterDimension = 4 };
struct cudaLaunchAttributeValue { struct { unsigned x, y, z; } clusterDim; };
struct cudaLaunchAttribute { cudaLaunchAttributeID id; cudaLaunchAttributeValue val; };
struct cudaLaunchConfig_t {
    dim3 gridDim, blockDim;
    size_t dynamicSmemBytes;
    cudaStream_t stream;
    cudaLaunchAttribute* attrs;
    unsigned numAttrs;
};
inline unsigned emul_cluster_dim(const cudaLaunchConfig_t* c) {
    for (unsigned i = 0; i < c->numAttrs; ++i)
        if (c->attrs[i].id == cudaLaunchAttributeClusterDimension) return c->attrs[i].val.clusterDim.x;
    return 1;
}
template <class F> inline cudaError_t cudaOccupancyMaxActiveClusters(int* n, F, const cudaLaunchConfig_t*) {
    const char* e = std::getenv("SIMT_EMUL_CLUSTERS");
    *n = e ? std::atoi(e) : 16;
    return cudaSuccess;
}
template <class... Exp, class... Act>
inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* c, void (*kern)(Exp...), Act&&... args) {
    simt::launch_cluster(c->gridDim, c->blockDim, c->dynamicSmemBytes, emul_cluster_dim(c), [&] { kern(args...); });
    return cudaSuccess;
}

// test hooks of the cluster audit build (-DEPNP_SPLIT_AUDIT, see pnp_device.cuh): reset the counters; read them as
// stores[kMaxCtas] followed by mismatches[kMaxCtas]
namespace simt {
struct Audit { long long stores[kMaxCtas], mismatches[kMaxCtas]; };
inline Audit& audit() { static Audit a{}; return a; }
}  // namespace simt
extern "C" inline __attribute__((used, visibility("default"))) void simt_audit_reset() { simt::audit() = simt::Audit{}; }
extern "C" inline __attribute__((used, visibility("default"))) void simt_audit_read(long long* out) {
    for (int c = 0; c < simt::kMaxCtas; ++c) { out[c] = simt::audit().stores[c]; out[simt::kMaxCtas + c] = simt::audit().mismatches[c]; }
}

// test hook: pick the fiber scheduling order (see run_cluster)
extern "C" inline __attribute__((used, visibility("default"))) void simt_set_schedule(int mode, unsigned long long seed) {
    simt::schedule_mode() = mode;
    simt::schedule_seed() = seed;
}
