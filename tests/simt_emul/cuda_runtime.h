// TEST-ONLY stand-in for <cuda_runtime.h>: lets g++ compile epro-pnp_b200/csrc/pnp_kernels.cu UNCHANGED
// (-DEPNP_SIMT_EMUL, this directory first on the include path) into a host library whose kernels execute under
// a small SIMT emulator: the 128 threads of a CTA are user-level fibers (ucontext) of one OS thread, scheduled
// round-robin and switched only at __syncthreads / warp shuffles, CTAs run one after another.
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

constexpr int kMaxThreads = 1024;
constexpr size_t kStackBytes = 512 * 1024;

struct Fiber {
    ucontext_t ctx;
    char* stack = nullptr;
    bool done = false;
};

struct BlockState {
    ucontext_t sched;
    std::vector<Fiber> fibers;
    const std::function<void()>* body = nullptr;
    int nthreads = 0, cur = 0, live = 0;
    int bar_count = 0;
    unsigned bar_gen = 0;
    int warp_live[kMaxThreads / 32];
    int warp_count[kMaxThreads / 32];
    unsigned warp_gen[kMaxThreads / 32];
    uint32_t slot[kMaxThreads];
    unsigned char* dyn_smem = nullptr;
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
    const unsigned gen = s.bar_gen;
    if (++s.bar_count >= s.live) { s.bar_count = 0; ++s.bar_gen; return; }
    while (s.bar_gen == gen) yield();
}

// bar.sync id, count: `count` threads of the CTA meet on barrier `id` (the kernels only use it with fixed sets)
inline void named_barrier(int id, int count) {
    static int cnt[16];
    static unsigned gen[16];
    const unsigned g = gen[id];
    if (++cnt[id] >= count) { cnt[id] = 0; ++gen[id]; return; }
    while (gen[id] == g) yield();
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
    --s.live;
    --s.warp_live[s.cur >> 5];
    // a thread that leaves must not strand the others on a barrier it no longer takes part in
    if (s.live > 0 && s.bar_count >= s.live) { s.bar_count = 0; ++s.bar_gen; }
    const int w = s.cur >> 5;
    if (s.warp_live[w] > 0 && s.warp_count[w] >= s.warp_live[w]) { s.warp_count[w] = 0; ++s.warp_gen[w]; }
    swapcontext(&f.ctx, &s.sched);
}

inline void run_block(int nthreads, const std::function<void()>& body) {
    BlockState& s = state();
    s.body = &body;
    s.nthreads = nthreads;
    s.live = nthreads;
    s.bar_count = 0;
    if ((int)s.fibers.size() < nthreads) s.fibers.resize(nthreads);
    for (int w = 0; w < (nthreads + 31) / 32; ++w) {
        s.warp_live[w] = std::min(32, nthreads - 32 * w);
        s.warp_count[w] = 0;
    }
    for (int t = 0; t < nthreads; ++t) {
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
    std::vector<int> order(nthreads);
    for (int t = 0; t < nthreads; ++t) order[t] = (schedule_mode() == 1) ? nthreads - 1 - t : t;
    uint64_t rng = schedule_seed() * 6364136223846793005ull + 1442695040888963407ull;
    long spins = 0;
    while (s.live > 0) {
        if (schedule_mode() == 2) {
            for (int t = nthreads - 1; t > 0; --t) {
                rng = rng * 6364136223846793005ull + 1442695040888963407ull;
                std::swap(order[t], order[(int)((rng >> 33) % (uint64_t)(t + 1))]);
            }
        }
        for (int i = 0; i < nthreads; ++i) {
            const int t = order[i];
            if (s.fibers[t].done) continue;
            s.cur = t;
            tidx() = uint3{(unsigned)t, 0, 0};
            swapcontext(&s.sched, &s.fibers[t].ctx);
        }
        if (++spins > 50000000L) { std::fprintf(stderr, "simt_emul: block never finished (deadlocked barrier?)\n"); std::abort(); }
    }
}

template <class F>
inline void launch(dim3 grid, dim3 block, size_t smem_bytes, F&& kernel_call) {
    BlockState& s = state();
    const std::function<void()> body = kernel_call;
    constexpr size_t kGuard = 16384;                  // canary behind the requested bytes: writes past the launch's
    unsigned char* smem = (unsigned char*)std::aligned_alloc(1024, ((smem_bytes + kGuard + 1023) / 1024 + 1) * 1024);
    s.dyn_smem = smem;                                // dynamic shared memory size must not go unnoticed
    gdim() = grid;
    bdim() = block;
    for (unsigned b = 0; b < grid.x; ++b) {
        bidx() = uint3{b, 0, 0};
        std::memset(smem, 0xCD, smem_bytes);          // poison: a read of never-written shared memory shows up
        std::memset(smem + smem_bytes, 0xEE, kGuard);
        run_block((int)block.x, body);
        for (size_t i = 0; i < kGuard; ++i)
            if (smem[smem_bytes + i] != 0xEE) {
                std::fprintf(stderr, "simt_emul: write %zu bytes past the %zu bytes of dynamic shared memory\n", i, smem_bytes);
                std::abort();
            }
    }
    s.dyn_smem = nullptr;
    std::free(smem);
}

}  // namespace simt

#define threadIdx (simt::tidx())
#define blockIdx (simt::bidx())
#define blockDim (simt::bdim())
#define gridDim (simt::gdim())

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
        for (int l = 0; l < 32 && base + l < s.nthreads; ++l) all &= (int)s.slot[base + l];
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
    static float xa[kMaxThreads][4], xb[kMaxThreads][2];
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

// test hook: pick the fiber scheduling order (see run_block)
extern "C" inline __attribute__((used, visibility("default"))) void simt_set_schedule(int mode, unsigned long long seed) {
    simt::schedule_mode() = mode;
    simt::schedule_seed() = seed;
}
