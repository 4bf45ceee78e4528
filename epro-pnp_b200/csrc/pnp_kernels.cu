// pnp_kernels.cu -- sm_90a kernels of the EPro-PnP hot path and their C ABI (include/epropnp_b200.h).
//
//   lm_warp_kernel (pnp_lm.cuh)      Levenberg-Marquardt / Gauss-Newton pose solve, ONE WARP per object: raw correspondences
//                                    TMA-staged into the warp's shared memory, 16 points per lane, shuffle-only reduction,
//                                    6x6 damped Cholesky + SE(3) retraction + trust region on lane 0, no block barrier.
//   amis_kernel (pnp_amis.cuh)       the AMIS Monte-Carlo loop, ONE CTA per object: TMA ring -> packed pair records, one
//                                    thread per sample, packed fp32x2 cost sweep, refits as block reductions; five CTAs per SM.
//   lm_stacked_kernel (pnp_lm.cuh)   the same solve from S stacked starts per object: the hypotheses of one object share
//                                    one staged copy of its points, H hypothesis warps per CTA, each warp lm_warp_kernel's body.
//   epnp_lm_amis_fused_f32           = lm_warp_kernel, then amis_kernel, on the caller's stream (no host round trip); the
//                                    split is what a measurement asked for: as one kernel the LM half ran latency-bound at
//                                    4 points per thread between block barriers (DESIGN.md section 4).
//   cost_kernel, evaluate_full_kernel, rslm_draw_kernel, rslm_kernel, cost_backward_kernel, gn_plus_backward_kernel, adaptive_delta_kernel,
//   mc_epilogue_kernel, mc_lse_backward_kernel      the steps either side of the path (CTA per object).
//   evaluate_backward_kernel         the backward of evaluate_full_kernel's residual / Jacobian / cost (CTA per object, any N).
//   cost_hvp_point_kernel, cost_hvp_pose_kernel    second order through the cost: Hessian-vector products, point-major
//                                    (CTA per object) and pose-major (thread per pose), points streamed from global memory.
//   evaluate_jvp_kernel, evaluate_jvp_cost_kernel   forward mode of evaluate_full_kernel: the Jacobian-vector product of
//                                    the residual, Jacobian and cost (CTA per pose and object), and of the cost alone at many
//                                    poses (thread per pose, points staged through shared memory).
//   cost_pose_backward_kernel, cost_pose_backward_split_kernel    the cost's gradient with respect to stacked poses: thread per
//                                    pose over the resident points; the split form on cost_split_kernel's clusters.
//   epnp_init_kernel (pnp_epnp.cuh)  EPnP initialiser with the confidence-quantile point selection, fp64, CTA per object.
//   amis_split_kernel (pnp_amis.cuh), cost_split_kernel, gn_plus_backward_split_kernel, epnp_init_split_kernel   the AMIS
//                                    loop, the stacked-pose cost, the pose_opt_plus backward and the EPnP initialiser for
//                                    objects whose points do not fit one SM: one thread-block CLUSTER of 2..8 CTAs per
//                                    object, each holding a point range, partial sums added in rank order over distributed
//                                    shared memory (sum_ranks, pnp_device.cuh).
//   push_split_kernel                the multi-GPU gather of the split solve: this rank's rows copied into its peers' buffers.
// No tensor cores: the only contraction is 6-deep, the work is FP32-pipe + MUFU bound (DESIGN.md).
// Build options: EPNP_PHASE_TIMERS (profiling), EPNP_SIMT_EMUL (g++ build for the test-only CPU emulator).
#include <cuda_runtime.h>
#include <math_constants.h>

#include <cstdlib>

#include "pnp_device.cuh"
#include "pnp_lm.cuh"
#include "pnp_amis.cuh"
#include "pnp_epnp.cuh"

namespace {

thread_local int g_last_cuda_error = 0;

// Shared-memory image of the CTA-per-object kernels that are not the AMIS loop: head, TMA ring, packed pair records.
template <int DOF> struct ObjHead {
    uint64_t bar[2];
    float red[2 * NW * 32];
    float ev[32];                           // reduced evaluation: NV floats
    float pose[8];
    float step[2 * DOF];                    // gn_plus_backward: step, v
};
struct ObjPlan { int stage, pts, total_bytes; };
template <int DOF> __host__ __device__ inline ObjPlan plan_obj(int N) {
    ObjPlan s;
    int off = (int)((sizeof(ObjHead<DOF>) + 127) / 128 * 128 / 4);
    s.stage = off; off += 2 * STAGE_FLOATS;
    s.pts = off; off += 16 * ((N + 1) / 2);
    s.total_bytes = off * 4;
    return s;
}

// cost of S poses per object: poses (S, B, D) -> cost (S, B)
template <int DOF>
__global__ void __launch_bounds__(NT, 4) cost_kernel(const KArgs a) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts4 = dyn + pl.pts;
    constexpr int PD = Dim<DOF>::POSE;
    const int obj = blockIdx.x;
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts4);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    for (int s = threadIdx.x; s < a.S_eval; s += NT) {
        float pose[PD];
#pragma unroll
        for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + ((size_t)s * a.B + obj) * PD + k);
        a.cost_out[(size_t)s * a.B + obj] = pose_cost<DOF>(pts4, a.N, pose, cam, delta);
    }
}

// cost_kernel for objects too large for one SM: one cluster of `ctas` CTAs per object (grid = B * ctas), rank r holding
// the points [r share, (r + 1) share) (split_share).  Every rank evaluates every pose on its own range, COST_SPLIT_TILE
// poses at a time (one per thread); rank 0 adds the ranks' partial costs (sum_ranks) and writes the result.
constexpr int COST_SPLIT_TILE = 512;
struct CostSplitPlan { int stage, pts, xbuf, total_bytes; };
__host__ __device__ inline CostSplitPlan plan_cost_split(int share) {
    CostSplitPlan s;
    int off = 128 / 4;                      // the two mbarriers of the staging ring, 128-byte aligned
    s.stage = off; off += 2 * STAGE_FLOATS;
    s.pts = off; off += 16 * ((share + 1) / 2);
    s.xbuf = off; off += 2 * COST_SPLIT_TILE;
    s.total_bytes = off * 4;
    return s;
}

template <int DOF>
__global__ void __launch_bounds__(COST_SPLIT_TILE, 1) cost_split_kernel(const KArgs a, const int ctas) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE, TILE = COST_SPLIT_TILE;
    const int share = split_share(a.N, ctas);
    const CostSplitPlan pl = plan_cost_split(share);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share);
    float* pts4 = dyn + pl.pts;
    Loader ld(a, reinterpret_cast<uint64_t*>(smem_raw), dyn + pl.stage);
    ld.load_range<TILE>(obj, pts4, p0, p1);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    const int npair = (p1 - p0 + 1) >> 1;
    for (int t = 0; t * TILE < a.S_eval; ++t) {
        const int s = t * TILE + tid;
        float part = 0.f;
        if (s < a.S_eval) {
            float pose[PD];
#pragma unroll
            for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + ((size_t)s * a.B + obj) * PD + k);
            part = pose_cost_pairs<DOF>(pts4, 0, npair, pose, cam, delta);
        }
        // tiles alternate between the two halves of xbuf: one cluster barrier per tile (a half is written again two tiles
        // later, after the next barrier, which rank 0 reaches only once its reads of this tile are done)
        float* x = dyn + pl.xbuf + (t & 1) * TILE + tid;
        *x = part;
        cluster_sync();
        if (rank == 0 && s < a.S_eval) {
            a.cost_out[(size_t)s * a.B + obj] = sum_ranks(x, ctas);
            SPLIT_AUDIT_STORES(1);
        }
    }
    cluster_sync();                         // no CTA leaves while rank 0 may still read its shared memory
}

// ------------------------------------------------------------------------------------------------
// Random-sample LM initialiser (RSLMSolver.solve, levenberg_marquardt.py:300-353) for one object per CTA:
// thread <-> hypothesis.  A thread runs the whole LM / GN iteration of its hypothesis serially over that
// hypothesis' n sampled correspondences (read out of the object's resident pair records: the (P*B, n, .) gathered
// copies, the P-fold repeated cameras and the P*B tiny solves of the reference do not exist), scores the result
// on ALL N points with the same sweep the AMIS loop uses, and the CTA keeps the cheapest hypothesis.
struct RslmArgs {
    KArgs k;                    // correspondences, camera, bounds, delta, B, N, LM parameters
    const int* inds;            // (P, B, n) indices of the sampled correspondences, within the object
    const float* start;         // (P, B, D) starting poses
    float* pose_best;           // (B, D)
    float* cost_best;           // (B)
    float* pose_all;            // [opt] (P, B, D)
    float* cost_all;            // [opt] (P, B)
    int P, n;
};

// Order of torch.min over the hypotheses (levenberg_marquardt.py:350): a NaN cost wins (min propagates NaN), then the
// smaller cost, then the earlier hypothesis.
__device__ __forceinline__ bool cheaper_hypothesis(float c, int h, float wc, int wh) {
    const bool cn = (c != c), wn = (wc != wc);
    if (cn != wn) return cn;
    if (cn) return h < wh;
    return c < wc || (c == wc && h < wh);
}

template <int DOF, bool CLIP>
__device__ __forceinline__ void eval_subset(const float* pts, const int* idx, int n, const float* pose, const Cam& cam,
                                            float delta, float huber_eps, float* acc) {
    // the LM kernel's per-point arithmetic (row-packed, explicitly rounded): no contraction is left to the compiler
    constexpr int NP = Dim<DOF>::NV - 1;
    float R[9];
    pose_to_rot<DOF>(pose, R);
    V2 acc2[NP];
#pragma unroll
    for (int i = 0; i < NP; ++i) acc2[i] = v2splat(0.f);
    const V2 kuv[3] = {v2(cam.k[0], cam.k[3]), v2(cam.k[1], cam.k[4]), v2(cam.k[2], cam.k[5])};
    float cost = 0.f;
    for (int i = 0; i < n; ++i) {
        const int j = __ldg(idx + i);
        const float* q = pts + (j >> 1) * 16 + (j & 1);
        point_normal_eq_rows<DOF, CLIP>(R, pose, cam, kuv, delta, huber_eps, q[0], q[2], q[4], q[6], q[8], q[10], q[12],
                                        acc2, cost);
    }
#pragma unroll
    for (int i = 0; i < NP; ++i) acc[i] = acc2[i].x + acc2[i].y;
    acc[NP] = cost;
}

template <int DOF>
__global__ void __launch_bounds__(NT, 2) rslm_kernel(const RslmArgs r) {
    const KArgs& a = r.k;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts = dyn + pl.pts;
    constexpr int PD = Dim<DOF>::POSE;
    const Params& p = a.p;
    const int tid = threadIdx.x, obj = blockIdx.x;
    float* best_cost = sh.red;                                  // [NT]
    int* best_hyp = reinterpret_cast<int*>(sh.red + NT);        // [NT]
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    float my_cost = CUDART_INF_F, my_pose[PD];
    int my_hyp = -1;
    for (int h = tid; h < r.P; h += NT) {
        const int* idx = r.inds + ((size_t)h * a.B + obj) * r.n;
        LMState<DOF> s;
#pragma unroll
        for (int i = 0; i < PD; ++i) s.pose[i] = __ldg(r.start + ((size_t)h * a.B + obj) * PD + i);
        s.radius = p.initial_radius;
        s.shrink = 2.0f;
        float acc[Dim<DOF>::NV];
        if (!p.fast_mode) {
            eval_subset<DOF, true>(pts, idx, r.n, s.pose, cam, delta, p.huber_eps, acc);
            lm_adopt<DOF>(s, acc);
            if (p.lm_iter > 0) lm_propose<DOF>(s, p);
            for (int k = 0; k < p.lm_iter; ++k) {
                eval_subset<DOF, true>(pts, idx, r.n, s.pose_new, cam, delta, p.huber_eps, acc);
                lm_update<DOF>(s, acc, p);
                if (k + 1 < p.lm_iter) lm_propose<DOF>(s, p);
            }
        } else {
            for (int k = 0; k < p.lm_iter; ++k) {
                eval_subset<DOF, false>(pts, idx, r.n, s.pose, cam, delta, p.huber_eps, acc);
                gn_advance<DOF>(s.pose, acc, p.eps, s.pose);
            }
        }
        const float c = pose_cost<DOF>(pts, a.N, s.pose, cam, delta);       // score on the full set
        if (r.pose_all) {
#pragma unroll
            for (int i = 0; i < PD; ++i) r.pose_all[((size_t)h * a.B + obj) * PD + i] = s.pose[i];
        }
        if (r.cost_all) r.cost_all[(size_t)h * a.B + obj] = c;
        if (my_hyp < 0 || cheaper_hypothesis(c, h, my_cost, my_hyp)) {
            my_cost = c; my_hyp = h;
#pragma unroll
            for (int i = 0; i < PD; ++i) my_pose[i] = s.pose[i];
        }
    }
    best_cost[tid] = my_cost;
    best_hyp[tid] = my_hyp;
    __syncthreads();
    if (tid == 0) {
        int w = -1;
        for (int t = 0; t < NT; ++t) {
            if (best_hyp[t] < 0) continue;
            if (w < 0 || cheaper_hypothesis(best_cost[t], best_hyp[t], best_cost[w], best_hyp[w])) w = t;
        }
        best_hyp[0] = w;                                    // the winning THREAD (it still holds the pose)
    }
    __syncthreads();
    if (tid == best_hyp[0]) {
#pragma unroll
        for (int i = 0; i < PD; ++i) r.pose_best[(size_t)obj * PD + i] = my_pose[i];
        r.cost_best[obj] = my_cost;
    }
}

// The RSLM initialiser for objects too large for one SM (epnp_rslm_split_f32) is three launches: this kernel refines
// the hypotheses, cost_split_kernel scores them on all N points on the object's cluster, rslm_select_kernel keeps the
// cheapest.  Here one thread per (hypothesis, object) -- thread t = h B + obj, grid over P B -- runs rslm_kernel's
// iterations on the n sampled correspondences read straight from the object's global rows (nothing is staged: a
// hypothesis touches n points, not N), and writes pose_all.  A hypothesis' pose is bit-identical to rslm_kernel's:
// the iterations below are rslm_kernel's, spelled out again because sharing one inlined body changes rslm_kernel<4>'s
// register allocation (its SASS is pinned).

// One object's rows of x3d / x2d / w2d in global memory.
struct GlobalRowPoints { const float *x3d, *x2d, *w2d; };

// eval_subset on points read from global memory: the same floats go into point_normal_eq_rows as from a pair record
// (store_point keeps -u and -v; the negation is exact).
template <int DOF, bool CLIP>
__device__ __forceinline__ void eval_subset(const GlobalRowPoints& g, const int* idx, int n, const float* pose,
                                            const Cam& cam, float delta, float huber_eps, float* acc) {
    constexpr int NP = Dim<DOF>::NV - 1;
    float R[9];
    pose_to_rot<DOF>(pose, R);
    V2 acc2[NP];
#pragma unroll
    for (int i = 0; i < NP; ++i) acc2[i] = v2splat(0.f);
    const V2 kuv[3] = {v2(cam.k[0], cam.k[3]), v2(cam.k[1], cam.k[4]), v2(cam.k[2], cam.k[5])};
    float cost = 0.f;
    for (int i = 0; i < n; ++i) {
        const int j = __ldg(idx + i);
        point_normal_eq_rows<DOF, CLIP>(R, pose, cam, kuv, delta, huber_eps, __ldg(g.x3d + 3 * j), __ldg(g.x3d + 3 * j + 1),
                                        __ldg(g.x3d + 3 * j + 2), -__ldg(g.x2d + 2 * j), -__ldg(g.x2d + 2 * j + 1),
                                        __ldg(g.w2d + 2 * j), __ldg(g.w2d + 2 * j + 1), acc2, cost);
    }
#pragma unroll
    for (int i = 0; i < NP; ++i) acc[i] = acc2[i].x + acc2[i].y;
    acc[NP] = cost;
}

template <int DOF>
__global__ void __launch_bounds__(NT) rslm_refine_kernel(const RslmArgs r) {
    const KArgs& a = r.k;
    constexpr int PD = Dim<DOF>::POSE;
    const Params& p = a.p;
    const size_t t = (size_t)blockIdx.x * NT + threadIdx.x;
    if (t >= (size_t)r.P * a.B) return;
    const int obj = (int)(t % (size_t)a.B);
    const size_t row = (size_t)obj * a.N;
    const GlobalRowPoints pts{a.x3d + row * 3, a.x2d + row * 2, a.w2d + row * 2};
    const int* idx = r.inds + t * r.n;
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    LMState<DOF> s;
#pragma unroll
    for (int i = 0; i < PD; ++i) s.pose[i] = __ldg(r.start + t * PD + i);
    s.radius = p.initial_radius;
    s.shrink = 2.0f;
    float acc[Dim<DOF>::NV];
    if (!p.fast_mode) {
        eval_subset<DOF, true>(pts, idx, r.n, s.pose, cam, delta, p.huber_eps, acc);
        lm_adopt<DOF>(s, acc);
        if (p.lm_iter > 0) lm_propose<DOF>(s, p);
        for (int k = 0; k < p.lm_iter; ++k) {
            eval_subset<DOF, true>(pts, idx, r.n, s.pose_new, cam, delta, p.huber_eps, acc);
            lm_update<DOF>(s, acc, p);
            if (k + 1 < p.lm_iter) lm_propose<DOF>(s, p);
        }
    } else {
        for (int k = 0; k < p.lm_iter; ++k) {
            eval_subset<DOF, false>(pts, idx, r.n, s.pose, cam, delta, p.huber_eps, acc);
            gn_advance<DOF>(s.pose, acc, p.eps, s.pose);
        }
    }
#pragma unroll
    for (int i = 0; i < PD; ++i) r.pose_all[t * PD + i] = s.pose[i];
}

// The winner of each object over h = 0 .. P-1 by cheaper_hypothesis (torch.min's order), one thread per object:
// pose_best and cost_best are copies of its pose_all / cost_all row.
template <int DOF>
__global__ void __launch_bounds__(NT) rslm_select_kernel(const RslmArgs r) {
    constexpr int PD = Dim<DOF>::POSE;
    const int B = r.k.B, obj = blockIdx.x * NT + threadIdx.x;
    if (obj >= B) return;
    int w = 0;
    float wc = r.cost_all[obj];
    for (int h = 1; h < r.P; ++h) {
        const float c = r.cost_all[(size_t)h * B + obj];
        if (cheaper_hypothesis(c, h, wc, w)) { wc = c; w = h; }
    }
#pragma unroll
    for (int i = 0; i < PD; ++i) r.pose_best[(size_t)obj * PD + i] = r.pose_all[((size_t)w * B + obj) * PD + i];
    r.cost_best[obj] = wc;
}

// ------------------------------------------------------------------------------------------------
// Everything RSLMSolver.solve does before its solves (levenberg_marquardt.py:283-324), one CTA per object:
//   * the centre-based translation guess (center_based_init, :283-298): rays = K^-1 [u v 1] dehomogenised, direction =
//     (mean ray, 1), depth = spread of the 3D points over spread of the rays (unbiased standard deviations: y-extent
//     for 4DoF, sqrt(2/3) |std3d| / |std ray| for 6DoF) -- two block reductions over the N points; skipped when the
//     caller passes its own t_init;
//   * per hypothesis (thread <-> hypothesis) n DISTINCT correspondence indices, drawn without replacement with
//     probabilities proportional to wbar_i = mean(w2d[i, :]) -- torch.multinomial(wbar, n) (:306-312).  Same algorithm
//     as torch's: an exponential race, the n smallest of E_i / wbar_i with E_i ~ Exp(1) (Efraimidis-Spirakis); a weight
//     that is not positive is never drawn.  The race keeps its n current winners in shared memory ([slot][thread]:
//     conflict-free) with the position of the worst of them; once the list is full an element is rejected by one
//     multiply and compare (E >= 1 - u), and pays for a logarithm only when it might enter
//     (~ n (1 + ln(N / n)) times per hypothesis).  With fewer hypotheses than threads several lanes share one race;
//     the subset comes out in ascending key order (= the order of the draw);
//   * the starting pose: that translation with a uniformly random orientation -- a normalised Gaussian quaternion,
//     (1,0,0,0) when its norm is below eps (:318-324), or a yaw uniform on [0, 2 pi) (:316-317).
// Philox-4x32-10 keyed by (seed; global object index, hypothesis, block): independent of B, P tiling and launch shape.
struct RslmDrawArgs {
    const float *x3d, *x2d, *w2d, *cam;     // (B, N, 3), (B, N, 2), (B, N, 2), (B, 3, 3)
    const float* t_init;                    // [opt] (B, 3): overrides the centre-based guess
    int* inds;                              // (P, B, n)
    float* start;                           // (P, B, D)
    float* t_out;                           // [opt] (B, 3): the translation guess that was used
    uint64_t seed;
    uint32_t obj_offset;
    int P, n, B, N;
    float eps;
};

constexpr uint32_t RSLM_TAG_SUBSET = 0x52534c4du, RSLM_TAG_START = 0x52534c53u;

// The body of rslm_draw_kernel and rslm_draw_seedptr_kernel.  `r` by value: taken by reference, the inlined body
// compiles to different (validated-kernel-changing) code.
template <int DOF>
__device__ __forceinline__ void rslm_draw_body(const RslmDrawArgs r) {
    EPNP_DYN_SMEM(unsigned char, draw_smem, 16);      // its own name: as a device function it shares the others' scope
    __shared__ float red[2 * NT];
    __shared__ float t0[3];
    __shared__ int counts[NT];
    float* wbar = reinterpret_cast<float*>(draw_smem);                       // [N]
    float* keys = wbar + ((r.N + 3) & ~3);                                  // [n][NT]
    int* slots = reinterpret_cast<int*>(keys + (size_t)r.n * NT);           // [n][NT]
    constexpr int PD = Dim<DOF>::POSE;
    const int tid = threadIdx.x, obj = blockIdx.x;
    const uint32_t gobj = r.obj_offset + (uint32_t)obj;
    for (int i = tid; i < r.N; i += NT) {
        const float2 w = *reinterpret_cast<const float2*>(r.w2d + ((size_t)obj * r.N + i) * 2);
        wbar[i] = 0.5f * (w.x + w.y);
    }
    if (r.t_init) {
        if (tid < 3) t0[tid] = __ldg(r.t_init + (size_t)obj * 3 + tid);
    } else {
        // K^-1 by the adjugate (general 3x3), then mean / unbiased variance of the two ray coordinates and of x3d
        float k[9], inv[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) k[i] = __ldg(r.cam + (size_t)obj * 9 + i);
        inv[0] = k[4] * k[8] - k[5] * k[7]; inv[1] = k[2] * k[7] - k[1] * k[8]; inv[2] = k[1] * k[5] - k[2] * k[4];
        inv[3] = k[5] * k[6] - k[3] * k[8]; inv[4] = k[0] * k[8] - k[2] * k[6]; inv[5] = k[2] * k[3] - k[0] * k[5];
        inv[6] = k[3] * k[7] - k[4] * k[6]; inv[7] = k[1] * k[6] - k[0] * k[7]; inv[8] = k[0] * k[4] - k[1] * k[3];
        const float idet = 1.0f / (k[0] * inv[0] + k[1] * inv[3] + k[2] * inv[6]);
#pragma unroll
        for (int i = 0; i < 9; ++i) inv[i] *= idet;
        const float* g2 = r.x2d + (size_t)obj * r.N * 2;
        const float* g3 = r.x3d + (size_t)obj * r.N * 3;
        auto ray = [&](int i, float& rx, float& ry) {
            const float u = __ldg(g2 + 2 * i), v = __ldg(g2 + 2 * i + 1);
            const float z = fmaxf(inv[6] * u + inv[7] * v + inv[8], 1e-6f);
            rx = (inv[0] * u + inv[1] * v + inv[2]) / z;
            ry = (inv[3] * u + inv[4] * v + inv[5]) / z;
        };
        float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        for (int i = tid; i < r.N; i += NT) {
            float rx, ry;
            ray(i, rx, ry);
            m[0] += rx; m[1] += ry; m[2] += __ldg(g3 + 3 * i); m[3] += __ldg(g3 + 3 * i + 1); m[4] += __ldg(g3 + 3 * i + 2);
        }
        block_sum<5>(m, red, 0);
        const float in = 1.0f / (float)r.N;
#pragma unroll
        for (int c = 0; c < 5; ++c) m[c] *= in;
        float v[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        for (int i = tid; i < r.N; i += NT) {
            float rx, ry;
            ray(i, rx, ry);
            const float d0 = rx - m[0], d1 = ry - m[1], d2 = __ldg(g3 + 3 * i) - m[2], d3 = __ldg(g3 + 3 * i + 1) - m[3],
                        d4 = __ldg(g3 + 3 * i + 2) - m[4];
            v[0] += d0 * d0; v[1] += d1 * d1; v[2] += d2 * d2; v[3] += d3 * d3; v[4] += d4 * d4;
        }
        block_sum<5>(v, red, 1);
        if (tid == 0) {
            const float iv = 1.0f / (float)max(r.N - 1, 1);             // unbiased (torch.std's default)
            float depth;
            if (DOF == 4) depth = sqrtf(v[3] * iv) / fmaxf(sqrtf(v[1] * iv), 1e-6f);
            else depth = 0.816496580927726f * sqrtf((v[2] + v[3] + v[4]) * iv) / fmaxf(sqrtf((v[0] + v[1]) * iv), 1e-6f);
            t0[0] = m[0] * depth; t0[1] = m[1] * depth; t0[2] = depth;
        }
    }
    __syncthreads();
    if (r.t_out && tid < 3) r.t_out[(size_t)obj * 3 + tid] = t0[tid];
    const Philox ph{(uint32_t)r.seed, (uint32_t)(r.seed >> 32)};
    // Fewer hypotheses than threads: G = 2, 4 or 8 lanes (of one warp) share a hypothesis.  Lane g races the Philox blocks
    // g, g + G, ... into its own list, then lane 0 folds the other lanes' winners into its list.  The n smallest keys of a
    // hypothesis do not depend on how the race was split, and the subset is written in ascending key order -- the order
    // in which a draw without replacement produces it -- so the output does not depend on G (or P, or the batch) either.
    int G = 1;
    while (G < 8 && r.P * (2 * G) <= NT) G *= 2;
    const int per_pass = NT / G, g = tid & (G - 1), nblk = (r.N + 3) >> 2;
    for (int h0 = 0; h0 < r.P; h0 += per_pass) {
        const int h = h0 + tid / G;
        const bool live = h < r.P;
        int cnt = 0, worst = 0;
        float thr = -1.0f;                                                  // the largest key in the list
        auto offer = [&](float key, int i) {
            if (cnt < r.n) {
                keys[cnt * NT + tid] = key; slots[cnt * NT + tid] = i;
                if (key > thr) { thr = key; worst = cnt; }
                ++cnt;
            } else if (key < thr) {
                keys[worst * NT + tid] = key; slots[worst * NT + tid] = i;
                thr = -1.0f;
                for (int s = 0; s < r.n; ++s) {
                    const float k = keys[s * NT + tid];
                    if (k > thr) { thr = k; worst = s; }
                }
            }
        };
        if (live) {
            for (int blk = g; blk < nblk; blk += G) {
                uint32_t u[4];
                ph(gobj, (uint32_t)h, (uint32_t)blk, RSLM_TAG_SUBSET, u);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * blk + j;
                    if (i >= r.N) break;
                    const float w = wbar[i];
                    if (!(w > 0.0f)) continue;
                    const float uu = u01(u[j]);
                    if (cnt == r.n && (1.0f - uu) >= thr * w) continue;    // E = -log u >= 1 - u: cannot beat the worst winner
                    offer(-fast_log(uu) / w, i);
                }
            }
        }
        if (G > 1) {
            counts[tid] = cnt;
            __syncwarp();
            if (live && g == 0) {
                for (int o = 1; o < G; ++o) {
                    const int c = counts[tid + o];
                    for (int s = 0; s < c; ++s) offer(keys[s * NT + tid + o], slots[s * NT + tid + o]);
                }
            }
        }
        if (live && g == 0) {
            // ascending (key, index): insertion sort of at most n entries
            for (int a = 1; a < cnt; ++a) {
                const float k = keys[a * NT + tid];
                const int i = slots[a * NT + tid];
                int bpos = a - 1;
                while (bpos >= 0 && (keys[bpos * NT + tid] > k || (keys[bpos * NT + tid] == k && slots[bpos * NT + tid] > i))) {
                    keys[(bpos + 1) * NT + tid] = keys[bpos * NT + tid]; slots[(bpos + 1) * NT + tid] = slots[bpos * NT + tid];
                    --bpos;
                }
                keys[(bpos + 1) * NT + tid] = k; slots[(bpos + 1) * NT + tid] = i;
            }
            // fewer than n positive weights (torch.multinomial raises): complete the subset with the first unused indices
            for (int i = 0; cnt < r.n && i < r.N; ++i) {
                if (wbar[i] > 0.0f) continue;
                slots[cnt * NT + tid] = i; ++cnt;
            }
            int* out = r.inds + ((size_t)h * r.B + obj) * r.n;
            for (int s = 0; s < r.n; ++s) out[s] = slots[s * NT + tid];
            float* st = r.start + ((size_t)h * r.B + obj) * PD;
            st[0] = t0[0]; st[1] = t0[1]; st[2] = t0[2];
            uint32_t v[4];
            ph(gobj, (uint32_t)h, 0u, RSLM_TAG_START, v);
            if (DOF == 4) {
                st[3] = u01(v[0]) * 6.283185307179586f;
            } else {
                float q[4];
                box_muller(v[0], v[1], q[0], q[1]);
                box_muller(v[2], v[3], q[2], q[3]);
                const float nrm = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
                const bool tiny = nrm < r.eps;
                const float inv = 1.0f / nrm;
                st[3] = tiny ? 1.0f : q[0] * inv; st[4] = tiny ? 0.0f : q[1] * inv;
                st[5] = tiny ? 0.0f : q[2] * inv; st[6] = tiny ? 0.0f : q[3] * inv;
            }
        }
        __syncwarp();                       // lane 0 has finished reading the other lanes' lists before they are reused
    }
}

template <int DOF>
__global__ void __launch_bounds__(NT) rslm_draw_kernel(const RslmDrawArgs r) {
    rslm_draw_body<DOF>(r);
}

// rslm_draw_kernel with the seed read from device memory at entry: a CUDA graph replaying the launch draws new subsets
// and start orientations whenever the seed there changes.
template <int DOF>
__global__ void __launch_bounds__(NT) rslm_draw_seedptr_kernel(const RslmDrawArgs r, const uint64_t* seed) {
    RslmDrawArgs s = r;
    s.seed = *seed;
    rslm_draw_body<DOF>(s);
}

// ------------------------------------------------------------------------------------------------
// Backward of pose_opt_plus = pose (+) gn_step(pose) w.r.t. the correspondences and the Huber delta (the
// derivative-regularisation branch of training, LMSolver.forward :66-68 with autograd on).  One CTA per object:
// re-evaluate the normal equations, let the serial lane form step, dL/dstep (through pose_add) and
// v = -(H + eps I)^-1 dL/dstep, then thread <-> correspondence with forward-mode duals (pnp::gn_step_point_backward).
struct GnBwArgs {
    KArgs k;                    // correspondences, camera, bounds, delta, poses = pose (B, D), p.eps / huber_eps / z_min
    const float* gplus;         // (B, D)  dL/d pose_opt_plus
    float *gx3d, *gx2d, *gw2d;  // [opt] (B, N, 3|2|2)
    float* gdelta;              // [opt] (B)
};

// The serial lane of the GN-plus backward kernels: step = the damped step at the pose, v = -(H + eps I)^-1 dL/dstep.
template <int DOF>
__device__ __forceinline__ void gn_plus_step_and_v(const float* ev, const float* pose_sh, const float* gplus, float eps,
                                                   float* step, float* vvec) {
    constexpr int PD = Dim<DOF>::POSE, NA = Dim<DOF>::NA;
    float add[DOF], st[DOF], sbar[DOF], vv[DOF], gout[PD], pose[PD];
#pragma unroll
    for (int i = 0; i < DOF; ++i) add[i] = eps;
#pragma unroll
    for (int i = 0; i < PD; ++i) { pose[i] = pose_sh[i]; gout[i] = __ldg(gplus + i); }
    damped_step_refined<DOF>(ev, ev + NA, add, st);
    pose_add_backward<DOF>(pose, st, gout, sbar);
    damped_step_refined<DOF>(ev, sbar, add, vv);
#pragma unroll
    for (int i = 0; i < DOF; ++i) { step[i] = st[i]; vvec[i] = vv[i]; }
}

// The per-point pass's registers: R and t of the pose, step and v (step = [step, v], as the serial lane left them).
template <int DOF>
__device__ __forceinline__ void gn_plus_regs(const float* pose_sh, const float* step, float (&R)[9], float (&t)[3],
                                             float (&sv)[DOF], float (&vv)[DOF]) {
    constexpr int PD = Dim<DOF>::POSE;
    float ps[PD];
#pragma unroll
    for (int i = 0; i < PD; ++i) ps[i] = pose_sh[i];
    pose_to_rot<DOF>(ps, R);
    t[0] = ps[0]; t[1] = ps[1]; t[2] = ps[2];
#pragma unroll
    for (int i = 0; i < DOF; ++i) { sv[i] = step[i]; vv[i] = step[DOF + i]; }
}

template <int DOF>
__global__ void __launch_bounds__(NT, 2) gn_plus_backward_kernel(const GnBwArgs g) {
    const KArgs& a = g.k;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts = dyn + pl.pts;
    constexpr int PD = Dim<DOF>::POSE;
    const int tid = threadIdx.x, obj = blockIdx.x;
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    if (tid < PD) sh.pose[tid] = __ldg(a.poses + (size_t)obj * PD + tid);
    __syncthreads();
    eval_normal_eq<DOF, true>(pts, a.N, sh.pose, cam, delta, a.p.huber_eps, sh.red, sh.ev);
    if (tid == 0) gn_plus_step_and_v<DOF>(sh.ev, sh.pose, g.gplus + (size_t)obj * PD, a.p.eps, sh.step, sh.step + DOF);
    __syncthreads();
    float R[9], t[3], sv[DOF], vv[DOF];
    gn_plus_regs<DOF>(sh.pose, sh.step, R, t, sv, vv);
    float gd[1] = {0.f};
    for (int n = tid; n < a.N; n += NT) {
        const float* q = pts + (n >> 1) * 16 + (n & 1);
        float gr[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        gn_step_point_backward<DOF>(R, t, cam, delta, a.p.huber_eps, q[0], q[2], q[4], -q[6], -q[8], q[10], q[12], vv, sv, gr);
        const size_t o = (size_t)obj * a.N + n;
        if (g.gx3d) { g.gx3d[o * 3] = gr[0]; g.gx3d[o * 3 + 1] = gr[1]; g.gx3d[o * 3 + 2] = gr[2]; }
        if (g.gx2d) { g.gx2d[o * 2] = gr[3]; g.gx2d[o * 2 + 1] = gr[4]; }
        if (g.gw2d) { g.gw2d[o * 2] = gr[5]; g.gw2d[o * 2 + 1] = gr[6]; }
        gd[0] += gr[7];
    }
    block_sum<1>(gd, sh.red, 0);
    if (tid == 0 && g.gdelta) g.gdelta[obj] = gd[0];
}

// gn_plus_backward_kernel for objects too large for one SM, on cost_split_kernel's plan: one cluster of `ctas` CTAs per
// object (grid = B * ctas), rank r holding the points [r share, (r + 1) share) (split_share) in plan_cost_split(share),
// with the head below in the 2 x COST_SPLIT_TILE floats the cost kernel uses for its partial costs -- so C and the point
// limit are the cost kernel's.  Every rank evaluates the normal equations on its own range, reads every rank's partial
// through distributed shared memory and adds them (sum_ranks): all ranks hold the same bits of H, g and cost, and their
// serial threads form the same step and v (no broadcast).  Each rank then writes the gradient rows of its own points;
// rank 0 adds the ranks' grad_delta partials.
constexpr int GNBW_SPLIT_T = 512;
template <int DOF> struct GnBwSplitHead {
    float red[GNBW_SPLIT_T];            // eval_normal_eq / block_sum scratch
    float part[32];                     // exchange slot 1: this rank's normal equations (NV floats)
    float gdpart[4];                    // exchange slot 2: this rank's grad_delta partial
    float ev[32];                       // the normal equations of the whole object
    float pose[8];
    float step[2 * DOF];                // step, v
};
static_assert(sizeof(GnBwSplitHead<6>) <= 2 * COST_SPLIT_TILE * sizeof(float), "the head must fit the partial-cost region");

template <int DOF>
__global__ void __launch_bounds__(GNBW_SPLIT_T, 1) gn_plus_backward_split_kernel(const GnBwArgs g, const int ctas) {
    constexpr int T = GNBW_SPLIT_T;
    const KArgs& a = g.k;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE, NA = Dim<DOF>::NA, NV = Dim<DOF>::NV;
    const int share = split_share(a.N, ctas);
    const CostSplitPlan pl = plan_cost_split(share);
    GnBwSplitHead<DOF>& sh = *reinterpret_cast<GnBwSplitHead<DOF>*>(dyn + pl.xbuf);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share), cnt = p1 - p0;
    float* pts = dyn + pl.pts;
    Loader ld(a, reinterpret_cast<uint64_t*>(smem_raw), dyn + pl.stage);
    ld.load_range<T>(obj, pts, p0, p1);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    if (tid < PD) sh.pose[tid] = __ldg(a.poses + (size_t)obj * PD + tid);
    __syncthreads();
    // Pass 1.  Ordering rule 1: each exchange slot is written once, before the cluster barrier after which its peers
    // read it, and never again -- the two slots are distinct, so no rank can overwrite what another is still reading.
    eval_normal_eq<DOF, true, T>(pts, cnt, sh.pose, cam, delta, a.p.huber_eps, sh.red, sh.part);
    cluster_sync();
    if (tid < NV) sh.ev[tid] = sum_ranks(sh.part + tid, ctas);
    __syncthreads();
    float* step = sh.step;              // [DOF]
    float* vvec = sh.step + DOF;        // [DOF]
    if (tid == 0) {                     // the resident kernel's serial sequence, on every rank
        float add[DOF], st[DOF], sbar[DOF], vv[DOF], gout[PD], pose[PD];
#pragma unroll
        for (int i = 0; i < DOF; ++i) add[i] = a.p.eps;
#pragma unroll
        for (int i = 0; i < PD; ++i) { pose[i] = sh.pose[i]; gout[i] = __ldg(g.gplus + (size_t)obj * PD + i); }
        damped_step_refined<DOF>(sh.ev, sh.ev + NA, add, st);
        pose_add_backward<DOF>(pose, st, gout, sbar);
        damped_step_refined<DOF>(sh.ev, sbar, add, vv);
#pragma unroll
        for (int i = 0; i < DOF; ++i) { step[i] = st[i]; vvec[i] = vv[i]; }
    }
    __syncthreads();
    // Pass 2: thread <-> correspondence over this rank's range; every gradient row is written by the rank that owns it.
    float R[9], t[3], sv[DOF], vv[DOF];
    {
        float ps[PD];
#pragma unroll
        for (int i = 0; i < PD; ++i) ps[i] = sh.pose[i];
        pose_to_rot<DOF>(ps, R);
        t[0] = ps[0]; t[1] = ps[1]; t[2] = ps[2];
#pragma unroll
        for (int i = 0; i < DOF; ++i) { sv[i] = step[i]; vv[i] = vvec[i]; }
    }
    float gd[1] = {0.f};
    for (int n = tid; n < cnt; n += T) {
        const float* q = pts + (n >> 1) * 16 + (n & 1);
        float gr[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        gn_step_point_backward<DOF>(R, t, cam, delta, a.p.huber_eps, q[0], q[2], q[4], -q[6], -q[8], q[10], q[12], vv, sv, gr);
        const size_t o = (size_t)obj * a.N + p0 + n;
        if (g.gx3d) { g.gx3d[o * 3] = gr[0]; g.gx3d[o * 3 + 1] = gr[1]; g.gx3d[o * 3 + 2] = gr[2]; SPLIT_AUDIT_STORES(3); }
        if (g.gx2d) { g.gx2d[o * 2] = gr[3]; g.gx2d[o * 2 + 1] = gr[4]; SPLIT_AUDIT_STORES(2); }
        if (g.gw2d) { g.gw2d[o * 2] = gr[5]; g.gw2d[o * 2 + 1] = gr[6]; SPLIT_AUDIT_STORES(2); }
        gd[0] += gr[7];
    }
    block_sum<1, T>(gd, sh.red, 0);
    if (tid == 0) sh.gdpart[0] = gd[0];
    cluster_sync();
#ifdef EPNP_SPLIT_AUDIT
    for (int k = tid; k < NV + 2 * DOF; k += T) {        // H, g, cost, step and v: rank 0's bits on every rank
        const float* x = k < NV ? sh.ev + k : sh.step + (k - NV);
        if (__float_as_uint(dsmem_ld(x, 0)) != __float_as_uint(*x)) SPLIT_AUDIT_MISMATCH();
    }
#endif
    if (rank == 0 && tid == 0 && g.gdelta) {
        g.gdelta[obj] = sum_ranks(sh.gdpart, ctas);
        SPLIT_AUDIT_STORES(1);
    }
    // Ordering rule 2: a CTA's shared memory disappears when it exits; this barrier keeps every CTA of the cluster alive
    // until rank 0 has read its grad_delta partial.
    cluster_sync();
}

// residual / Jacobian / cost written out per point (API parity with evaluate_pnp's out_* tensors)
template <int DOF>
__global__ void __launch_bounds__(NT) evaluate_full_kernel(const KArgs a, float* residual, float* jac, float* cost,
                                                         int clip, float huber_eps) {
    __shared__ float red[NW];
    const int obj = blockIdx.x;
    constexpr int PD = Dim<DOF>::POSE;
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    float pose[PD], R[9];
#pragma unroll
    for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + (size_t)obj * PD + k);
    pose_to_rot<DOF>(pose, R);
    float csum = 0.f;
    for (int n = threadIdx.x; n < a.N; n += NT) {
        const size_t g = (size_t)obj * a.N + n;
        float r[2], j[2 * DOF];
        csum += point_residual_jac<DOF>(R, pose, cam, delta, huber_eps, clip != 0,
                                        a.x3d[g * 3], a.x3d[g * 3 + 1], a.x3d[g * 3 + 2],
                                        a.x2d[g * 2], a.x2d[g * 2 + 1], a.w2d[g * 2], a.w2d[g * 2 + 1], r, j);
        if (residual) { residual[g * 2] = r[0]; residual[g * 2 + 1] = r[1]; }
        if (jac) {
#pragma unroll
            for (int k = 0; k < 2 * DOF; ++k) jac[g * 2 * DOF + k] = j[k];
        }
    }
    if (cost) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) csum += __shfl_xor_sync(0xffffffffu, csum, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = csum;
        __syncthreads();
        if (threadIdx.x == 0) cost[obj] = (red[0] + red[1]) + (red[2] + red[3]);
    }
}

// ------------------------------------------------------------------------------------------------
// Backward of the Monte-Carlo cost: for every object, sum over its poses p (pose_init and all AMIS samples)
// of g[p] * d cost(pose p; x3d, x2d, w2d, delta) / d(x3d, x2d, w2d, delta).
// One CTA per object; thread <-> correspondence (up to BW_PPT per thread, accumulators in registers); the
// poses' pre-multiplied projections K[R|t] and upstream gradients are staged once in shared memory and read
// as broadcasts, so the (pose, point) loop touches no global memory.
constexpr int BW_PPT = 4;               // correspondences per thread and tile
constexpr int BW_POSE_TILE = 1024;      // poses staged per tile (13 floats each)

// Reverse mode of the cost for TWO correspondences at once (packed fp32x2; same math per half as
// pnp::point_cost_backward, with s = s2 * rsqrt(s2) and delta / s = delta * rsqrt(s2) from one MUFU.RSQ).
// g[0..2] += dL/d(X,Y,Z), g[3..4] += dL/d(u,v), g[5..6] += dL/d(wu,wv); gd += dL/d delta (both halves).
template <bool BOUNDED>
__device__ __forceinline__ void pair_cost_backward(const float (&P)[12], const Cam& cam, float delta, float gj,
                                                   float2 X, float2 Y, float2 Z, float2 nu, float2 nv, float2 wu,
                                                   float2 wv, float2 (&g)[7], float2& gd) {
    const float2 xh = v2fma(splat(P[0]), X, v2fma(splat(P[1]), Y, v2fma(splat(P[2]), Z, splat(P[3]))));
    const float2 yh = v2fma(splat(P[4]), X, v2fma(splat(P[5]), Y, v2fma(splat(P[6]), Z, splat(P[7]))));
    const float2 zh = v2fma(splat(P[8]), X, v2fma(splat(P[9]), Y, v2fma(splat(P[10]), Z, splat(P[11]))));
    const float2 iz = make_float2(FastRcp()(fmaxf(zh.x, cam.z_min)), FastRcp()(fmaxf(zh.y, cam.z_min)));
    const float2 px = v2mul(xh, iz), py = v2mul(yh, iz);
    float2 pxc = px, pyc = py;
    if (BOUNDED) {
        pxc.x = fminf(fmaxf(px.x, cam.lbx), cam.ubx); pxc.y = fminf(fmaxf(px.y, cam.lbx), cam.ubx);
        pyc.x = fminf(fmaxf(py.x, cam.lby), cam.uby); pyc.y = fminf(fmaxf(py.y, cam.lby), cam.uby);
    }
    const float2 ex = v2add(pxc, nu), ey = v2add(pyc, nv);
    const float2 rx = v2mul(ex, wu), ry = v2mul(ey, wv);
    const float2 s2 = v2fma(rx, rx, v2mul(ry, ry));
    const float2 rs = make_float2(FastRsqrt()(fmaxf(s2.x, 1e-30f)), FastRsqrt()(fmaxf(s2.y, 1e-30f)));
    const float2 s = v2mul(s2, rs);
    const bool in0 = s.x <= delta, in1 = s.y <= delta;
    const float2 ko = v2mul(splat(gj * delta), rs);                 // outlier: g * delta / s
    const float2 k = make_float2(in0 ? gj : ko.x, in1 ? gj : ko.y);
    const float2 grx = v2mul(k, rx), gry = v2mul(k, ry);
    g[5] = v2fma(grx, ex, g[5]);
    g[6] = v2fma(gry, ey, g[6]);
    const float2 gex = v2mul(grx, wu), gey = v2mul(gry, wv);
    g[3] = v2fma(gex, splat(-1.0f), g[3]);
    g[4] = v2fma(gey, splat(-1.0f), g[4]);
    float2 gpx = gex, gpy = gey;
    if (BOUNDED) {
        gpx.x = (pxc.x == px.x) ? gex.x : 0.f; gpx.y = (pxc.y == px.y) ? gex.y : 0.f;
        gpy.x = (pyc.x == py.x) ? gey.x : 0.f; gpy.y = (pyc.y == py.y) ? gey.y : 0.f;
    }
    const float2 gxh = v2mul(gpx, iz), gyh = v2mul(gpy, iz);
    const float2 tz = v2fma(gxh, px, v2mul(gyh, py));
    const float2 gzh = make_float2(zh.x >= cam.z_min ? -tz.x : 0.f, zh.y >= cam.z_min ? -tz.y : 0.f);
    g[0] = v2fma(splat(P[0]), gxh, v2fma(splat(P[4]), gyh, v2fma(splat(P[8]), gzh, g[0])));
    g[1] = v2fma(splat(P[1]), gxh, v2fma(splat(P[5]), gyh, v2fma(splat(P[9]), gzh, g[1])));
    g[2] = v2fma(splat(P[2]), gxh, v2fma(splat(P[6]), gyh, v2fma(splat(P[10]), gzh, g[2])));
    const float2 over = v2add(s, splat(-delta));
    gd = v2fma(make_float2(in0 ? 0.f : over.x, in1 ? 0.f : over.y), splat(gj), gd);
}

struct BwArgs {
    const float *x3d, *x2d, *w2d, *cam, *lb, *ub, *delta;
    const float *poses_a, *grad_a;      // (B, PA, D), (B, PA)
    const float *poses_b, *grad_b;      // [opt] (B, PB, D), (B, PB)
    float *gx3d, *gx2d, *gw2d, *gdelta;
    int B, N, PA, PB;
    float z_min;
};

template <int DOF>
__global__ void __launch_bounds__(NT, 4) cost_backward_kernel(const BwArgs a) {
    EPNP_DYN_SMEM(float, bw_smem, 16);
    float* Pm = bw_smem;                                 // [tile][12]
    float* gs = bw_smem + BW_POSE_TILE * 12;             // [tile]
    float* red = gs + BW_POSE_TILE;                      // 2 * NW * 32
    constexpr int PD = Dim<DOF>::POSE;
    const int tid = threadIdx.x;
    const int P_total = a.PA + a.PB;
    for (int obj = blockIdx.x; obj < a.B; obj += gridDim.x) {
        KArgs ka{};
        ka.cam = a.cam; ka.lb = a.lb; ka.ub = a.ub; ka.p.z_min = a.z_min;
        const Cam cam = load_cam(ka, obj);
        const float delta = __ldg(a.delta + obj);
        float2 gd2 = make_float2(0.f, 0.f);
        for (int base = 0; base < a.N; base += NT * BW_PPT) {
            // BW_PPT = 4 correspondences per thread = 2 packed pairs: pair p holds points base + (2p)*NT + tid (.x)
            // and base + (2p+1)*NT + tid (.y); out-of-range slots get zero weights (exactly zero contribution)
            constexpr int NP = BW_PPT / 2;
            float2 X[NP], Y[NP], Z[NP], nu[NP], nv[NP], wu[NP], wv[NP], g[NP][7];
#pragma unroll
            for (int k = 0; k < NP; ++k) {
                float v7[2][7];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int n = base + (2 * k + h) * NT + tid;
                    const bool ok = n < a.N;
                    const size_t q = (size_t)obj * a.N + (ok ? n : 0);
                    v7[h][0] = __ldg(a.x3d + q * 3); v7[h][1] = __ldg(a.x3d + q * 3 + 1); v7[h][2] = __ldg(a.x3d + q * 3 + 2);
                    v7[h][3] = -__ldg(a.x2d + q * 2); v7[h][4] = -__ldg(a.x2d + q * 2 + 1);
                    v7[h][5] = ok ? __ldg(a.w2d + q * 2) : 0.f; v7[h][6] = ok ? __ldg(a.w2d + q * 2 + 1) : 0.f;
                }
                X[k] = make_float2(v7[0][0], v7[1][0]); Y[k] = make_float2(v7[0][1], v7[1][1]); Z[k] = make_float2(v7[0][2], v7[1][2]);
                nu[k] = make_float2(v7[0][3], v7[1][3]); nv[k] = make_float2(v7[0][4], v7[1][4]);
                wu[k] = make_float2(v7[0][5], v7[1][5]); wv[k] = make_float2(v7[0][6], v7[1][6]);
#pragma unroll
                for (int c = 0; c < 7; ++c) g[k][c] = make_float2(0.f, 0.f);
            }
            for (int p0 = 0; p0 < P_total; p0 += BW_POSE_TILE) {
                const int np = min(BW_POSE_TILE, P_total - p0);
                __syncthreads();                          // previous tile fully consumed
                for (int j = tid; j < np; j += NT) {
                    const int pi = p0 + j;
                    const bool in_a = pi < a.PA;
                    const float* src = in_a ? a.poses_a + ((size_t)obj * a.PA + pi) * PD
                                            : a.poses_b + ((size_t)obj * a.PB + (pi - a.PA)) * PD;
                    float pose[PD], R[9], Pj[12];
#pragma unroll
                    for (int c = 0; c < PD; ++c) pose[c] = __ldg(src + c);
                    pose_to_rot<DOF>(pose, R);
                    make_proj(cam.k, R, pose, Pj);
#pragma unroll
                    for (int c = 0; c < 12; ++c) Pm[j * 12 + c] = Pj[c];
                    gs[j] = in_a ? __ldg(a.grad_a + (size_t)obj * a.PA + pi) : __ldg(a.grad_b + (size_t)obj * a.PB + (pi - a.PA));
                }
                __syncthreads();
                for (int j = 0; j < np; ++j) {
                    const float4 r0 = reinterpret_cast<const float4*>(Pm)[3 * j];
                    const float4 r1 = reinterpret_cast<const float4*>(Pm)[3 * j + 1];
                    const float4 r2 = reinterpret_cast<const float4*>(Pm)[3 * j + 2];
                    const float Pj[12] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
                    const float gj = gs[j];
#pragma unroll
                    for (int k = 0; k < NP; ++k) {
                        if (cam.bounded) pair_cost_backward<true>(Pj, cam, delta, gj, X[k], Y[k], Z[k], nu[k], nv[k], wu[k], wv[k], g[k], gd2);
                        else pair_cost_backward<false>(Pj, cam, delta, gj, X[k], Y[k], Z[k], nu[k], nv[k], wu[k], wv[k], g[k], gd2);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < NP; ++k) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int n = base + (2 * k + h) * NT + tid;
                    if (n < a.N) {
                        const size_t q = (size_t)obj * a.N + n;
                        auto pick = [&](int c) { return h == 0 ? g[k][c].x : g[k][c].y; };
                        if (a.gx3d) { a.gx3d[q * 3] = pick(0); a.gx3d[q * 3 + 1] = pick(1); a.gx3d[q * 3 + 2] = pick(2); }
                        if (a.gx2d) { a.gx2d[q * 2] = pick(3); a.gx2d[q * 2 + 1] = pick(4); }
                        if (a.gw2d) { a.gw2d[q * 2] = pick(5); a.gw2d[q * 2 + 1] = pick(6); }
                    }
                }
            }
        }
        const float gdelta = gd2.x + gd2.y;
        // padded (n >= N) lanes carry zero weights: their residual is 0 -> inlier -> no delta contribution
        float gd[1] = {gdelta};
        __syncthreads();
        block_sum<1>(gd, red, 0);
        if (tid == 0 && a.gdelta) a.gdelta[obj] = gd[0];
    }
}

// ------------------------------------------------------------------------------------------------
// Backward of the cost with respect to the POSE: grad_pose[b, p] = grad[b, p] * d cost(pose[b, p]) / d pose[b, p] for
// stacked poses given object-major.  The shape of the work is cost_kernel's: one CTA per object, its points resident as
// pair records, thread <-> pose, every thread sweeping all points as shared-memory broadcasts.  Each thread owns its
// output row: no atomics, no cross-thread sum, so a row depends on nothing but its object and its pose.
// Per point the sweep takes the forward chain of pair_cost_backward and stops at h = d cost / d (xh, yh, zh), the
// gradient in homogeneous image coordinates K x_cam (zero where the reference's autograd gives zero: no gradient
// through a depth clamped at z_min, none through a coordinate clamped at lb / ub, none at s = 0; rho' = 1 up to delta,
// delta / s above).  It accumulates 12 sums per pose, the same for both DOF: sum h (3) and sum h x3d^T (3 x 3).  After
// the sweep d cost / d t = K^T sum h, G = d cost / d R = K^T sum h x3d^T, and the rotation parameters get <G, dR/dq_k>
// for the four raw components of the un-normalised quat_to_rot (not a tangent vector), or <G, dR/dyaw>.
struct PoseBwArgs {
    KArgs k;                    // correspondences, camera, bounds, delta, poses = (B, P, D) object-major, p.z_min
    const float* grad;          // (B, P)  dL/d cost
    float* gpose;               // (B, P, D)
    int P;
};

template <bool BOUNDED>
__device__ __forceinline__ void pair_pose_grad(const float (&P)[12], const Cam& cam, float delta, const float4 q0,
                                               const float4 q1, const float4 q2, const float4 q3, float2 (&h)[12]) {
    const float2 X = make_float2(q0.x, q0.y), Y = make_float2(q0.z, q0.w), Z = make_float2(q1.x, q1.y);
    const float2 nu = make_float2(q1.z, q1.w), nv = make_float2(q2.x, q2.y);
    const float2 wu = make_float2(q2.z, q2.w), wv = make_float2(q3.x, q3.y);
    const float2 xh = v2fma(splat(P[0]), X, v2fma(splat(P[1]), Y, v2fma(splat(P[2]), Z, splat(P[3]))));
    const float2 yh = v2fma(splat(P[4]), X, v2fma(splat(P[5]), Y, v2fma(splat(P[6]), Z, splat(P[7]))));
    const float2 zh = v2fma(splat(P[8]), X, v2fma(splat(P[9]), Y, v2fma(splat(P[10]), Z, splat(P[11]))));
    const float2 iz = make_float2(FastRcp()(fmaxf(zh.x, cam.z_min)), FastRcp()(fmaxf(zh.y, cam.z_min)));
    const float2 px = v2mul(xh, iz), py = v2mul(yh, iz);
    float2 pxc = px, pyc = py;
    if (BOUNDED) {
        pxc.x = fminf(fmaxf(px.x, cam.lbx), cam.ubx); pxc.y = fminf(fmaxf(px.y, cam.lbx), cam.ubx);
        pyc.x = fminf(fmaxf(py.x, cam.lby), cam.uby); pyc.y = fminf(fmaxf(py.y, cam.lby), cam.uby);
    }
    const float2 rx = v2mul(v2add(pxc, nu), wu), ry = v2mul(v2add(pyc, nv), wv);
    const float2 s2 = v2fma(rx, rx, v2mul(ry, ry));
    const float2 rs = make_float2(FastRsqrt()(fmaxf(s2.x, 1e-30f)), FastRsqrt()(fmaxf(s2.y, 1e-30f)));
    const float2 s = v2mul(s2, rs);
    const float2 k = make_float2(s.x <= delta ? 1.f : delta * rs.x, s.y <= delta ? 1.f : delta * rs.y);    // rho'
    float2 gpx = v2mul(v2mul(k, rx), wu), gpy = v2mul(v2mul(k, ry), wv);
    if (BOUNDED) {
        gpx.x = (pxc.x == px.x) ? gpx.x : 0.f; gpx.y = (pxc.y == px.y) ? gpx.y : 0.f;
        gpy.x = (pyc.x == py.x) ? gpy.x : 0.f; gpy.y = (pyc.y == py.y) ? gpy.y : 0.f;
    }
    const float2 gxh = v2mul(gpx, iz), gyh = v2mul(gpy, iz);
    const float2 tz = v2fma(gxh, px, v2mul(gyh, py));
    const float2 gzh = make_float2(zh.x >= cam.z_min ? -tz.x : 0.f, zh.y >= cam.z_min ? -tz.y : 0.f);
    h[0] = v2add(h[0], gxh); h[1] = v2add(h[1], gyh); h[2] = v2add(h[2], gzh);
    h[3] = v2fma(gxh, X, h[3]); h[4] = v2fma(gxh, Y, h[4]); h[5] = v2fma(gxh, Z, h[5]);
    h[6] = v2fma(gyh, X, h[6]); h[7] = v2fma(gyh, Y, h[7]); h[8] = v2fma(gyh, Z, h[8]);
    h[9] = v2fma(gzh, X, h[9]); h[10] = v2fma(gzh, Y, h[10]); h[11] = v2fma(gzh, Z, h[11]);
}

// hs = the 12 sums of `pose` over the pair records [0, npair)
template <int DOF>
__device__ __forceinline__ void pose_grad_sums(const float* pts, int npair, const float* pose, const Cam& cam,
                                               float delta, float (&hs)[12]) {
    float R[9], P[12];
    pose_to_rot<DOF>(pose, R);
    make_proj(cam.k, R, pose, P);
    float2 h[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) h[k] = splat(0.f);
    const float4* q = reinterpret_cast<const float4*>(pts);
    if (cam.bounded) {
        for (int j = 0; j < npair; ++j) pair_pose_grad<true>(P, cam, delta, q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3], h);
    } else {
        for (int j = 0; j < npair; ++j) pair_pose_grad<false>(P, cam, delta, q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3], h);
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) hs[k] = h[k].x + h[k].y;
}

// The contraction after the sweep: out[0..D) = up * d cost / d pose from the 12 sums.
template <int DOF>
__device__ __forceinline__ void pose_grad_contract(const float (&hs)[12], const float* pose, const Cam& cam, float up,
                                                   float* out) {
    const float* K = cam.k;
    float G[9];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        out[i] = up * (K[i] * hs[0] + K[3 + i] * hs[1] + K[6 + i] * hs[2]);
#pragma unroll
        for (int c = 0; c < 3; ++c) G[i * 3 + c] = K[i] * hs[3 + c] + K[3 + i] * hs[6 + c] + K[6 + i] * hs[9 + c];
    }
    if (DOF == 6) {
        // dR/dw = 2 [w -z y; z w -x; -y x w]   dR/dx = 2 [x y z; y -x -w; z w -x]
        // dR/dy = 2 [-y x w; x y z; -w z -y]   dR/dz = 2 [-z -w x; w -z y; x y z]      (quat_to_rot, q = [w x y z])
        const float w = pose[3], x = pose[4], y = pose[5], z = pose[6];
        const float a01 = G[1] + G[3], a02 = G[2] + G[6], a12 = G[5] + G[7];        // symmetric parts
        const float d10 = G[3] - G[1], d02 = G[2] - G[6], d21 = G[7] - G[5];        // antisymmetric parts
        out[3] = 2.f * up * (w * (G[0] + G[4] + G[8]) + x * d21 + y * d02 + z * d10);
        out[4] = 2.f * up * (x * (G[0] - G[4] - G[8]) + w * d21 + y * a01 + z * a02);
        out[5] = 2.f * up * (y * (G[4] - G[0] - G[8]) + w * d02 + x * a01 + z * a12);
        out[6] = 2.f * up * (z * (G[8] - G[0] - G[4]) + w * d10 + x * a02 + y * a12);
    } else {
        // R = [c 0 s; 0 1 0; -s 0 c]: dR/dyaw = [-s 0 c; 0 0 0; -c 0 -s]
        float sn, cs;
        sincosf(pose[3], &sn, &cs);
        out[3] = up * (cs * (G[2] - G[6]) - sn * (G[0] + G[8]));
    }
}

template <int DOF>
__global__ void __launch_bounds__(NT, 4) cost_pose_backward_kernel(const PoseBwArgs g) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const KArgs& a = g.k;
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts = dyn + pl.pts;
    constexpr int PD = Dim<DOF>::POSE;
    const int obj = blockIdx.x;
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    for (int p = threadIdx.x; p < g.P; p += NT) {
        const size_t row = (size_t)obj * g.P + p;
        float pose[PD], hs[12], out[PD];
#pragma unroll
        for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + row * PD + k);
        pose_grad_sums<DOF>(pts, (a.N + 1) >> 1, pose, cam, delta, hs);
        pose_grad_contract<DOF>(hs, pose, cam, __ldg(g.grad + row), out);
#pragma unroll
        for (int k = 0; k < PD; ++k) g.gpose[row * PD + k] = out[k];
    }
}

// cost_pose_backward_kernel for objects too large for one SM, on cost_split_kernel's plan and cluster size: rank r
// holds the points [r share, (r + 1) share) and sweeps them for a tile of COST_SPLIT_TILE poses (one per thread).  The
// 12 sums of a pose cross ranks through the staging ring, which is free once the points are loaded and holds them for
// POSE_BW_PASS poses: the tile is exchanged pass by pass -- the pass's threads write their sums, a cluster barrier,
// rank 0 adds the ranks' sums (sum_ranks), contracts and stores, a second barrier frees the slot.
constexpr int POSE_BW_PASS = 128;
static_assert(12 * POSE_BW_PASS <= 2 * STAGE_FLOATS, "a pass's sums must fit the staging ring");
static_assert(COST_SPLIT_TILE % POSE_BW_PASS == 0, "whole passes per tile");

template <int DOF>
__global__ void __launch_bounds__(COST_SPLIT_TILE, 1) cost_pose_backward_split_kernel(const PoseBwArgs g, const int ctas) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE, TILE = COST_SPLIT_TILE;
    const KArgs& a = g.k;
    const int share = split_share(a.N, ctas);
    const CostSplitPlan pl = plan_cost_split(share);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share);
    float* pts = dyn + pl.pts;
    float* slot = dyn + pl.stage;                       // [12][POSE_BW_PASS]
    Loader ld(a, reinterpret_cast<uint64_t*>(smem_raw), dyn + pl.stage);
    ld.load_range<TILE>(obj, pts, p0, p1);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    const int npair = (p1 - p0 + 1) >> 1;
    for (int t0 = 0; t0 < g.P; t0 += TILE) {
        const int p = t0 + tid;
        const size_t row = (size_t)obj * g.P + (p < g.P ? p : 0);
        float pose[PD], hs[12];
#pragma unroll
        for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + row * PD + k);
        if (p < g.P) pose_grad_sums<DOF>(pts, npair, pose, cam, delta, hs);
        const int in_tile = min(TILE, g.P - t0);
        for (int q0 = 0; q0 < in_tile; q0 += POSE_BW_PASS) {
            const bool mine = tid >= q0 && tid < q0 + POSE_BW_PASS && p < g.P;
            float* x = slot + (tid - q0);
            if (mine) {
#pragma unroll
                for (int k = 0; k < 12; ++k) x[k * POSE_BW_PASS] = hs[k];
            }
            cluster_sync();
            if (rank == 0 && mine) {
                float sum[12], out[PD];
#pragma unroll
                for (int k = 0; k < 12; ++k) sum[k] = sum_ranks(x + k * POSE_BW_PASS, ctas);
                pose_grad_contract<DOF>(sum, pose, cam, __ldg(g.grad + row), out);
#pragma unroll
                for (int k = 0; k < PD; ++k) g.gpose[row * PD + k] = out[k];
                SPLIT_AUDIT_STORES(PD);
            }
            cluster_sync();                             // the slot is read: the next pass may write it, or a CTA leave
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Backward of the cost with respect to the CAMERA: sum_p g[b, p] * d cost(pose[b, p]) / d (K_b, lb_b, ub_b) over the
// two pose sets of BwArgs (A: (B, PA, D) with (B, PA) upstream; B [opt]: (B, PB, D) with (B, PB)), so the Monte-Carlo
// backward (the samples with -dL/dlogw and the cost_init pose) is one launch.  cost_pose_backward_kernel's shape: one
// CTA per object, thread <-> pose.  Per point pair_camera_grad takes pair_pose_grad's chain to the same 12 sums of
// h = d cost / d (xh, yh, zh) and adds four: the gradient with respect to a clamped coordinate, which the pose path
// drops, goes to the bound that clamped it (torch.maximum / torch.minimum in the reference).  Since x_h = K (R X + t),
// d cost / d K = (sum h X^T) R^T + (sum h) t^T is linear in the sums: after each pose's sweep they contract to 13 values
// (K row-major, then lbx lby ubx uby) times the pose's upstream, and each thread adds them over its own poses.  One
// fixed-order block reduction per object, no atomics: the result depends on neither B nor the loader.
constexpr int CAM_GRADS = 13;
struct CamBwArgs {
    KArgs k;                            // correspondences, camera, bounds, delta, p.z_min
    const float *poses_a, *grad_a;      // (B, PA, D), (B, PA)
    const float *poses_b, *grad_b;      // [opt] (B, PB, D), (B, PB)
    float *gcam, *glb, *gub;            // [opt] (B, 3, 3), (B, 2), (B, 2)
    int PA, PB;
};

template <bool BOUNDED>
__device__ __forceinline__ void pair_camera_grad(const float (&P)[12], const Cam& cam, float delta, const float4 q0,
                                                 const float4 q1, const float4 q2, const float4 q3, float2 (&h)[16]) {
    const float2 X = make_float2(q0.x, q0.y), Y = make_float2(q0.z, q0.w), Z = make_float2(q1.x, q1.y);
    const float2 nu = make_float2(q1.z, q1.w), nv = make_float2(q2.x, q2.y);
    const float2 wu = make_float2(q2.z, q2.w), wv = make_float2(q3.x, q3.y);
    const float2 xh = v2fma(splat(P[0]), X, v2fma(splat(P[1]), Y, v2fma(splat(P[2]), Z, splat(P[3]))));
    const float2 yh = v2fma(splat(P[4]), X, v2fma(splat(P[5]), Y, v2fma(splat(P[6]), Z, splat(P[7]))));
    const float2 zh = v2fma(splat(P[8]), X, v2fma(splat(P[9]), Y, v2fma(splat(P[10]), Z, splat(P[11]))));
    const float2 iz = make_float2(FastRcp()(fmaxf(zh.x, cam.z_min)), FastRcp()(fmaxf(zh.y, cam.z_min)));
    const float2 px = v2mul(xh, iz), py = v2mul(yh, iz);
    float2 pxc = px, pyc = py;
    if (BOUNDED) {
        pxc.x = fminf(fmaxf(px.x, cam.lbx), cam.ubx); pxc.y = fminf(fmaxf(px.y, cam.lbx), cam.ubx);
        pyc.x = fminf(fmaxf(py.x, cam.lby), cam.uby); pyc.y = fminf(fmaxf(py.y, cam.lby), cam.uby);
    }
    const float2 rx = v2mul(v2add(pxc, nu), wu), ry = v2mul(v2add(pyc, nv), wv);
    const float2 s2 = v2fma(rx, rx, v2mul(ry, ry));
    const float2 rs = make_float2(FastRsqrt()(fmaxf(s2.x, 1e-30f)), FastRsqrt()(fmaxf(s2.y, 1e-30f)));
    const float2 s = v2mul(s2, rs);
    const float2 k = make_float2(s.x <= delta ? 1.f : delta * rs.x, s.y <= delta ? 1.f : delta * rs.y);    // rho'
    float2 gpx = v2mul(v2mul(k, rx), wu), gpy = v2mul(v2mul(k, ry), wv);
    if (BOUNDED) {
        // a clamped coordinate equals the bound it sits on: ub when it is ub (the outer min), else lb
        const bool cx0 = pxc.x != px.x, cx1 = pxc.y != px.y, cy0 = pyc.x != py.x, cy1 = pyc.y != py.y;
        const bool ux0 = pxc.x == cam.ubx, ux1 = pxc.y == cam.ubx, uy0 = pyc.x == cam.uby, uy1 = pyc.y == cam.uby;
        h[12] = v2add(h[12], make_float2(cx0 && !ux0 ? gpx.x : 0.f, cx1 && !ux1 ? gpx.y : 0.f));
        h[13] = v2add(h[13], make_float2(cy0 && !uy0 ? gpy.x : 0.f, cy1 && !uy1 ? gpy.y : 0.f));
        h[14] = v2add(h[14], make_float2(cx0 && ux0 ? gpx.x : 0.f, cx1 && ux1 ? gpx.y : 0.f));
        h[15] = v2add(h[15], make_float2(cy0 && uy0 ? gpy.x : 0.f, cy1 && uy1 ? gpy.y : 0.f));
        gpx.x = cx0 ? 0.f : gpx.x; gpx.y = cx1 ? 0.f : gpx.y;
        gpy.x = cy0 ? 0.f : gpy.x; gpy.y = cy1 ? 0.f : gpy.y;
    }
    const float2 gxh = v2mul(gpx, iz), gyh = v2mul(gpy, iz);
    const float2 tz = v2fma(gxh, px, v2mul(gyh, py));
    const float2 gzh = make_float2(zh.x >= cam.z_min ? -tz.x : 0.f, zh.y >= cam.z_min ? -tz.y : 0.f);
    h[0] = v2add(h[0], gxh); h[1] = v2add(h[1], gyh); h[2] = v2add(h[2], gzh);
    h[3] = v2fma(gxh, X, h[3]); h[4] = v2fma(gxh, Y, h[4]); h[5] = v2fma(gxh, Z, h[5]);
    h[6] = v2fma(gyh, X, h[6]); h[7] = v2fma(gyh, Y, h[7]); h[8] = v2fma(gyh, Z, h[8]);
    h[9] = v2fma(gzh, X, h[9]); h[10] = v2fma(gzh, Y, h[10]); h[11] = v2fma(gzh, Z, h[11]);
}

// acc += up * d cost(pose) / d (K, lb, ub) over the pair records [0, npair): the 16 sums, then their contraction
template <int DOF>
__device__ __forceinline__ void camera_grad_pose(const float* pts, int npair, const float* pose, const Cam& cam,
                                                 float delta, float up, float (&acc)[CAM_GRADS]) {
    float R[9], P[12];
    pose_to_rot<DOF>(pose, R);
    make_proj(cam.k, R, pose, P);
    float2 h[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) h[k] = splat(0.f);
    const float4* q = reinterpret_cast<const float4*>(pts);
    if (cam.bounded) {
        for (int j = 0; j < npair; ++j) pair_camera_grad<true>(P, cam, delta, q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3], h);
    } else {
        for (int j = 0; j < npair; ++j) pair_camera_grad<false>(P, cam, delta, q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3], h);
    }
    float hs[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) hs[k] = h[k].x + h[k].y;
    // d cost / d K[i][j] = sum_c (sum h_i X_c) R[j][c] + (sum h_i) t_j
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            acc[i * 3 + j] += up * (hs[3 + 3 * i] * R[3 * j] + hs[4 + 3 * i] * R[3 * j + 1] + hs[5 + 3 * i] * R[3 * j + 2]
                                    + hs[i] * pose[j]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[9 + k] += up * hs[12 + k];
}

// The poses of both sets that thread threadIdx.x takes (stride T), each swept over the pair records [0, npair).
template <int DOF, int T>
__device__ __forceinline__ void camera_grad_poses(const CamBwArgs& g, int obj, const float* pts, int npair,
                                                  const Cam& cam, float delta, float (&acc)[CAM_GRADS]) {
    constexpr int PD = Dim<DOF>::POSE;
    for (int p = threadIdx.x; p < g.PA + g.PB; p += T) {
        const bool in_a = p < g.PA;
        const size_t row = in_a ? (size_t)obj * g.PA + p : (size_t)obj * g.PB + (p - g.PA);
        const float* src = (in_a ? g.poses_a : g.poses_b) + row * PD;
        float pose[PD];
#pragma unroll
        for (int k = 0; k < PD; ++k) pose[k] = __ldg(src + k);
        camera_grad_pose<DOF>(pts, npair, pose, cam, delta, __ldg((in_a ? g.grad_a : g.grad_b) + row), acc);
    }
}

// The requested outputs of one object from its 13 totals.  Returns the number of floats stored.
__device__ __forceinline__ int store_camera_grad(float* gcam, float* glb, float* gub, int obj,
                                                 const float (&v)[CAM_GRADS]) {
    int n = 0;
    if (gcam) {
#pragma unroll
        for (int k = 0; k < 9; ++k) gcam[(size_t)obj * 9 + k] = v[k];
        n += 9;
    }
    if (glb) { glb[(size_t)obj * 2] = v[9]; glb[(size_t)obj * 2 + 1] = v[10]; n += 2; }
    if (gub) { gub[(size_t)obj * 2] = v[11]; gub[(size_t)obj * 2 + 1] = v[12]; n += 2; }
    return n;
}

template <int DOF>
__global__ void __launch_bounds__(NT, 4) cost_camera_backward_kernel(const CamBwArgs g) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const KArgs& a = g.k;
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts = dyn + pl.pts;
    const int obj = blockIdx.x;
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    float acc[CAM_GRADS];
#pragma unroll
    for (int k = 0; k < CAM_GRADS; ++k) acc[k] = 0.f;
    camera_grad_poses<DOF, NT>(g, obj, pts, (a.N + 1) >> 1, cam, delta, acc);
    block_sum<CAM_GRADS>(acc, sh.red, 0);
    if (threadIdx.x == 0) store_camera_grad(g.gcam, g.glb, g.gub, obj, acc);
}

// cost_camera_backward_kernel for objects too large for one SM, on cost_split_kernel's plan and cluster size: rank r
// sweeps its points [r share, (r + 1) share) for every pose, contracts and reduces to 13 floats in the partial-cost
// region; after a cluster barrier rank 0 adds the ranks' 13 in rank order (sum_ranks) and stores; a second barrier keeps
// every CTA resident until then.  A rank with an empty range contributes zeros and passes both barriers.  The result
// depends on ctas (the order of that sum), never on B.
template <int DOF>
__global__ void __launch_bounds__(COST_SPLIT_TILE, 1) cost_camera_backward_split_kernel(const CamBwArgs g, const int ctas) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int T = COST_SPLIT_TILE;
    const KArgs& a = g.k;
    const int share = split_share(a.N, ctas);
    const CostSplitPlan pl = plan_cost_split(share);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share);
    float* pts = dyn + pl.pts;
    float* red = dyn + pl.xbuf;                         // block_sum scratch, one half: T floats
    float* part = red + T;                              // exchange slot: this rank's 13 totals
    Loader ld(a, reinterpret_cast<uint64_t*>(smem_raw), dyn + pl.stage);
    ld.load_range<T>(obj, pts, p0, p1);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    float acc[CAM_GRADS];
#pragma unroll
    for (int k = 0; k < CAM_GRADS; ++k) acc[k] = 0.f;
    camera_grad_poses<DOF, T>(g, obj, pts, (p1 - p0 + 1) >> 1, cam, delta, acc);
    block_sum<CAM_GRADS, T>(acc, red, 0);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) part[k] = acc[k];
    }
    cluster_sync();
    if (rank == 0 && threadIdx.x == 0) {
        float v[CAM_GRADS];
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) v[k] = sum_ranks(part + k, ctas);
        const int stored = store_camera_grad(g.gcam, g.glb, g.gub, obj, v);
        SPLIT_AUDIT_STORES(stored);
        (void)stored;
    }
    cluster_sync();                                     // no CTA leaves while rank 0 may still read its slot
}

// ------------------------------------------------------------------------------------------------
// Hessian-vector product of the cost f = sum_p g_p sum_i c(pose_p, point_i; K, lb, ub, delta): the backward of the three
// cost backwards above.  One tangent v (optional parts: x3d, x2d, w2d, delta, every pose, K, lb, ub) rides along as a
// Dual<1> through the forward of one (pose, point) pair and through its reverse-mode gradient, written out for every
// input with the gates of the first-order kernels: no tangent and no gradient through a depth clamped at z_min; a clamped
// coordinate takes the tangent of the bound it sits on (ub when it equals ub, the outer min, else lb) and passes its
// gradient to that bound only; the Huber branch is the forward's (inlier c = s^2 / 2, outlier c = delta s - delta^2 / 2).
// The gradient's tangents are the Hessian's rows times v, the cost's own tangent is grad c . v.  The arithmetic is the
// math of the first-order kernels, not their instruction sequence (exact divides and square roots here).
typedef Dual<1> D1;
__device__ __forceinline__ D1 d1(float v, float d) { D1 r; r.v = v; r.d[0] = d; return r; }

struct HvpPair {
    D1 cost;
    D1 g[8];            // d c / d (X, Y, Z, u, v, wu, wv, delta)
    D1 gxc[3];          // d c / d x_cam (= d c / d t)
    D1 h[3], xc[3];     // d c / d (K x_cam) and x_cam: d c / d K = h xc^T
    D1 gb[4];           // d c / d (lbx, lby, ubx, uby)
};

__device__ __forceinline__ void pair_cost_hvp(const D1 (&R)[9], const D1 (&t)[3], const D1 (&K)[9], const D1 (&bnd)[4],
                                              const Cam& cam, const D1& delta, const D1 (&pt)[7], HvpPair& o) {
    const D1 &X = pt[0], &Y = pt[1], &Z = pt[2], &u = pt[3], &v = pt[4], &wu = pt[5], &wv = pt[6];
#pragma unroll
    for (int r = 0; r < 3; ++r) o.xc[r] = R[3 * r] * X + R[3 * r + 1] * Y + R[3 * r + 2] * Z + t[r];
    const D1 xh = K[0] * o.xc[0] + K[1] * o.xc[1] + K[2] * o.xc[2];
    const D1 yh = K[3] * o.xc[0] + K[4] * o.xc[1] + K[5] * o.xc[2];
    const D1 zh = K[6] * o.xc[0] + K[7] * o.xc[1] + K[8] * o.xc[2];
    const bool z_free = zh.v >= cam.z_min;
    const D1 iz = dual_recip(dual_gate(zh, fmaxf(zh.v, cam.z_min), z_free));
    const D1 px = xh * iz, py = yh * iz;
    D1 pxc = px, pyc = py;
    bool lx = false, ux = false, ly = false, uy = false;     // coordinate clamped at lb / at ub
    if (cam.bounded) {
        const float cx = fminf(fmaxf(px.v, cam.lbx), cam.ubx), cy = fminf(fmaxf(py.v, cam.lby), cam.uby);
        ux = cx != px.v && cx == cam.ubx; lx = cx != px.v && !ux;
        uy = cy != py.v && cy == cam.uby; ly = cy != py.v && !uy;
        if (ux || lx) pxc = ux ? bnd[2] : bnd[0];
        if (uy || ly) pyc = uy ? bnd[3] : bnd[1];
    }
    const D1 ex = pxc - u, ey = pyc - v;
    const D1 rx = ex * wu, ry = ey * wv;
    const D1 s2 = rx * rx + ry * ry;
    D1 k;
    if (sqrtf(s2.v) <= delta.v) {
        o.cost = s2 * 0.5f;
        k = dual_const<1>(1.f);
        o.g[7] = dual_const<1>(0.f);
    } else {
        const D1 s = dual_sqrt(s2);
        o.cost = delta * s - delta * delta * 0.5f;
        k = delta * dual_recip(s);
        o.g[7] = s - delta;
    }
    const D1 grx = k * rx, gry = k * ry;
    o.g[5] = grx * ex; o.g[6] = gry * ey;
    const D1 gex = grx * wu, gey = gry * wv;
    o.g[3] = gex * -1.f; o.g[4] = gey * -1.f;
    const D1 zero = dual_const<1>(0.f);
    o.gb[0] = lx ? gex : zero; o.gb[1] = ly ? gey : zero; o.gb[2] = ux ? gex : zero; o.gb[3] = uy ? gey : zero;
    o.h[0] = (lx || ux) ? zero : gex * iz;
    o.h[1] = (ly || uy) ? zero : gey * iz;
    o.h[2] = z_free ? (o.h[0] * px + o.h[1] * py) * -1.f : zero;
#pragma unroll
    for (int c = 0; c < 3; ++c) o.gxc[c] = K[c] * o.h[0] + K[3 + c] * o.h[1] + K[6 + c] * o.h[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) o.g[c] = R[c] * o.gxc[0] + R[3 + c] * o.gxc[1] + R[6 + c] * o.gxc[2];
}

struct HvpArgs {
    KArgs k;                    // correspondences, camera, bounds, delta, poses = (B, P, D) object-major, p.z_min
    const float* grad;          // (B, P)  g_p
    const float *tx3d, *tx2d, *tw2d, *tdelta, *tpose, *tcam, *tlb, *tub;          // [opt] the tangent v
    float *hx3d, *hx2d, *hw2d, *hdelta, *hpose, *hgrad, *hcam, *hlb, *hub;         // [opt] H v and grad c_p . v
    int P;
};

__device__ __forceinline__ float tan_at(const float* t, size_t i) { return t ? __ldg(t + i) : 0.f; }

// K, the bounds and delta of one object with their tangents
__device__ __forceinline__ void hvp_object(const HvpArgs& g, int obj, Cam& cam, D1 (&K)[9], D1 (&bnd)[4], D1& delta) {
    cam = load_cam(g.k, obj);
#pragma unroll
    for (int i = 0; i < 9; ++i) K[i] = d1(cam.k[i], tan_at(g.tcam, (size_t)obj * 9 + i));
    bnd[0] = d1(cam.lbx, tan_at(g.tlb, 2 * (size_t)obj)); bnd[1] = d1(cam.lby, tan_at(g.tlb, 2 * (size_t)obj + 1));
    bnd[2] = d1(cam.ubx, tan_at(g.tub, 2 * (size_t)obj)); bnd[3] = d1(cam.uby, tan_at(g.tub, 2 * (size_t)obj + 1));
    delta = d1(__ldg(g.k.delta + obj), tan_at(g.tdelta, obj));
}

__device__ __forceinline__ void hvp_point(const HvpArgs& g, size_t q, D1 (&pt)[7]) {
    const KArgs& a = g.k;
#pragma unroll
    for (int c = 0; c < 3; ++c) pt[c] = d1(__ldg(a.x3d + q * 3 + c), tan_at(g.tx3d, q * 3 + c));
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        pt[3 + c] = d1(__ldg(a.x2d + q * 2 + c), tan_at(g.tx2d, q * 2 + c));
        pt[5 + c] = d1(__ldg(a.w2d + q * 2 + c), tan_at(g.tw2d, q * 2 + c));
    }
}

// R and t of pose row `row` with their tangents; p[] the raw components (t, then w x y z or the yaw)
template <int DOF>
__device__ __forceinline__ void hvp_pose(const HvpArgs& g, size_t row, D1 (&R)[9], D1 (&t)[3], D1 (&p)[Dim<DOF>::POSE]) {
    constexpr int PD = Dim<DOF>::POSE;
#pragma unroll
    for (int k = 0; k < PD; ++k) p[k] = d1(__ldg(g.k.poses + row * PD + k), tan_at(g.tpose, row * PD + k));
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = p[i];
    if (DOF == 6) {
        const D1 &w = p[3], &x = p[4], &y = p[5], &z = p[6];
        const D1 ww = w * w, xx = x * x, yy = y * y, zz = z * z;
        R[0] = ww + xx - yy - zz; R[1] = (x * y - w * z) * 2.f; R[2] = (x * z + w * y) * 2.f;
        R[3] = (x * y + w * z) * 2.f; R[4] = ww - xx + yy - zz; R[5] = (y * z - w * x) * 2.f;
        R[6] = (x * z - w * y) * 2.f; R[7] = (y * z + w * x) * 2.f; R[8] = ww - xx - yy + zz;
    } else {
        float r[9];
        yaw_to_rot(p[3].v, r);                                  // d cos = -sin, d sin = cos
        const float dy = p[3].d[0];
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = dual_const<1>(r[i]);
        R[0].d[0] = -r[2] * dy; R[2].d[0] = r[0] * dy; R[6].d[0] = -r[0] * dy; R[8].d[0] = -r[2] * dy;
    }
}

// Point-major: one CTA per object, thread <-> point, every thread sweeping the object's poses (lifted once per tile into
// shared memory).  Writes g_p-weighted H v at the points, and reduces the delta, K and bound rows with one fixed-order
// block sum.  No atomics.
constexpr int HVP_POSE_TILE = 128;
constexpr int HVP_POSE_REC = 25;                // R, t: value and tangent (24), g_p

template <int DOF>
__global__ void __launch_bounds__(NT) cost_hvp_point_kernel(const HvpArgs g) {
    __shared__ float rec[HVP_POSE_TILE * HVP_POSE_REC];
    __shared__ float red[2 * NW * 32];
    constexpr int PD = Dim<DOF>::POSE;
    const KArgs& a = g.k;
    const int obj = blockIdx.x, tid = threadIdx.x;
    Cam cam;
    D1 K[9], bnd[4], delta;
    hvp_object(g, obj, cam, K, bnd, delta);
    float acc[14];                              // delta, K (row-major), lbx lby ubx uby
#pragma unroll
    for (int k = 0; k < 14; ++k) acc[k] = 0.f;
    for (int base = 0; base < a.N; base += NT) {
        const int n = base + tid;
        const bool ok = n < a.N;
        const size_t q = (size_t)obj * a.N + (ok ? n : 0);
        D1 pt[7];
        hvp_point(g, q, pt);
        float hp[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int p0 = 0; p0 < g.P; p0 += HVP_POSE_TILE) {
            const int np = min(HVP_POSE_TILE, g.P - p0);
            __syncthreads();                    // the previous tile is consumed
            for (int j = tid; j < np; j += NT) {
                const size_t row = (size_t)obj * g.P + p0 + j;
                D1 R[9], t[3], p[PD];
                hvp_pose<DOF>(g, row, R, t, p);
                float* r = rec + j * HVP_POSE_REC;
#pragma unroll
                for (int i = 0; i < 9; ++i) { r[2 * i] = R[i].v; r[2 * i + 1] = R[i].d[0]; }
#pragma unroll
                for (int i = 0; i < 3; ++i) { r[18 + 2 * i] = t[i].v; r[19 + 2 * i] = t[i].d[0]; }
                r[24] = __ldg(g.grad + row);
            }
            __syncthreads();
            if (!ok) continue;
            for (int j = 0; j < np; ++j) {
                const float* r = rec + j * HVP_POSE_REC;
                D1 R[9], t[3];
#pragma unroll
                for (int i = 0; i < 9; ++i) R[i] = d1(r[2 * i], r[2 * i + 1]);
#pragma unroll
                for (int i = 0; i < 3; ++i) t[i] = d1(r[18 + 2 * i], r[19 + 2 * i]);
                const float gj = r[24];
                HvpPair o;
                pair_cost_hvp(R, t, K, bnd, cam, delta, pt, o);
#pragma unroll
                for (int k = 0; k < 7; ++k) hp[k] = fmaf(gj, o.g[k].d[0], hp[k]);
                acc[0] = fmaf(gj, o.g[7].d[0], acc[0]);
#pragma unroll
                for (int i = 0; i < 3; ++i) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) acc[1 + 3 * i + c] = fmaf(gj, (o.h[i] * o.xc[c]).d[0], acc[1 + 3 * i + c]);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[10 + k] = fmaf(gj, o.gb[k].d[0], acc[10 + k]);
            }
        }
        if (ok) {
            if (g.hx3d) { g.hx3d[q * 3] = hp[0]; g.hx3d[q * 3 + 1] = hp[1]; g.hx3d[q * 3 + 2] = hp[2]; }
            if (g.hx2d) { g.hx2d[q * 2] = hp[3]; g.hx2d[q * 2 + 1] = hp[4]; }
            if (g.hw2d) { g.hw2d[q * 2] = hp[5]; g.hw2d[q * 2 + 1] = hp[6]; }
        }
    }
    block_sum<14>(acc, red, 0);
    if (tid == 0) {
        if (g.hdelta) g.hdelta[obj] = acc[0];
        float cg[CAM_GRADS];
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) cg[k] = acc[1 + k];
        store_camera_grad(g.hcam, g.hlb, g.hub, obj, cg);
    }
}

// Pose-major: thread <-> pose, every thread streaming its object's points from global memory (the same point for all
// threads of a CTA at a time: L1 broadcasts).  Per pose it sums d c / d t and G = d c / d R = sum (d c / d x_cam) X^T
// with their tangents, then contracts them with the lifted raw pose components as pose_grad_contract does: the tangent of
// that contraction times g_p is the pose's H v; the summed tangent of the cost is grad c_p . v.
template <int DOF>
__global__ void __launch_bounds__(NT) cost_hvp_pose_kernel(const HvpArgs g, const int tiles) {
    constexpr int PD = Dim<DOF>::POSE;
    const KArgs& a = g.k;
    const int obj = blockIdx.x / tiles, p = (blockIdx.x % tiles) * NT + threadIdx.x;
    if (p >= g.P) return;
    const size_t row = (size_t)obj * g.P + p;
    Cam cam;
    D1 K[9], bnd[4], delta, R[9], t[3], q[PD];
    hvp_object(g, obj, cam, K, bnd, delta);
    hvp_pose<DOF>(g, row, R, t, q);
    D1 gt[3], G[9];
#pragma unroll
    for (int i = 0; i < 3; ++i) gt[i] = dual_const<1>(0.f);
#pragma unroll
    for (int i = 0; i < 9; ++i) G[i] = dual_const<1>(0.f);
    float dc = 0.f;
    for (int n = 0; n < a.N; ++n) {
        D1 pt[7];
        hvp_point(g, (size_t)obj * a.N + n, pt);
        HvpPair o;
        pair_cost_hvp(R, t, K, bnd, cam, delta, pt, o);
        dc += o.cost.d[0];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            gt[i] = gt[i] + o.gxc[i];
#pragma unroll
            for (int c = 0; c < 3; ++c) G[3 * i + c] = G[3 * i + c] + o.gxc[i] * pt[c];
        }
    }
    D1 out[PD];
#pragma unroll
    for (int i = 0; i < 3; ++i) out[i] = gt[i];
    if (DOF == 6) {
        const D1 &w = q[3], &x = q[4], &y = q[5], &z = q[6];
        const D1 a01 = G[1] + G[3], a02 = G[2] + G[6], a12 = G[5] + G[7];
        const D1 d10 = G[3] - G[1], d02 = G[2] - G[6], d21 = G[7] - G[5];
        out[3] = (w * (G[0] + G[4] + G[8]) + x * d21 + y * d02 + z * d10) * 2.f;
        out[4] = (x * (G[0] - G[4] - G[8]) + w * d21 + y * a01 + z * a02) * 2.f;
        out[5] = (y * (G[4] - G[0] - G[8]) + w * d02 + x * a01 + z * a12) * 2.f;
        out[6] = (z * (G[8] - G[0] - G[4]) + w * d10 + x * a02 + y * a12) * 2.f;
    } else {
        float sn, cs;
        sincosf(q[3].v, &sn, &cs);
        const D1 s = d1(sn, cs * q[3].d[0]), c = d1(cs, -sn * q[3].d[0]);
        out[3] = c * (G[2] - G[6]) - s * (G[0] + G[8]);
    }
    const float gp = __ldg(g.grad + row);
    if (g.hpose) {
#pragma unroll
        for (int k = 0; k < PD; ++k) g.hpose[row * PD + k] = gp * out[k].d[0];
    }
    if (g.hgrad) g.hgrad[row] = dc;
}

// ------------------------------------------------------------------------------------------------
// The camera gradient of pose_opt_plus = pose (+) gn_step(pose): gn_plus_backward_kernel's structure (normal equations at
// the pose; the serial lane forms step and v), then thread <-> correspondence with gn_step_point_camera_backward (Dual<13>
// seeded at K and the bounds), and one block reduction of 13 floats per object.  A launch of its own, made only when the
// camera needs a gradient; gn_plus_backward's launch and outputs do not change.
struct GnCamBwArgs {
    KArgs k;                    // correspondences, camera, bounds, delta, poses = pose (B, D), p.eps / huber_eps / z_min
    const float* gplus;         // (B, D)  dL/d pose_opt_plus
    float *gcam, *glb, *gub;    // [opt] (B, 3, 3), (B, 2), (B, 2)
};

// acc += the camera gradient of the points [0, cnt) of the pair records, thread tid of T.
template <int DOF, int T>
__device__ __forceinline__ void gn_plus_camera_points(const float* pts, int cnt, const float* pose_sh, const float* step,
                                                      const Cam& cam, float delta, float huber_eps,
                                                      float (&acc)[CAM_GRADS]) {
    float R[9], t[3], sv[DOF], vv[DOF];
    gn_plus_regs<DOF>(pose_sh, step, R, t, sv, vv);
    for (int n = threadIdx.x; n < cnt; n += T) {
        const float* q = pts + (n >> 1) * 16 + (n & 1);
        gn_step_point_camera_backward<DOF>(R, t, cam, delta, huber_eps, q[0], q[2], q[4], -q[6], -q[8], q[10], q[12], vv,
                                           sv, acc);
    }
}

template <int DOF>
__global__ void __launch_bounds__(NT, 2) gn_plus_camera_backward_kernel(const GnCamBwArgs g) {
    const KArgs& a = g.k;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    ObjHead<DOF>& sh = *reinterpret_cast<ObjHead<DOF>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    const ObjPlan pl = plan_obj<DOF>(a.N);
    float* pts = dyn + pl.pts;
    constexpr int PD = Dim<DOF>::POSE;
    const int tid = threadIdx.x, obj = blockIdx.x;
    Loader ld(a, sh.bar, dyn + pl.stage);
    ld.load_object(obj, pts);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    if (tid < PD) sh.pose[tid] = __ldg(a.poses + (size_t)obj * PD + tid);
    __syncthreads();
    eval_normal_eq<DOF, true>(pts, a.N, sh.pose, cam, delta, a.p.huber_eps, sh.red, sh.ev);
    if (tid == 0) gn_plus_step_and_v<DOF>(sh.ev, sh.pose, g.gplus + (size_t)obj * PD, a.p.eps, sh.step, sh.step + DOF);
    __syncthreads();
    float acc[CAM_GRADS];
#pragma unroll
    for (int k = 0; k < CAM_GRADS; ++k) acc[k] = 0.f;
    gn_plus_camera_points<DOF, NT>(pts, a.N, sh.pose, sh.step, cam, delta, a.p.huber_eps, acc);
    block_sum<CAM_GRADS>(acc, sh.red, 0);
    if (tid == 0) store_camera_grad(g.gcam, g.glb, g.gub, obj, acc);
}

// gn_plus_camera_backward_kernel for objects too large for one SM, on gn_plus_backward_split_kernel's clusters and head
// layout: every rank reduces the normal equations of its own range, the ranks' partials are added in rank order on every
// rank (all form the same step and v), each rank reduces the 13 camera partials of its own points, and after one more
// cluster barrier rank 0 adds them in rank order and stores; a final barrier keeps every CTA resident until then.
template <int DOF> struct GnCamSplitHead {
    float red[GNBW_SPLIT_T];            // eval_normal_eq / block_sum scratch
    float part[32];                     // exchange slot 1: this rank's normal equations (NV floats)
    float cpart[16];                    // exchange slot 2: this rank's 13 camera partials
    float ev[32];                       // the normal equations of the whole object
    float pose[8];
    float step[2 * DOF];                // step, v
};
static_assert(sizeof(GnCamSplitHead<6>) <= 2 * COST_SPLIT_TILE * sizeof(float), "the head must fit the partial-cost region");

template <int DOF>
__global__ void __launch_bounds__(GNBW_SPLIT_T, 1) gn_plus_camera_backward_split_kernel(const GnCamBwArgs g,
                                                                                       const int ctas) {
    constexpr int T = GNBW_SPLIT_T;
    const KArgs& a = g.k;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE, NV = Dim<DOF>::NV;
    const int share = split_share(a.N, ctas);
    const CostSplitPlan pl = plan_cost_split(share);
    GnCamSplitHead<DOF>& sh = *reinterpret_cast<GnCamSplitHead<DOF>*>(dyn + pl.xbuf);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share), cnt = p1 - p0;
    float* pts = dyn + pl.pts;
    Loader ld(a, reinterpret_cast<uint64_t*>(smem_raw), dyn + pl.stage);
    ld.load_range<T>(obj, pts, p0, p1);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    if (tid < PD) sh.pose[tid] = __ldg(a.poses + (size_t)obj * PD + tid);
    __syncthreads();
    // each exchange slot is written once, before the cluster barrier after which its peers read it
    eval_normal_eq<DOF, true, T>(pts, cnt, sh.pose, cam, delta, a.p.huber_eps, sh.red, sh.part);
    cluster_sync();
    if (tid < NV) sh.ev[tid] = sum_ranks(sh.part + tid, ctas);
    __syncthreads();
    if (tid == 0) gn_plus_step_and_v<DOF>(sh.ev, sh.pose, g.gplus + (size_t)obj * PD, a.p.eps, sh.step, sh.step + DOF);
    __syncthreads();
    float acc[CAM_GRADS];
#pragma unroll
    for (int k = 0; k < CAM_GRADS; ++k) acc[k] = 0.f;
    gn_plus_camera_points<DOF, T>(pts, cnt, sh.pose, sh.step, cam, delta, a.p.huber_eps, acc);
    block_sum<CAM_GRADS, T>(acc, sh.red, 0);
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) sh.cpart[k] = acc[k];
    }
    cluster_sync();
#ifdef EPNP_SPLIT_AUDIT
    for (int k = tid; k < NV + 2 * DOF; k += T) {        // H, g, cost, step and v: rank 0's bits on every rank
        const float* x = k < NV ? sh.ev + k : sh.step + (k - NV);
        if (__float_as_uint(dsmem_ld(x, 0)) != __float_as_uint(*x)) SPLIT_AUDIT_MISMATCH();
    }
#endif
    if (rank == 0 && tid == 0) {
        float v[CAM_GRADS];
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) v[k] = sum_ranks(sh.cpart + k, ctas);
        const int stored = store_camera_grad(g.gcam, g.glb, g.gub, obj, v);
        SPLIT_AUDIT_STORES(stored);
        (void)stored;
    }
    cluster_sync();                                     // no CTA leaves while rank 0 may still read its slot
}

// ------------------------------------------------------------------------------------------------
// Second order through pose_opt_plus = pose (+) gn_step(pose): the backward of gn_plus_backward_kernel and
// gn_plus_camera_backward_kernel.  With f(theta, gplus) = gplus . (pose (+) step(theta)), theta = (x3d, x2d, w2d, delta,
// K, lb, ub) and the pose detached, those kernels compute grad_theta f.  Along a tangent u of theta this kernel returns
// H u = d(grad_theta f) / d theta . u for every input of theta, and J u = d pose_opt_plus / d theta . u (the derivative
// of u . grad_theta f with respect to gplus).  u rides along as a Dual<1> through the whole first-order computation:
//   1. the normal equations H = sum J~^T J~, g = sum J~^T r~ and their tangents, in one fixed-order block reduction;
//   2. the serial lane: step and dstep = -(H + eps I)^-1 (dH step + dg); sbar = pose_add_backward(step) and its tangent
//      (the second derivative of the quaternion normalisation); v = -(H + eps I)^-1 sbar and dv = -(H + eps I)^-1
//      (dH v + dsbar); J u, pose_add's tangent;
//   3. thread <-> correspondence: gn_step_vjp's scalar b . (J~ v) + a . (r~ + J~ step), a = J~ v, b = r~ + J~ step, with
//      its derivatives with respect to the point's inputs and delta (or K and the bounds) carried by a Dual<ND> whose
//      scalar is itself a Dual<1> (HD<ND>): the value parts are the first-order rows, their tangents the rows of H u.
// The gates are the first-order kernels': the depth's tangent passes iff zh >= z_min, a clamped coordinate is its bound
// (value, tangent and seed), the clip mask is constant, and each Huber side keeps its branch, huber_eps included.  A body
// of its own rather than gn_step_vjp over a generic scalar: that would put a nested Dual through pnp_math.cuh's operators,
// which every validated backward kernel is built from.  The points stream from global memory, so any N up to
// epnp_max_points_split runs; no atomics.  The arguments are HvpArgs with grad = gplus (B, D) and hgrad = J u (B, D);
// the pose fields (tpose, hpose, P) are unused.
template <int ND> struct HD {
    D1 v;
    D1 d[ND];
};
template <int ND> __device__ __forceinline__ HD<ND> hd(const D1& c) {
    HD<ND> r; r.v = c;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = dual_const<1>(0.f);
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> hd_seed(const D1& c, int k) {
    HD<ND> r = hd<ND>(c); r.d[k] = dual_const<1>(1.f); return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator+(const HD<ND>& a, const HD<ND>& b) {
    HD<ND> r; r.v = a.v + b.v;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] + b.d[i];
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator-(const HD<ND>& a, const HD<ND>& b) {
    HD<ND> r; r.v = a.v - b.v;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] - b.d[i];
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator*(const HD<ND>& a, const HD<ND>& b) {
    HD<ND> r; r.v = a.v * b.v;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.v * b.d[i] + a.d[i] * b.v;
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator*(const HD<ND>& a, const D1& b) {
    HD<ND> r; r.v = a.v * b;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] * b;
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator*(const HD<ND>& a, float c) {
    HD<ND> r; r.v = a.v * c;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] * c;
    return r;
}
template <int ND> __device__ __forceinline__ HD<ND> operator+(const HD<ND>& a, const D1& b) { HD<ND> r = a; r.v = a.v + b; return r; }
template <int ND> __device__ __forceinline__ HD<ND> operator+(const HD<ND>& a, float c) { HD<ND> r = a; r.v = a.v + c; return r; }

// The scalar operations the per-point body below needs, for S = D1 (the normal equations) and S = HD<ND>.
__device__ __forceinline__ float hval(const D1& a) { return a.v; }
template <int ND> __device__ __forceinline__ float hval(const HD<ND>& a) { return a.v.v; }
__device__ __forceinline__ D1 hconst(const D1&, float c) { return dual_const<1>(c); }
template <int ND> __device__ __forceinline__ HD<ND> hconst(const HD<ND>&, float c) { return hd<ND>(dual_const<1>(c)); }
__device__ __forceinline__ D1 hlift(const D1&, const D1& w) { return w; }
template <int ND> __device__ __forceinline__ HD<ND> hlift(const HD<ND>&, const D1& w) { return hd<ND>(w); }
__device__ __forceinline__ D1 hgate(const D1& a, float value, bool pass) { return dual_gate(a, value, pass); }
template <int ND> __device__ __forceinline__ HD<ND> hgate(const HD<ND>& a, float value, bool pass) {
    HD<ND> r; r.v = dual_gate(a.v, value, pass);
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = pass ? a.d[i] : dual_const<1>(0.f);
    return r;
}
__device__ __forceinline__ D1 hrecip(const D1& a) { return dual_recip(a); }
template <int ND> __device__ __forceinline__ HD<ND> hrecip(const HD<ND>& a) {
    HD<ND> r; r.v = dual_recip(a.v);
    const D1 k = r.v * r.v * -1.f;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] * k;
    return r;
}
__device__ __forceinline__ D1 hsqrt(const D1& a) { return dual_sqrt(a); }
template <int ND> __device__ __forceinline__ HD<ND> hsqrt(const HD<ND>& a) {            // a > 0
    HD<ND> r; r.v = dual_sqrt(a.v);
    const D1 k = dual_recip(r.v) * 0.5f;
#pragma unroll
    for (int i = 0; i < ND; ++i) r.d[i] = a.d[i] * k;
    return r;
}

// One correspondence at the detached pose (R, t), in the scalar S: the rotated point, the (clamped) projection and its
// inverse depth, the Huber-scaled residual r~ and the row factors wu sqrt(rho') / wv sqrt(rho') (0 on a clipped row).
template <class S> struct GnPt { S xr, yr, zr, iz, px, py, rx, ry, sx, sy; };

template <class S>
__device__ __forceinline__ void gn_pt_eval(const float (&R)[9], const float (&t)[3], const S (&K)[9], const S (&bnd)[4],
                                           const Cam& c, const S& delta, float huber_eps, const S (&pt)[7], GnPt<S>& o) {
    const S &X = pt[0], &Y = pt[1], &Z = pt[2], &u = pt[3], &v = pt[4], &wu = pt[5], &wv = pt[6];
    o.xr = X * R[0] + Y * R[1] + Z * R[2];
    o.yr = X * R[3] + Y * R[4] + Z * R[5];
    o.zr = X * R[6] + Y * R[7] + Z * R[8];
    const S xc = o.xr + t[0], yc = o.yr + t[1], zc = o.zr + t[2];
    const S xh = K[0] * xc + K[1] * yc + K[2] * zc;
    const S yh = K[3] * xc + K[4] * yc + K[5] * zc;
    const S zh = K[6] * xc + K[7] * yc + K[8] * zc;
    const float z = fmaxf(hval(zh), c.z_min);
    o.iz = hrecip(hgate(zh, z, hval(zh) >= c.z_min));
    o.px = xh * o.iz; o.py = yh * o.iz;
    if (c.bounded) {
        const float cx = fminf(fmaxf(hval(o.px), c.lbx), c.ubx), cy = fminf(fmaxf(hval(o.py), c.lby), c.uby);
        if (cx != hval(o.px)) o.px = cx == c.ubx ? bnd[2] : bnd[0];
        if (cy != hval(o.py)) o.py = cy == c.uby ? bnd[3] : bnd[1];
    }
    const S rx = (o.px - u) * wu, ry = (o.py - v) * wv;
    const S s2 = rx * rx + ry * ry;
    const float s = sqrtf(hval(s2)), dl = hval(delta);
    S sc = hconst(s2, 1.0f);                                // sqrt(rho') = sqrt(min(delta / max(s, eps), 1))
    if (!(s <= dl && dl >= huber_eps)) {
        const float sm = fmaxf(s, huber_eps);
        if (dl / sm < 1.0f) {
            const S sd = (s >= huber_eps && s > 0.f) ? hsqrt(s2) : hconst(s2, sm);
            sc = hsqrt(delta * hrecip(sd));
        }
    }
    o.rx = rx * sc; o.ry = ry * sc;
    const bool cz = z == c.z_min;
    const bool clip_x = cz || (c.bounded && (hval(o.px) == c.lbx || hval(o.px) == c.ubx));
    const bool clip_y = cz || (c.bounded && (hval(o.py) == c.lby || hval(o.py) == c.uby));
    o.sx = clip_x ? hconst(sc, 0.f) : wu * sc;
    o.sy = clip_y ? hconst(sc, 0.f) : wv * sc;
}

// (J~ w)_u and (J~ w)_v of that correspondence for a DOF-vector w
template <int DOF, class S>
__device__ __forceinline__ void gn_pt_jrow(const GnPt<S>& p, const S (&K)[9], const D1 (&w)[DOF], S& ju, S& jv) {
    S mx, my, mz;
    if constexpr (DOF == 6) {
        mx = (p.yr * w[5] - p.zr * w[4]) * 2.0f + w[0];
        my = (p.zr * w[3] - p.xr * w[5]) * 2.0f + w[1];
        mz = (p.xr * w[4] - p.yr * w[3]) * 2.0f + w[2];
    } else {
        mx = p.zr * w[3] + w[0];
        my = hlift(p.zr, w[1]);
        mz = p.xr * (w[3] * -1.f) + w[2];
    }
    ju = (K[0] * mx + K[1] * my + (K[2] - p.px) * mz) * p.iz * p.sx;
    jv = (K[3] * mx + K[4] * my + (K[5] - p.py) * mz) * p.iz * p.sy;
}

// hv[k] += the tangent of d(b . (J~ v) + a . (r~ + J~ step)) / d(seed k), a and b held at their values and tangents
template <int DOF, int ND>
__device__ __forceinline__ void gn_pt_hvp(const float (&R)[9], const float (&t)[3], const HD<ND> (&K)[9],
                                          const HD<ND> (&bnd)[4], const Cam& c, const HD<ND>& delta, float huber_eps,
                                          const HD<ND> (&pt)[7], const D1 (&sv)[DOF], const D1 (&vv)[DOF],
                                          float (&hv)[ND]) {
    GnPt<HD<ND>> p;
    gn_pt_eval(R, t, K, bnd, c, delta, huber_eps, pt, p);
    HD<ND> Au, Av, Bu, Bv;
    gn_pt_jrow<DOF>(p, K, vv, Au, Av);
    gn_pt_jrow<DOF>(p, K, sv, Bu, Bv);
    const D1 au = Au.v, av = Av.v, bu = p.rx.v + Bu.v, bv = p.ry.v + Bv.v;
#pragma unroll
    for (int k = 0; k < ND; ++k)
        hv[k] += (bu * Au.d[k] + au * (p.rx.d[k] + Bu.d[k]) + bv * Av.d[k] + av * (p.ry.d[k] + Bv.d[k])).d[0];
}

// pose (+) step and pose_add_backward with the step carrying its tangent (the pose and gplus are constants)
template <int DOF>
__device__ __forceinline__ void gn_hvp_quat(const float* pose, const D1* step, D1 (&q)[4], D1& inv) {
    const float w = pose[3], x = pose[4], y = pose[5], z = pose[6];
    const D1 &a = step[3], &b = step[4], &c = step[5];
    q[0] = (a * x + b * y + c * z) + w;
    q[1] = (a * -w + b * -z + c * y) + x;
    q[2] = (a * z + b * -w + c * -x) + y;
    q[3] = (a * -y + b * x + c * -w) + z;
    const D1 n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    inv = dual_recip(sqrtf(n2.v) > 1e-12f ? dual_sqrt(n2) : dual_const<1>(1e-12f));
}

template <int DOF>
__device__ __forceinline__ void gn_hvp_pose_add(const float* pose, const D1* step, D1* out) {
#pragma unroll
    for (int i = 0; i < 3; ++i) out[i] = step[i] + pose[i];
    if constexpr (DOF == 4) {
        out[3] = step[3] + pose[3];
    } else {
        D1 q[4], inv;
        gn_hvp_quat<DOF>(pose, step, q, inv);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[3 + i] = q[i] * inv;
    }
}

template <int DOF>
__device__ __forceinline__ void gn_hvp_pose_add_backward(const float* pose, const D1* step, const float* gout, D1* gstep) {
#pragma unroll
    for (int i = 0; i < 3; ++i) gstep[i] = dual_const<1>(gout[i]);
    if constexpr (DOF == 4) {
        gstep[3] = dual_const<1>(gout[3]);
    } else {
        const float w = pose[3], x = pose[4], y = pose[5], z = pose[6];
        D1 q[4], inv;
        gn_hvp_quat<DOF>(pose, step, q, inv);
        const D1 dot = (q[0] * gout[3] + q[1] * gout[4] + q[2] * gout[5] + q[3] * gout[6]) * inv * inv;
        D1 gq[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) gq[i] = (q[i] * dot * -1.f + gout[3 + i]) * inv;
        gstep[3] = gq[0] * x + gq[1] * -w + gq[2] * z + gq[3] * -y;
        gstep[4] = gq[0] * y + gq[1] * -z + gq[2] * -w + gq[3] * x;
        gstep[5] = gq[0] * z + gq[1] * y + gq[2] * -x + gq[3] * -w;
    }
}

// out = dH w + r, dH packed upper-triangular
template <int DOF>
__device__ __forceinline__ void gn_hvp_rhs(const float* dh, const float* w, const float* r, float* out) {
#pragma unroll
    for (int i = 0; i < DOF; ++i) {
        float s = r[i];
#pragma unroll
        for (int j = 0; j < DOF; ++j) s = fmaf(dh[i <= j ? tri(i, j, DOF) : tri(j, i, DOF)], w[j], s);
        out[i] = s;
    }
}

template <int DOF>
__global__ void __launch_bounds__(NT) gn_plus_hvp_kernel(const HvpArgs g) {
    constexpr int PD = Dim<DOF>::POSE, NA = Dim<DOF>::NA, NG = NA + DOF;
    __shared__ float red[2 * NW * 32];
    __shared__ float sh[4 * DOF];                           // step, dstep, v, dv
    const KArgs& a = g.k;
    const int obj = blockIdx.x, tid = threadIdx.x;
    Cam cam;
    D1 K[9], bnd[4], delta;
    hvp_object(g, obj, cam, K, bnd, delta);
    float pose[PD], R[9], t[3];
#pragma unroll
    for (int i = 0; i < PD; ++i) pose[i] = __ldg(a.poses + (size_t)obj * PD + i);
    pose_to_rot<DOF>(pose, R);
    t[0] = pose[0]; t[1] = pose[1]; t[2] = pose[2];
    // 1. H, g (packed as eval_normal_eq's ev, without the cost) and their tangents
    float hv[NG], ht[NG];
#pragma unroll
    for (int k = 0; k < NG; ++k) { hv[k] = 0.f; ht[k] = 0.f; }
    for (int n = tid; n < a.N; n += NT) {
        D1 pt[7];
        hvp_point(g, (size_t)obj * a.N + n, pt);
        GnPt<D1> p;
        gn_pt_eval(R, t, K, bnd, cam, delta, a.p.huber_eps, pt, p);
        D1 ju[DOF], jv[DOF];
#pragma unroll
        for (int i = 0; i < DOF; ++i) {
            D1 e[DOF];
#pragma unroll
            for (int j = 0; j < DOF; ++j) e[j] = dual_const<1>(i == j ? 1.f : 0.f);
            gn_pt_jrow<DOF>(p, K, e, ju[i], jv[i]);
        }
        int idx = 0;
#pragma unroll
        for (int i = 0; i < DOF; ++i) {
#pragma unroll
            for (int k = i; k < DOF; ++k) {
                const D1 h = ju[i] * ju[k] + jv[i] * jv[k];
                hv[idx] += h.v; ht[idx] += h.d[0]; ++idx;
            }
        }
#pragma unroll
        for (int i = 0; i < DOF; ++i) {
            const D1 gi = ju[i] * p.rx + jv[i] * p.ry;
            hv[NA + i] += gi.v; ht[NA + i] += gi.d[0];
        }
    }
    block_sum<NG>(hv, red, 0);
    block_sum<NG>(ht, red, 1);
    // 2. the serial lane
    if (tid == 0) {
        float add[DOF], st[DOF], ds[DOF], vv[DOF], dv[DOF], rhs[DOF], sb[DOF], gout[PD];
#pragma unroll
        for (int i = 0; i < DOF; ++i) add[i] = a.p.eps;
#pragma unroll
        for (int i = 0; i < PD; ++i) gout[i] = __ldg(g.grad + (size_t)obj * PD + i);
        damped_step_refined<DOF>(hv, hv + NA, add, st);
        gn_hvp_rhs<DOF>(ht, st, ht + NA, rhs);
        damped_step_refined<DOF>(hv, rhs, add, ds);
        D1 step[DOF], sbar[DOF];
#pragma unroll
        for (int i = 0; i < DOF; ++i) step[i] = d1(st[i], ds[i]);
        gn_hvp_pose_add_backward<DOF>(pose, step, gout, sbar);
#pragma unroll
        for (int i = 0; i < DOF; ++i) { sb[i] = sbar[i].v; rhs[i] = sbar[i].d[0]; }
        damped_step_refined<DOF>(hv, sb, add, vv);
        gn_hvp_rhs<DOF>(ht, vv, rhs, rhs);
        damped_step_refined<DOF>(hv, rhs, add, dv);
        if (g.hgrad) {
            D1 plus[PD];
            gn_hvp_pose_add<DOF>(pose, step, plus);
#pragma unroll
            for (int i = 0; i < PD; ++i) g.hgrad[(size_t)obj * PD + i] = plus[i].d[0];
        }
#pragma unroll
        for (int i = 0; i < DOF; ++i) { sh[i] = st[i]; sh[DOF + i] = ds[i]; sh[2 * DOF + i] = vv[i]; sh[3 * DOF + i] = dv[i]; }
    }
    __syncthreads();
    // 3. thread <-> correspondence
    D1 sv[DOF], vv[DOF];
#pragma unroll
    for (int i = 0; i < DOF; ++i) { sv[i] = d1(sh[i], sh[DOF + i]); vv[i] = d1(sh[2 * DOF + i], sh[3 * DOF + i]); }
    const bool pts_out = g.hx3d || g.hx2d || g.hw2d || g.hdelta, cam_out = g.hcam || g.hlb || g.hub;
    float acc[1 + CAM_GRADS];                               // delta, K (row-major), lbx lby ubx uby
#pragma unroll
    for (int k = 0; k < 1 + CAM_GRADS; ++k) acc[k] = 0.f;
    for (int n = tid; n < a.N; n += NT) {
        const size_t q = (size_t)obj * a.N + n;
        D1 pt[7];
        hvp_point(g, q, pt);
        if (pts_out) {
            HD<8> P[7], Kh[9], Bh[4];
#pragma unroll
            for (int k = 0; k < 7; ++k) P[k] = hd_seed<8>(pt[k], k);
#pragma unroll
            for (int k = 0; k < 9; ++k) Kh[k] = hd<8>(K[k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) Bh[k] = hd<8>(bnd[k]);
            float hp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            gn_pt_hvp<DOF, 8>(R, t, Kh, Bh, cam, hd_seed<8>(delta, 7), a.p.huber_eps, P, sv, vv, hp);
            if (g.hx3d) { g.hx3d[q * 3] = hp[0]; g.hx3d[q * 3 + 1] = hp[1]; g.hx3d[q * 3 + 2] = hp[2]; }
            if (g.hx2d) { g.hx2d[q * 2] = hp[3]; g.hx2d[q * 2 + 1] = hp[4]; }
            if (g.hw2d) { g.hw2d[q * 2] = hp[5]; g.hw2d[q * 2 + 1] = hp[6]; }
            acc[0] += hp[7];
        }
        if (cam_out) {
            HD<CAM_GRADS> P[7], Kh[9], Bh[4];
#pragma unroll
            for (int k = 0; k < 7; ++k) P[k] = hd<CAM_GRADS>(pt[k]);
#pragma unroll
            for (int k = 0; k < 9; ++k) Kh[k] = hd_seed<CAM_GRADS>(K[k], k);
#pragma unroll
            for (int k = 0; k < 4; ++k) Bh[k] = hd_seed<CAM_GRADS>(bnd[k], 9 + k);
            float hc[CAM_GRADS];
#pragma unroll
            for (int k = 0; k < CAM_GRADS; ++k) hc[k] = 0.f;
            gn_pt_hvp<DOF, CAM_GRADS>(R, t, Kh, Bh, cam, hd<CAM_GRADS>(delta), a.p.huber_eps, P, sv, vv, hc);
#pragma unroll
            for (int k = 0; k < CAM_GRADS; ++k) acc[1 + k] += hc[k];
        }
    }
    block_sum<1 + CAM_GRADS>(acc, red, 0);
    if (tid == 0) {
        if (g.hdelta) g.hdelta[obj] = acc[0];
        float cg[CAM_GRADS];
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) cg[k] = acc[1 + k];
        store_camera_grad(g.hcam, g.hlb, g.hub, obj, cg);
    }
}

// ------------------------------------------------------------------------------------------------
// Backward of evaluate_full_kernel's residual, Jacobian and cost at S stacked poses (S, B, D): the vector-Jacobian
// product with any of the upstream gradients g_res (S, B, 2N), g_jac (S, B, 2N, DOF) and g_cost (S, B), differentiated
// per (pose, point) by the three forms of point_residual_jac_backward (pnp_math.cuh).  One CTA per object, the points
// streamed from global memory as evaluate_full_kernel reads them, so there is no point limit and no split form.
//   1. thread <-> point, the poses in order inside the thread: the point's x3d / x2d / w2d gradients are summed over the
//      poses in registers and stored once; delta's and the camera's partials are added over the thread's points and
//      reduced by one fixed-order block_sum each.
//   2. per pose, thread <-> point again with the pose form, and one fixed-order block_sum of the D components.
// No atomics; every output element is written by one thread; an object's results depend on nothing else in the batch,
// and on which gradients were requested only through which of the passes run.
struct EvalBwArgs {
    KArgs k;                                // correspondences, camera, bounds, delta, poses (S, B, D), p.z_min / huber_eps
    const float *g_res, *g_jac, *g_cost;    // [opt] (S, B, 2N), (S, B, 2N, DOF), (S, B)
    float *gx3d, *gx2d, *gw2d, *gdelta;     // [opt] (B, N, 3|2|2), (B)
    float* gpose;                           // [opt] (S, B, D)
    float *gcam, *glb, *gub;                // [opt] (B, 3, 3), (B, 2), (B, 2)
    int S, clip;
};

// The upstream of (pose row `row` = s B + b, point n); gr / gj are left unset (and null returned) when not given.
template <int DOF>
__device__ __forceinline__ float eval_bw_upstream(const EvalBwArgs& g, size_t row, int n, float (&gr)[2],
                                                  float (&gj)[2 * DOF], const float*& pr, const float*& pj) {
    const size_t p = row * g.k.N + n;
    pr = pj = nullptr;
    if (g.g_res) { gr[0] = __ldg(g.g_res + 2 * p); gr[1] = __ldg(g.g_res + 2 * p + 1); pr = gr; }
    if (g.g_jac) {
#pragma unroll
        for (int k = 0; k < 2 * DOF; ++k) gj[k] = __ldg(g.g_jac + p * 2 * DOF + k);
        pj = gj;
    }
    return g.g_cost ? __ldg(g.g_cost + row) : 0.f;
}

template <int DOF>
__global__ void __launch_bounds__(NT) evaluate_backward_kernel(const EvalBwArgs g) {
    __shared__ float red[2 * NW * 32];
    const KArgs& a = g.k;
    constexpr int PD = Dim<DOF>::POSE;
    const int obj = blockIdx.x, tid = threadIdx.x;
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj), heps = a.p.huber_eps;
    const bool clip = g.clip != 0;
    const bool want_pts = g.gx3d || g.gx2d || g.gw2d || g.gdelta, want_cam = g.gcam || g.glb || g.gub;
    if (want_pts || want_cam) {
        float gd = 0.f, gk[CAM_GRADS];
#pragma unroll
        for (int k = 0; k < CAM_GRADS; ++k) gk[k] = 0.f;
        for (int n = tid; n < a.N; n += NT) {
            const size_t q = (size_t)obj * a.N + n;
            const float X = __ldg(a.x3d + q * 3), Y = __ldg(a.x3d + q * 3 + 1), Z = __ldg(a.x3d + q * 3 + 2);
            const float u = __ldg(a.x2d + q * 2), v = __ldg(a.x2d + q * 2 + 1);
            const float wu = __ldg(a.w2d + q * 2), wv = __ldg(a.w2d + q * 2 + 1);
            float gp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int s = 0; s < g.S; ++s) {
                const size_t row = (size_t)s * a.B + obj;
                float pose[PD], R[9], gr[2], gj[2 * DOF];
#pragma unroll
                for (int k = 0; k < PD; ++k) pose[k] = __ldg(a.poses + row * PD + k);
                pose_to_rot<DOF>(pose, R);
                const float *pr, *pj;
                const float gc = eval_bw_upstream<DOF>(g, row, n, gr, gj, pr, pj);
                if (want_pts)
                    point_residual_jac_backward<DOF>(R, pose, cam, delta, heps, clip, X, Y, Z, u, v, wu, wv, pr, pj, gc, gp);
                if (want_cam)
                    point_residual_jac_camera_backward<DOF>(R, pose, cam, delta, heps, clip, X, Y, Z, u, v, wu, wv, pr,
                                                            pj, gc, gk);
            }
            if (g.gx3d) { g.gx3d[q * 3] = gp[0]; g.gx3d[q * 3 + 1] = gp[1]; g.gx3d[q * 3 + 2] = gp[2]; }
            if (g.gx2d) { g.gx2d[q * 2] = gp[3]; g.gx2d[q * 2 + 1] = gp[4]; }
            if (g.gw2d) { g.gw2d[q * 2] = gp[5]; g.gw2d[q * 2 + 1] = gp[6]; }
            gd += gp[7];
        }
        if (want_pts) {
            float v[1] = {gd};
            block_sum<1>(v, red, 0);
            if (tid == 0 && g.gdelta) g.gdelta[obj] = v[0];
        }
        if (want_cam) {
            block_sum<CAM_GRADS>(gk, red, 1);
            if (tid == 0) store_camera_grad(g.gcam, g.glb, g.gub, obj, gk);
        }
    }
    if (!g.gpose) return;
    __syncthreads();                                    // pass 1's reductions are read: the scratch may be rewritten
    for (int s = 0; s < g.S; ++s) {
        const size_t row = (size_t)s * a.B + obj;
        float pose[PD], acc[PD];
#pragma unroll
        for (int k = 0; k < PD; ++k) { pose[k] = __ldg(a.poses + row * PD + k); acc[k] = 0.f; }
        for (int n = tid; n < a.N; n += NT) {
            const size_t q = (size_t)obj * a.N + n;
            float gr[2], gj[2 * DOF];
            const float *pr, *pj;
            const float gc = eval_bw_upstream<DOF>(g, row, n, gr, gj, pr, pj);
            point_residual_jac_pose_backward<DOF>(pose, cam, delta, heps, clip, __ldg(a.x3d + q * 3),
                                                  __ldg(a.x3d + q * 3 + 1), __ldg(a.x3d + q * 3 + 2),
                                                  __ldg(a.x2d + q * 2), __ldg(a.x2d + q * 2 + 1),
                                                  __ldg(a.w2d + q * 2), __ldg(a.w2d + q * 2 + 1), pr, pj, gc, acc);
        }
        // alternate halves: a half is rewritten only after the next reduction's barrier, which follows every read of it
        block_sum<PD>(acc, red, s & 1);
        if (tid == 0) {
#pragma unroll
            for (int k = 0; k < PD; ++k) g.gpose[row * PD + k] = acc[k];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Forward mode of evaluate_full_kernel's residual, Jacobian and cost at S stacked poses (S, B, D): the Jacobian-vector
// product with one tangent v (optional parts: x3d, x2d, w2d, delta, every pose, K, lb, ub), the transpose of what
// evaluate_backward_kernel computes.  Every input is a Dual<1> seeded with its tangent and pushed through
// point_residual_jac's formulas as residual_jac_vjp writes them, with its gates: no tangent through a depth clamped at
// z_min, a clamped coordinate takes its bound's tangent (ub when it equals ub, the outer min, else lb), the clip mask is
// constant, the Huber scale keeps its branches and huber_eps, the Jacobian's rows are differentiated as written, and
// the rotation is the forward's (ww + xx - yy - zz, ...) of the raw pose components.  A body of its own: the validated
// backwards' instantiations of residual_jac_vjp stay as they are.
struct JvpArgs {
    HvpArgs h;                  // problem, poses (S, B, D) as rows s B + b, the tangent (t_pose (S, B, D)); h.P = S
    float *dres, *djac, *dcost; // [opt] (S, B, 2N), (S, B, 2N, DOF), (S, B)
    int clip;
};

// One (pose, point): the cost with its tangent; r~ and the Jacobian's two rows (u then v) too when RJ.
template <int DOF, bool RJ>
__device__ __forceinline__ D1 point_residual_jac_jvp(const D1 (&R)[9], const D1 (&t)[3], const D1 (&K)[9],
                                                     const D1 (&bnd)[4], const Cam& cam, const D1& delta,
                                                     float huber_eps, bool clip, const D1 (&pt)[7], D1* r, D1* j) {
    const D1 &X = pt[0], &Y = pt[1], &Z = pt[2], &u = pt[3], &v = pt[4], &wu = pt[5], &wv = pt[6];
    const D1 xr = X * R[0] + Y * R[1] + Z * R[2];
    const D1 yr = X * R[3] + Y * R[4] + Z * R[5];
    const D1 zr = X * R[6] + Y * R[7] + Z * R[8];
    const D1 xc = xr + t[0], yc = yr + t[1], zc = zr + t[2];
    const D1 xh = K[0] * xc + K[1] * yc + K[2] * zc;
    const D1 yh = K[3] * xc + K[4] * yc + K[5] * zc;
    const D1 zh = K[6] * xc + K[7] * yc + K[8] * zc;
    const D1 z = dual_gate(zh, fmaxf(zh.v, cam.z_min), zh.v >= cam.z_min);
    const D1 iz = dual_recip(z);
    D1 px = xh * iz, py = yh * iz;
    if (cam.bounded) {
        const float cx = fminf(fmaxf(px.v, cam.lbx), cam.ubx), cy = fminf(fmaxf(py.v, cam.lby), cam.uby);
        if (cx != px.v) px = cx == cam.ubx ? bnd[2] : bnd[0];
        if (cy != py.v) py = cy == cam.uby ? bnd[3] : bnd[1];
    }
    const D1 rx = (px - u) * wu, ry = (py - v) * wv;
    const D1 s2 = rx * rx + ry * ry;
    const float s = sqrtf(s2.v), dl = delta.v;
    const D1 cost = s <= dl ? s2 * 0.5f : delta * dual_sqrt(s2) - delta * delta * 0.5f;
    if constexpr (RJ) {
        D1 sc = dual_const<1>(1.0f);
        if (!(s <= dl && dl >= huber_eps)) {
            const float sm = fmaxf(s, huber_eps);
            if (dl / sm < 1.0f) {
                const D1 sd = (s >= huber_eps && s > 0.f) ? dual_sqrt(s2) : dual_const<1>(sm);
                sc = dual_sqrt(dual_recip(sd) * delta);
            }
        }
        r[0] = rx * sc; r[1] = ry * sc;
        if (j) {
            const bool cz = (z.v == cam.z_min);
            const bool clip_x = clip && (cz || (cam.bounded && (px.v == cam.lbx || px.v == cam.ubx)));
            const bool clip_y = clip && (cz || (cam.bounded && (py.v == cam.lby || py.v == cam.uby)));
            const D1 sx = clip_x ? dual_const<1>(0.f) : sc * wu;
            const D1 sy = clip_y ? dual_const<1>(0.f) : sc * wv;
            D1* jx = j; D1* jy = j + DOF;
            jx[0] = K[0] * iz; jx[1] = K[1] * iz; jx[2] = (K[2] - px) * iz;
            jy[0] = K[3] * iz; jy[1] = K[4] * iz; jy[2] = (K[5] - py) * iz;
            if (DOF == 6) {
                const D1 ax = xr * 2.0f, ay = yr * 2.0f, az = zr * 2.0f;
                jx[3] = jx[1] * az - jx[2] * ay; jx[4] = jx[2] * ax - jx[0] * az; jx[5] = jx[0] * ay - jx[1] * ax;
                jy[3] = jy[1] * az - jy[2] * ay; jy[4] = jy[2] * ax - jy[0] * az; jy[5] = jy[0] * ay - jy[1] * ax;
            } else {
                jx[3] = jx[0] * zr - jx[2] * xr;
                jy[3] = jy[0] * zr - jy[2] * xr;
            }
#pragma unroll
            for (int i = 0; i < DOF; ++i) { jx[i] = jx[i] * sx; jy[i] = jy[i] * sy; }
        }
    }
    return cost;
}

// Point-major: one CTA per (pose, object) row s B + b, as evaluate_full_kernel runs one CTA per object, thread <-> point
// with the points streamed from global memory (any N).  d cost is one fixed-order block sum.
template <int DOF>
__global__ void __launch_bounds__(NT) evaluate_jvp_kernel(const JvpArgs g) {
    __shared__ float red[2 * NW * 32];
    constexpr int PD = Dim<DOF>::POSE;
    const KArgs& a = g.h.k;
    const size_t row = blockIdx.x;
    const int obj = (int)(row % a.B), tid = threadIdx.x;
    Cam cam;
    D1 K[9], bnd[4], delta, R[9], t[3], p[PD];
    hvp_object(g.h, obj, cam, K, bnd, delta);
    hvp_pose<DOF>(g.h, row, R, t, p);
    const float heps = a.p.huber_eps;
    float dc = 0.f;
    for (int n = tid; n < a.N; n += NT) {
        D1 pt[7], r[2], j[2 * DOF];
        hvp_point(g.h, (size_t)obj * a.N + n, pt);
        dc += point_residual_jac_jvp<DOF, true>(R, t, K, bnd, cam, delta, heps, g.clip != 0, pt, r,
                                                g.djac ? j : nullptr).d[0];
        const size_t o = row * a.N + n;
        if (g.dres) { g.dres[2 * o] = r[0].d[0]; g.dres[2 * o + 1] = r[1].d[0]; }
        if (g.djac) {
#pragma unroll
            for (int k = 0; k < 2 * DOF; ++k) g.djac[o * 2 * DOF + k] = j[k].d[0];
        }
    }
    if (g.dcost) {
        float v[1] = {dc};
        block_sum<1>(v, red, 0);
        if (tid == 0) g.dcost[row] = v[0];
    }
}

// Pose-major, d cost alone (many poses per object: the Monte-Carlo log-weights): thread <-> pose, grid B x tiles of NT
// poses, the object's points staged NT at a time (value and tangent) in shared memory and read as broadcasts.  Each
// pose's sum runs over the points in order.
constexpr int JVP_POSE_MAJOR_MIN_S = 64;        // below it the pose-major CTAs would be mostly idle

template <int DOF>
__global__ void __launch_bounds__(NT) evaluate_jvp_cost_kernel(const JvpArgs g, const int tiles) {
    __shared__ float pts[NT * 14];
    constexpr int PD = Dim<DOF>::POSE;
    const KArgs& a = g.h.k;
    const int obj = blockIdx.x / tiles, s = (blockIdx.x % tiles) * NT + threadIdx.x;
    const bool ok = s < g.h.P;
    const size_t row = (size_t)(ok ? s : 0) * a.B + obj;
    Cam cam;
    D1 K[9], bnd[4], delta, R[9], t[3], p[PD];
    hvp_object(g.h, obj, cam, K, bnd, delta);
    hvp_pose<DOF>(g.h, row, R, t, p);
    float dc = 0.f;
    for (int base = 0; base < a.N; base += NT) {
        const int np = min(NT, a.N - base);
        __syncthreads();                        // the previous tile is consumed
        if (threadIdx.x < np) {
            D1 pt[7];
            hvp_point(g.h, (size_t)obj * a.N + base + threadIdx.x, pt);
#pragma unroll
            for (int c = 0; c < 7; ++c) {
                pts[threadIdx.x * 14 + 2 * c] = pt[c].v;
                pts[threadIdx.x * 14 + 2 * c + 1] = pt[c].d[0];
            }
        }
        __syncthreads();
        if (!ok) continue;
        for (int i = 0; i < np; ++i) {
            D1 pt[7];
#pragma unroll
            for (int c = 0; c < 7; ++c) pt[c] = d1(pts[i * 14 + 2 * c], pts[i * 14 + 2 * c + 1]);
            dc += point_residual_jac_jvp<DOF, false>(R, t, K, bnd, cam, delta, 0.f, false, pt, nullptr, nullptr).d[0];
        }
    }
    if (ok) g.dcost[row] = dc;
}

// AdaptiveHuberPnPCost.set_param: delta = mean(w2d) * sqrt(var_x + var_y) * relative_delta
__global__ void __launch_bounds__(NT) adaptive_delta_kernel(const float* x2d, const float* w2d, float rel,
                                                          float* delta, int N) {
    __shared__ float red[2 * NW * 32];
    const int obj = blockIdx.x;
    const float2* x = reinterpret_cast<const float2*>(x2d) + (size_t)obj * N;
    const float2* w = reinterpret_cast<const float2*>(w2d) + (size_t)obj * N;
    float s[3] = {0.f, 0.f, 0.f};
    for (int n = threadIdx.x; n < N; n += NT) {
        const float2 a = x[n], b = w[n];
        s[0] += a.x; s[1] += a.y; s[2] += b.x + b.y;
    }
    block_sum<3>(s, red, 0);
    const float mx = s[0] / N, my = s[1] / N, mw = s[2] / (2.f * N);
    float v[2] = {0.f, 0.f};
    for (int n = threadIdx.x; n < N; n += NT) {
        const float2 a = x[n];
        v[0] = fmaf(a.x - mx, a.x - mx, v[0]); v[1] = fmaf(a.y - my, a.y - my, v[1]);
    }
    block_sum<2>(v, red, 1);
    if (threadIdx.x == 0) delta[obj] = mw * sqrtf((v[0] + v[1]) / (float)(N - 1)) * rel;
}

// Epilogue on the AMIS outputs (the step after the path; SURVEY.md section 8 row f4).  One CTA per object reads the
// object's M log-weights (and, for the score, the x / z components of its M pose samples) once and writes
//   lse[b]      = logsumexp_m logw[b, m]                        (Monte-Carlo pose loss: loss_pred)
//   loss[b]     = cost_target[b] + lse[b], NaN -> 0              (the per-object loss before its mean)
//   weights     = softmax_m logw[b, :]                           (Det: pose_sample_logweights.softmax(dim=0))
//   score_te[b] = sum_m weights[m] * clamp((2.5 - log2 |(x,z)_m - (x,z)_opt|) / 4, 0, 1)   (Det 'te' MC score)
// with torch's conventions at the infinities (all -inf -> lse -inf, any NaN -> NaN).
template <int PD>
__global__ void __launch_bounds__(NT) mc_epilogue_kernel(const float* logw, const float* samples, const float* pose_opt,
                                                       const float* cost_target, float* lse_out, float* loss_out,
                                                       float* weights, float* score_out, int M) {
    __shared__ float red[2 * NW * 32];
    const int obj = blockIdx.x, tid = threadIdx.x;
    const float* l = logw + (size_t)obj * M;
    float mx = -CUDART_INF_F;
    bool any_nan = false;
    for (int m = tid; m < M; m += NT) { const float v = __ldg(l + m); mx = fmaxf(mx, v); any_nan |= (v != v); }
    mx = block_max(mx, red, 0);
    const float ref = (fabsf(mx) == CUDART_INF_F) ? 0.f : mx;          // torch.logsumexp: an infinite max is not subtracted
    const bool want_score = samples != nullptr && pose_opt != nullptr && score_out != nullptr;
    float ox = 0.f, oz = 0.f;
    if (want_score) { ox = __ldg(pose_opt + (size_t)obj * PD); oz = __ldg(pose_opt + (size_t)obj * PD + 2); }
    float acc[3] = {0.f, 0.f, any_nan ? 1.f : 0.f};                    // sum e, sum e * score, NaN seen
    for (int m = tid; m < M; m += NT) {
        const float e = expf(__ldg(l + m) - ref);
        acc[0] += e;
        if (want_score) {
            const float* sp = samples + ((size_t)obj * M + m) * PD;
            const float dx = __ldg(sp) - ox, dz = __ldg(sp + 2) - oz;
            const float dev = sqrtf(fmaf(dx, dx, dz * dz));
            const float sc = fminf(fmaxf((2.5f - log2f(dev)) * 0.25f, 0.f), 1.f);
            acc[1] = fmaf(e, sc, acc[1]);
        }
    }
    block_sum<3>(acc, red, 1);
    const float nan_in = acc[2] > 0.f ? CUDART_NAN_F : 0.f;            // fmaxf drops NaNs: put them back
    const float lse = logf(acc[0]) + ref + nan_in;
    const float inv = (mx == CUDART_INF_F) ? CUDART_NAN_F : 1.0f / acc[0];   // softmax: inf - inf poisons the whole object
    if (tid == 0) {
        if (lse_out) lse_out[obj] = lse;
        if (loss_out) {
            const float v = (cost_target ? __ldg(cost_target + obj) : 0.f) + lse;
            loss_out[obj] = (v != v) ? 0.f : v;
        }
        if (want_score) score_out[obj] = acc[1] * inv + nan_in;
    }
    if (weights) {
        float* w = weights + (size_t)obj * M;
        for (int m = tid; m < M; m += NT) w[m] = expf(__ldg(l + m) - ref) * inv;
    }
}

// Backward of lse (and of the NaN -> 0 mask): grad_logw[b, m] = g[b] * exp(logw[b, m] - lse[b]); g[b] == 0 gives exact zeros
// (masked objects have lse = NaN).
__global__ void __launch_bounds__(NT) mc_lse_backward_kernel(const float* logw, const float* lse, const float* g,
                                                           float* grad_logw, int M) {
    const int obj = blockIdx.x;
    const float gb = __ldg(g + obj), ls = __ldg(lse + obj);
    const float* l = logw + (size_t)obj * M;
    float* o = grad_logw + (size_t)obj * M;
    for (int m = threadIdx.x; m < M; m += NT) o[m] = (gb == 0.f) ? 0.f : gb * expf(__ldg(l + m) - ls);
}
// ------------------------------------------------------------------------------------------------
// EPnP initialiser of the 6DoF test-time solve (lib/test.py:178-194 of the reference; math in pnp_epnp.cuh), one CTA per
// object:
//   1. conf_i = (w2d[i,0] + w2d[i,1]) / 2 as order-preserving uint32 keys in shared memory; a NaN confidence makes the
//      object's pose NaN with n_sel = 0 (np.quantile returns NaN, the mask is empty, cv2 refuses);
//   2. the order statistics s[k], s[k+1] of np.quantile by a binary radix select on the keys: 32 MSB-first passes, each
//      a block-wide count of the keys below both candidate prefixes -- no sort, no atomics;
//   3. the kept points (conf >= threshold) compacted once into shared memory, in index order: each thread owns a
//      contiguous run of indices, an exclusive scan of the per-thread counts places them.  Only the kept ~20 % are
//      read from x3d / x2d, by plain loads: a TMA stage of whole rows would move five times the bytes;
//   4. fp64 passes over the kept points with block reductions: centroid, scatter, then the 56 sums behind M^T M and
//      the Procrustes fit; lane 0 of warp 0 solves the small problems (pnp_epnp.cuh);
//   5. one more pass scores the three candidates by reprojection error; the cheapest is written.
// Shared memory: keys (N) + kept points (5 N floats) = 24 N bytes, within what epnp_max_points(6, 0, 0) allows.
struct EpnpInitArgs {
    const float *x3d, *x2d, *w2d, *cam;
    float* pose;                // (B, 7)
    int* n_sel;                 // [opt] (B)
    int N;
    float q;
};

__host__ __device__ inline int epnp_init_smem_bytes(int N) { return N * 6 * 4; }

// fp64 butterfly exchange as two 32-bit exchanges of its halves (the bits move unchanged, as a 64-bit shuffle moves them)
__device__ __forceinline__ double shfl_xor_f64(double v, int o) {
    uint32_t h[2];
    memcpy(h, &v, 8);
    h[0] = __float_as_uint(__shfl_xor_sync(0xffffffffu, __uint_as_float(h[0]), o));
    h[1] = __float_as_uint(__shfl_xor_sync(0xffffffffu, __uint_as_float(h[1]), o));
    memcpy(&v, h, 8);
    return v;
}

// block-wide fp64 sums of K values per thread (T threads, whole groups of four warps); every thread gets the totals,
// warp partials added as sum_warp_partials adds them
template <int K, int T = NT>
__device__ __forceinline__ void block_sum_f64(double (&v)[K], double* red) {
    static_assert(T % 128 == 0, "block_sum_f64: whole groups of four warps");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) v[k] += shfl_xor_f64(v[k], o);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) red[warp * K + k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) {
        v[k] = (red[k] + red[K + k]) + (red[2 * K + k] + red[3 * K + k]);
#pragma unroll
        for (int w = 4; w < T / 32; w += 4)
            v[k] += (red[w * K + k] + red[(w + 1) * K + k]) + (red[(w + 2) * K + k] + red[(w + 3) * K + k]);
    }
    __syncthreads();                    // red is free again
}

__global__ void __launch_bounds__(NT) epnp_init_kernel(const EpnpInitArgs a) {
    static_assert(NW == 4, "block_sum_f64 adds four warp partials");
    // 128: the alignment the other kernels declare for this (module-wide) symbol; a different one here moves their
    // dynamic shared memory base
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    __shared__ double red[NW * epnp::NSUM];
    __shared__ float fred[2 * NW * 32];
    __shared__ int counts[NT];
    __shared__ epnp::Control cp;
    __shared__ epnp::Candidate cand[3];
    const int tid = threadIdx.x, obj = blockIdx.x, N = a.N;
    uint32_t* keys = reinterpret_cast<uint32_t*>(smem_raw);            // [N]
    float* P = reinterpret_cast<float*>(smem_raw) + N;                 // [5][N]: X Y Z u v of the kept points
    const float* g3 = a.x3d + (size_t)obj * N * 3;
    const float* g2 = a.x2d + (size_t)obj * N * 2;
    int n = N;
    if (a.w2d) {
        const float* gw = a.w2d + (size_t)obj * N * 2;
        float nan_count[1] = {0.f};
        for (int i = tid; i < N; i += NT) {
            const float c = (__ldg(gw + 2 * i) + __ldg(gw + 2 * i + 1)) * 0.5f;
            keys[i] = epnp::conf_key(c);
            nan_count[0] += (c != c) ? 1.f : 0.f;
        }
        block_sum<1>(nan_count, fred, 0);
        if (nan_count[0] > 0.f) {
            if (tid == 0) {
#pragma unroll
                for (int i = 0; i < 7; ++i) a.pose[(size_t)obj * 7 + i] = CUDART_NAN_F;
                if (a.n_sel) a.n_sel[obj] = 0;
            }
            return;
        }
        const epnp::QuantileRank r = epnp::quantile_rank(N, a.q);
        uint32_t lo = 0u, hi = 0u;          // the largest v with #{key < v} <= k (= s[k]), and the same for k1
        for (int bit = 31; bit >= 0; --bit) {
            const uint32_t ca = lo | (1u << bit), cb = hi | (1u << bit);
            float c[2] = {0.f, 0.f};                // counts <= N are exact in fp32
            for (int i = tid; i < N; i += NT) {
                const uint32_t k = keys[i];
                c[0] += k < ca ? 1.f : 0.f;
                c[1] += k < cb ? 1.f : 0.f;
            }
            block_sum<2>(c, fred, bit & 1);
            if (c[0] <= (float)r.k) lo = ca;
            if (c[1] <= (float)r.k1) hi = cb;
        }
        const float thr = epnp::quantile_threshold(epnp::key_conf(lo), epnp::key_conf(hi), r.g);
        const int per = (N + NT - 1) / NT, i0 = min(N, tid * per), i1 = min(N, i0 + per);
        int mine = 0;
        for (int i = i0; i < i1; ++i) mine += epnp::key_conf(keys[i]) >= thr ? 1 : 0;
        counts[tid] = mine;
        __syncthreads();
        int off = 0;
        n = 0;
        for (int t = 0; t < NT; ++t) {
            off += t < tid ? counts[t] : 0;
            n += counts[t];
        }
        for (int i = i0; i < i1; ++i) {
            if (!(epnp::key_conf(keys[i]) >= thr)) continue;
            P[off] = __ldg(g3 + 3 * i); P[N + off] = __ldg(g3 + 3 * i + 1); P[2 * N + off] = __ldg(g3 + 3 * i + 2);
            P[3 * N + off] = __ldg(g2 + 2 * i); P[4 * N + off] = __ldg(g2 + 2 * i + 1);
            ++off;
        }
    } else {
        for (int i = tid; i < N; i += NT) {
            P[i] = __ldg(g3 + 3 * i); P[N + i] = __ldg(g3 + 3 * i + 1); P[2 * N + i] = __ldg(g3 + 3 * i + 2);
            P[3 * N + i] = __ldg(g2 + 2 * i); P[4 * N + i] = __ldg(g2 + 2 * i + 1);
        }
    }
    __syncthreads();
    float Kf[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) Kf[i] = __ldg(a.cam + (size_t)obj * 9 + i);
    const epnp::Intrinsics in = epnp::intrinsics(Kf);
    double c0[3] = {0.0, 0.0, 0.0};
    for (int j = tid; j < n; j += NT) { c0[0] += P[j]; c0[1] += P[N + j]; c0[2] += P[2 * N + j]; }
    block_sum_f64<3>(c0, red);
#pragma unroll
    for (int c = 0; c < 3; ++c) c0[c] /= n;
    double S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = tid; j < n; j += NT) {
        const double dx = P[j] - c0[0], dy = P[N + j] - c0[1], dz = P[2 * N + j] - c0[2];
        S[0] += dx * dx; S[1] += dx * dy; S[2] += dx * dz; S[3] += dy * dy; S[4] += dy * dz; S[5] += dz * dz;
    }
    block_sum_f64<6>(S, red);
    if (tid == 0) epnp::control_points(c0, S, n, cp);
    __syncthreads();
    double acc[epnp::NSUM];
#pragma unroll
    for (int k = 0; k < epnp::NSUM; ++k) acc[k] = 0.0;
    for (int j = tid; j < n; j += NT) epnp::accumulate_point(cp, in, P[j], P[N + j], P[2 * N + j], P[3 * N + j], P[4 * N + j], acc);
    block_sum_f64<epnp::NSUM>(acc, red);
    if (tid == 0) {
        double al[4];
        epnp::barycentric(cp, P[0], P[N], P[2 * N], al);
        epnp::solve_candidates(acc, cp, in, al, n, cand);
    }
    __syncthreads();
    double err[3] = {0.0, 0.0, 0.0};
    for (int j = tid; j < n; j += NT) {
#pragma unroll
        for (int c = 0; c < 3; ++c) err[c] += epnp::reproj_error(cand[c], in, P[j], P[N + j], P[2 * N + j], P[3 * N + j], P[4 * N + j]);
    }
    block_sum_f64<3>(err, red);
    if (tid == 0) {
        epnp::write_pose(cand[epnp::pick_candidate(err)], a.pose + (size_t)obj * 7);
        if (a.n_sel) a.n_sel[obj] = n;
    }
}

// epnp_init_kernel for objects too large for one SM (epnp_epnp_init_split_f32): one cluster of `ctas` CTAs per object
// (grid = B * ctas), rank r holding the points [r share, (r + 1) share) (split_share).  Each rank runs the resident
// kernel's steps over its own range.  What crosses ranks goes through an exchange slot in the rank's shared memory and
// one cluster barrier, after which every rank adds the ranks' values (sum_ranks):
//   1. the NaN counts: an object with a NaN confidence anywhere takes the NaN path on every rank;
//   2. per radix-select pass, the two counts over the global N (integers, exact in fp32: the threshold and the kept set
//      are np.quantile's over all N points whatever ctas is);
//   3. the kept counts: n, and the lowest rank holding a kept point.  That rank's first kept point is the object's first
//      in index order, which fixes the sign of the camera-frame control points; every rank reads it from there;
//   4. the fp64 partials of the centroid, the scatter, the 56 EPnP sums and the three reprojection errors.
// So every rank holds the same bits and runs control_points / solve_candidates itself (no broadcast); rank 0 alone
// writes pose and n_sel.
// Ordering: each exchange slot is written once, before the cluster barrier after which its peers read it -- except the
// radix counts, whose two halves alternate by pass: a half is written again two passes later, past the next barrier,
// which no rank reaches before its reads of that half are done.  Every rank passes the same barriers whatever its range
// holds (empty, nothing kept, the NaN path), and a last one keeps each CTA resident while its peers may read it.
// Shared memory, all dynamic (a peer can only address the dynamic window): the head below, then the keys (share) and
// the kept points (5 share floats), i.e. 24 share bytes + the head (about 8.5 KB).  cost_split_kernel takes
// 32 share + 11 KB at the same share (plan_cost_split), and the static_assert below keeps the head within that margin,
// so every C the cost kernel's plan allows (split_ctas_for(6, N, 0, 0)) fits this kernel too.
constexpr int EPNP_SPLIT_T = 256;
struct EpnpSplitAgreed {                // what every rank ends with, bit for bit (the audit build compares it)
    epnp::Control cp;
    epnp::Candidate cand[3];
    double c0[3], S[6], acc[epnp::NSUM], err[3];    // sums over the whole object
    float thr;
    int n, first, best;                             // kept points, lowest rank keeping one, winning candidate
};
struct EpnpSplitHead {
    double red[EPNP_SPLIT_T / 32 * epnp::NSUM];     // block_sum_f64 scratch
    double xc0[3], xS[6], xacc[epnp::NSUM], xerr[3]; // exchange slots: this rank's fp64 partials
    EpnpSplitAgreed g;
    float fred[2 * EPNP_SPLIT_T];                   // block_sum scratch, two halves
    float xsel[2][2];                               // exchange slot: radix counts, half = pass parity
    float xnan, xkept;                              // exchange slots: NaN count, kept count
    int counts[EPNP_SPLIT_T];                       // kept points per thread (compaction)
};
constexpr int EPNP_SPLIT_HEAD_BYTES = (int)((sizeof(EpnpSplitHead) + 127) / 128 * 128);
static_assert(EPNP_SPLIT_HEAD_BYTES <= 128 + (2 * STAGE_FLOATS + 2 * COST_SPLIT_TILE) * 4,
              "the EPnP split image must not exceed the cost split image at any share");
__host__ __device__ inline int epnp_split_smem_bytes(int share) { return EPNP_SPLIT_HEAD_BYTES + share * 6 * 4; }

// this rank's block sums of K fp64 values -> `slot`; one cluster barrier; thread k < K adds slot k of every rank into
// tot[k]; every thread gets the totals in v.  (The totals go on in a thread-local array, as in
// epnp_init_kernel: pnp_epnp.cuh's out-of-line functions then see the address spaces they see there, and
// epnp_init_kernel's code does not change.)
template <int K>
__device__ __forceinline__ void cluster_sum_f64(double (&v)[K], double* red, double* slot, double* tot, int ctas) {
    block_sum_f64<K, EPNP_SPLIT_T>(v, red);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) slot[k] = v[k];
    }
    cluster_sync();
    if (threadIdx.x < K) tot[threadIdx.x] = sum_ranks(slot + threadIdx.x, ctas);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = tot[k];
}

__global__ void __launch_bounds__(EPNP_SPLIT_T, 1) epnp_init_split_kernel(const EpnpInitArgs a, const int ctas) {
    constexpr int T = EPNP_SPLIT_T;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    EpnpSplitHead& h = *reinterpret_cast<EpnpSplitHead*>(smem_raw);
    const int N = a.N, share = split_share(N, ctas);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(N, rank * share), cnt = min(N, p0 + share) - p0;
    uint32_t* keys = reinterpret_cast<uint32_t*>(smem_raw + EPNP_SPLIT_HEAD_BYTES);    // [share]
    float* P = reinterpret_cast<float*>(keys + share);                                 // [5][share]: X Y Z u v, kept
    const float* g3 = a.x3d + ((size_t)obj * N + p0) * 3;
    const float* g2 = a.x2d + ((size_t)obj * N + p0) * 2;
    int nk = cnt;                           // this rank's kept points
    float thr = 0.f;
    if (a.w2d) {
        const float* gw = a.w2d + ((size_t)obj * N + p0) * 2;
        float nan_count[1] = {0.f};
        for (int i = tid; i < cnt; i += T) {
            const float c = (__ldg(gw + 2 * i) + __ldg(gw + 2 * i + 1)) * 0.5f;
            keys[i] = epnp::conf_key(c);
            nan_count[0] += (c != c) ? 1.f : 0.f;
        }
        block_sum<1, T>(nan_count, h.fred, 0);
        if (tid == 0) h.xnan = nan_count[0];
        cluster_sync();
        if (sum_ranks(&h.xnan, ctas) > 0.f) {       // the same decision on every rank
            if (rank == 0 && tid == 0) {
#pragma unroll
                for (int i = 0; i < 7; ++i) a.pose[(size_t)obj * 7 + i] = CUDART_NAN_F;
                if (a.n_sel) a.n_sel[obj] = 0;
                SPLIT_AUDIT_STORES(a.n_sel ? 8 : 7);
            }
            cluster_sync();                         // no CTA leaves while a peer may still read its NaN count
            return;
        }
        const epnp::QuantileRank r = epnp::quantile_rank(N, a.q);
        uint32_t lo = 0u, hi = 0u;
        for (int bit = 31; bit >= 0; --bit) {
            const uint32_t ca = lo | (1u << bit), cb = hi | (1u << bit);
            float c[2] = {0.f, 0.f};
            for (int i = tid; i < cnt; i += T) {
                const uint32_t k = keys[i];
                c[0] += k < ca ? 1.f : 0.f;
                c[1] += k < cb ? 1.f : 0.f;
            }
            block_sum<2, T>(c, h.fred, bit & 1);
            float* x = h.xsel[bit & 1];
            if (tid == 0) { x[0] = c[0]; x[1] = c[1]; }
            cluster_sync();
            if (sum_ranks(x, ctas) <= (float)r.k) lo = ca;
            if (sum_ranks(x + 1, ctas) <= (float)r.k1) hi = cb;
        }
        thr = epnp::quantile_threshold(epnp::key_conf(lo), epnp::key_conf(hi), r.g);
        const int per = (cnt + T - 1) / T, i0 = min(cnt, tid * per), i1 = min(cnt, i0 + per);
        int mine = 0;
        for (int i = i0; i < i1; ++i) mine += epnp::key_conf(keys[i]) >= thr ? 1 : 0;
        h.counts[tid] = mine;
        __syncthreads();
        int off = 0;
        nk = 0;
        for (int t = 0; t < T; ++t) {
            off += t < tid ? h.counts[t] : 0;
            nk += h.counts[t];
        }
        for (int i = i0; i < i1; ++i) {
            if (!(epnp::key_conf(keys[i]) >= thr)) continue;
            P[off] = __ldg(g3 + 3 * i); P[share + off] = __ldg(g3 + 3 * i + 1); P[2 * share + off] = __ldg(g3 + 3 * i + 2);
            P[3 * share + off] = __ldg(g2 + 2 * i); P[4 * share + off] = __ldg(g2 + 2 * i + 1);
            ++off;
        }
    } else {
        for (int i = tid; i < cnt; i += T) {
            P[i] = __ldg(g3 + 3 * i); P[share + i] = __ldg(g3 + 3 * i + 1); P[2 * share + i] = __ldg(g3 + 3 * i + 2);
            P[3 * share + i] = __ldg(g2 + 2 * i); P[4 * share + i] = __ldg(g2 + 2 * i + 1);
        }
    }
    if (tid == 0) h.xkept = (float)nk;
    cluster_sync();                         // also publishes the kept points to the peers
    int n = 0, first = -1;
    for (int r = 0; r < ctas; ++r) {
        const int k = (int)dsmem_ld(&h.xkept, r);
        if (first < 0 && k > 0) first = r;
        n += k;
    }
    float Kf[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) Kf[i] = __ldg(a.cam + (size_t)obj * 9 + i);
    const epnp::Intrinsics in = epnp::intrinsics(Kf);
    double c0[3] = {0.0, 0.0, 0.0};
    for (int j = tid; j < nk; j += T) { c0[0] += P[j]; c0[1] += P[share + j]; c0[2] += P[2 * share + j]; }
    cluster_sum_f64<3>(c0, h.red, h.xc0, h.g.c0, ctas);
#pragma unroll
    for (int c = 0; c < 3; ++c) c0[c] /= n;
    double S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = tid; j < nk; j += T) {
        const double dx = P[j] - c0[0], dy = P[share + j] - c0[1], dz = P[2 * share + j] - c0[2];
        S[0] += dx * dx; S[1] += dx * dy; S[2] += dx * dz; S[3] += dy * dy; S[4] += dy * dz; S[5] += dz * dz;
    }
    cluster_sum_f64<6>(S, h.red, h.xS, h.g.S, ctas);
    if (tid == 0) epnp::control_points<1>(c0, S, n, h.g.cp);
    __syncthreads();
    double acc[epnp::NSUM];
#pragma unroll
    for (int k = 0; k < epnp::NSUM; ++k) acc[k] = 0.0;
    for (int j = tid; j < nk; j += T)
        epnp::accumulate_point(h.g.cp, in, P[j], P[share + j], P[2 * share + j], P[3 * share + j], P[4 * share + j], acc);
    cluster_sum_f64<epnp::NSUM>(acc, h.red, h.xacc, h.g.acc, ctas);
    if (tid == 0) {
        double al[4];               // the object's first kept point: the first one of rank `first`
        epnp::barycentric(h.g.cp, dsmem_ld(P, first), dsmem_ld(P + share, first), dsmem_ld(P + 2 * share, first), al);
        epnp::solve_candidates<1>(acc, h.g.cp, in, al, n, h.g.cand);
    }
    __syncthreads();
    double err[3] = {0.0, 0.0, 0.0};
    for (int j = tid; j < nk; j += T) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
            err[c] += epnp::reproj_error(h.g.cand[c], in, P[j], P[share + j], P[2 * share + j], P[3 * share + j], P[4 * share + j]);
    }
    cluster_sum_f64<3>(err, h.red, h.xerr, h.g.err, ctas);
    if (tid == 0) {
        h.g.thr = thr; h.g.n = n; h.g.first = first; h.g.best = epnp::pick_candidate(err);
        if (rank == 0) {
            epnp::write_pose(h.g.cand[h.g.best], a.pose + (size_t)obj * 7);
            if (a.n_sel) a.n_sel[obj] = n;
            SPLIT_AUDIT_STORES(a.n_sel ? 8 : 7);
        }
    }
#ifdef EPNP_SPLIT_AUDIT
    cluster_sync();                         // rank 0's agreed state is complete
    const float* w = reinterpret_cast<const float*>(&h.g);
    for (int k = tid; k < (int)(sizeof(EpnpSplitAgreed) / 4); k += T)
        if (__float_as_uint(dsmem_ld(w + k, 0)) != __float_as_uint(w[k])) SPLIT_AUDIT_MISMATCH();
#endif
    // a CTA's shared memory disappears when it exits: no CTA leaves while a peer may still read its error partials
    cluster_sync();
}

// The gather of the cluster-split push call (epnp_lm_amis_fused_split_push_f32), launched after the solve on the same
// stream: this rank's finished rows -- logw (B, M) and pose (B, PD), each one contiguous run -- go to rows
// [row0, row0 + B) of every peer's full-batch buffers, float4 where the run's length and every address allow.  A copy
// of what the solve wrote, so the peers hold the single-GPU split result by construction (no second compilation of the
// AMIS body, DESIGN.md section 5).  Its own loop: the out-of-line push_rows is fitted by ptxas to all its callers, so a
// new caller could change amis_kernel's code.
__device__ __forceinline__ void push_run(float* const* peer, int n_peers, size_t dst_off, const float* src, size_t n) {
    float* dst[EPNP_MAX_PEERS];
    uintptr_t any = reinterpret_cast<uintptr_t>(src);
#pragma unroll
    for (int r = 0; r < EPNP_MAX_PEERS; ++r) {
        dst[r] = r < n_peers ? peer[r] + dst_off : nullptr;
        any |= reinterpret_cast<uintptr_t>(dst[r]);
    }
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
    if ((n & 3) == 0 && (any & 15u) == 0) {
        for (size_t q = i0; q < n / 4; q += step) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(src) + q);
#pragma unroll
            for (int r = 0; r < EPNP_MAX_PEERS; ++r)
                if (r < n_peers) reinterpret_cast<float4*>(dst[r])[q] = v;
        }
    } else {
        for (size_t i = i0; i < n; i += step) {
            const float v = __ldg(src + i);
#pragma unroll
            for (int r = 0; r < EPNP_MAX_PEERS; ++r)
                if (r < n_peers) dst[r][i] = v;
        }
    }
}

__global__ void __launch_bounds__(NT) push_split_kernel(const float* logw, const float* pose, const PushArgs push,
                                                        const size_t row0, const int B, const int M, const int PD) {
    push_run(push.logw, push.n, row0 * M, logw, (size_t)B * M);
    push_run(push.pose, push.n, row0 * PD, pose, (size_t)B * PD);
}

// ------------------------------------------------------------------------------------------------
// Host side
int cuda_fail(cudaError_t e) { g_last_cuda_error = (int)e; return EPNP_ERR_CUDA; }

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The problem fields of a KArgs: correspondences, cameras, bounds [opt] and Huber scales of B objects of N points.
KArgs problem_args(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats, const float* lb,
                   const float* ub, const float* delta, int B, int N) {
    KArgs a{};
    a.x3d = x3d; a.x2d = x2d; a.w2d = w2d; a.cam = cam_mats; a.lb = lb; a.ub = ub; a.delta = delta;
    a.B = B; a.N = N;
    return a;
}

int check_common(const KArgs& a) {
    if (!a.x3d || !a.x2d || !a.w2d || !a.cam || !a.delta) return EPNP_ERR_BAD_ARG;
    if ((a.lb == nullptr) != (a.ub == nullptr)) return EPNP_ERR_BAD_ARG;
    if (a.B < 0 || a.N <= 0) return EPNP_ERR_BAD_ARG;
    if (a.p.dof != 4 && a.p.dof != 6) return EPNP_ERR_BAD_ARG;
    return EPNP_OK;
}

// f(std::integral_constant<int, 6>{}) for dof = 6, else the <4> form: the DOF instantiation of a kernel or plan.
template <class F>
auto by_dof(int dof, F f) {
    return dof == 6 ? f(std::integral_constant<int, 6>{}) : f(std::integral_constant<int, 4>{});
}

int device_sms(int* sms) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_fail(e);
    e = cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
    return e == cudaSuccess ? EPNP_OK : cuda_fail(e);
}

bool tma_ok(const KArgs& a) { return (a.N % 4 == 0) && aligned16(a.x3d) && aligned16(a.x2d) && aligned16(a.w2d); }

// The launch fields of a KArgs: the loader's TMA switch and the SM count.
int prepare_launch(KArgs& a) { a.use_tma = tma_ok(a); return device_sms(&a.num_sms); }

// The shared-memory check and launch fields of a launch that holds each object's points in one CTA.
int prepare_resident(KArgs& a, int smem_bytes) {
    if ((size_t)smem_bytes > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    return prepare_launch(a);
}

// What a launch sets on its kernel first: nothing, the dynamic shared-memory size, or that size and the full shared
// memory carve-out of the SM (which several resident CTAs of nearly 228 KB between them need).  Which kernels ask for
// the carve-out is a tuning choice, made at each launch.
enum class SmemAttr { none, size, size_and_carveout };

template <class Kern>
cudaError_t set_smem_attr(Kern kern, int smem_bytes, SmemAttr attr) {
    if (attr == SmemAttr::none) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess || attr == SmemAttr::size) return e;
    return cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}

// A plain (non-cluster) launch of `grid` CTAs of `block` threads: the kernel's attributes, the launch, its error.
template <class Kern, class... Args>
int launch_plain(Kern kern, int grid, int block, int smem_bytes, SmemAttr attr, cudaStream_t stream, Args... args) {
    cudaError_t e = set_smem_attr(kern, smem_bytes, attr);
    if (e != cudaSuccess) return cuda_fail(e);
    EPNP_LAUNCH(kern, grid, block, smem_bytes, stream, args...);
    e = cudaGetLastError();
    return e == cudaSuccess ? EPNP_OK : cuda_fail(e);
}

// One CTA of NT threads per object (grid = B): the hardware scheduler hands CTAs to SMs as slots free up, the CTAs'
// serial and parallel phases de-synchronise and there is no lock-step tail, as a persistent grid would have.
template <int T = NT, class Kern, class... Extra>
int launch_cta_per_object(Kern kern, KArgs& a, int smem_bytes, cudaStream_t stream, Extra... extra) {
    if (a.B == 0) return EPNP_OK;
    const int rc = prepare_resident(a, smem_bytes);
    if (rc != EPNP_OK) return rc;
    return launch_plain(kern, a.B, T, smem_bytes, SmemAttr::size_and_carveout, stream, a, extra...);
}

// LM / GN solve: one CTA of WARPS warps per object (one warp unless the point set is long).  Outputs: a.pose_opt,
// a.pose_cov [opt] (stride a.cov_stride), a.cost [opt], a.pose_plus [opt], a.cost_init [opt].
template <int DOF, bool STAGED, int WARPS>
int launch_lm_as(KArgs& a, cudaStream_t stream) {
    return launch_plain(lm_warp_kernel<DOF, STAGED, WARPS>, a.B, 32 * WARPS, lm_smem_bytes<DOF, WARPS>(a.N, STAGED),
                        STAGED ? SmemAttr::size_and_carveout : SmemAttr::none, stream, a);
}

// Warps per object: a function of N ONLY, so that an object's result does not depend on how large a batch (or which
// shard of it) it is solved in -- the summation order of the 28 sums changes with the warp count.  Dense coordinate maps
// (N >= 2048: 16+ points per lane even with 8 warps) get 8 warps, everything else one.
int lm_warps_per_object(int N) { return N >= 2048 ? 8 : 1; }

int launch_lm(KArgs& a, cudaStream_t stream) {
    if (a.B == 0) return EPNP_OK;
    const int rc = prepare_launch(a);
    if (rc != EPNP_OK) return rc;
    const bool staged = a.N <= LM_STAGE_MAX_N, one_warp = lm_warps_per_object(a.N) == 1;
    return by_dof(a.p.dof, [&](auto D) {
        if (staged) return one_warp ? launch_lm_as<D, true, 1>(a, stream) : launch_lm_as<D, true, 8>(a, stream);
        return one_warp ? launch_lm_as<D, false, 1>(a, stream) : launch_lm_as<D, false, 8>(a, stream);
    });
}

// Hypothesis warps per CTA of the staged stacked LM kernel for S starts: the CTAs of an object take equal shares of the
// starts, at most LM_STACK_MAX_H each.  A function of S only (not B), like lm_warps_per_object of N.
int lm_stack_h(int S) {
    const int chunks = (S + LM_STACK_MAX_H - 1) / LM_STACK_MAX_H;
    return (S + chunks - 1) / chunks;
}

template <int DOF, bool STAGED, int WARPS>
int launch_lm_stacked_as(KArgs& a, int S, int H, cudaStream_t stream) {
    const int chunks = (S + H - 1) / H;
    const int smem_bytes = H * lm_head_bytes<DOF, WARPS>() + (STAGED ? 28 * lm_padded_points(a.N) : 0);
    return launch_plain(lm_stacked_kernel<DOF, STAGED, WARPS>, a.B * chunks, 32 * WARPS * H, smem_bytes,
                        STAGED ? SmemAttr::size_and_carveout : SmemAttr::none, stream, a, S, H);
}

// LM / GN solve of S stacked starts per object (a.pose_init (S, B, D), outputs in rows s B + b): the staged objects'
// hypotheses share one staged copy of the points, H of them per CTA; the others run one start per CTA with
// lm_warp_kernel's warp count and point order.  Either way each start's sums are those of launch_lm.
int launch_lm_stacked(KArgs& a, int S, cudaStream_t stream) {
    if (a.B == 0 || S == 0) return EPNP_OK;
    const int rc = prepare_launch(a);
    if (rc != EPNP_OK) return rc;
    return by_dof(a.p.dof, [&](auto D) {
        if (a.N <= LM_STAGE_MAX_N) return launch_lm_stacked_as<D, true, 1>(a, S, lm_stack_h(S), stream);
        if (lm_warps_per_object(a.N) == 1) return launch_lm_stacked_as<D, false, 1>(a, S, 1, stream);
        return launch_lm_stacked_as<D, false, 8>(a, S, 1, stream);
    });
}

// The LM launch of the fused calls; its pose and covariance are the AMIS kernel's inputs.
int launch_lm_for_amis(KArgs& a, cudaStream_t stream) {
    const int rc = launch_lm(a, stream);
    a.pose_opt_in = a.pose_opt;
    a.pose_cov_in = a.pose_cov;
    return rc;
}

inline bool amis_dense(int N) { return N >= AMIS_DENSE_MIN_N; }
template <int DOF> int amis_smem_bytes(int N, int M) {
    return amis_dense(N) ? plan_amis<DOF, AMIS_T_DENSE>(N, M).total_bytes : plan_amis<DOF, NT>(N, M).total_bytes;
}

// f(std::integral_constant<int, T>{}) with T the threads per CTA of the resident AMIS kernel for N points.
template <class F>
int by_amis_threads(int N, F f) {
    return amis_dense(N) ? f(std::integral_constant<int, AMIS_T_DENSE>{}) : f(std::integral_constant<int, NT>{});
}

// seed_ptr [opt]: the AMIS kernel reads the seed from this device address (amis_seedptr_kernel) instead of a.seed.
int launch_amis(KArgs& a, const PushArgs* push, cudaStream_t stream, const uint64_t* seed_ptr = nullptr) {
    const PushArgs pa = push ? *push : PushArgs{};
    return by_dof(a.p.dof, [&](auto D) {
        const int smem_bytes = amis_smem_bytes<D>(a.N, a.p.mc_samples);
        return by_amis_threads(a.N, [&](auto T) {
            if (seed_ptr) return launch_cta_per_object<T>(amis_seedptr_kernel<D, T>, a, smem_bytes, stream, pa, seed_ptr);
            return launch_cta_per_object<T>(amis_kernel<D, T>, a, smem_bytes, stream, pa);
        });
    });
}

// Cluster-split launches (amis_split_kernel, cost_split_kernel, gn_plus_backward_split_kernel, epnp_init_split_kernel):
// `ctas` CTAs of T threads for each of B objects; the kernel takes (Args, ctas).  Args holding a KArgs get its launch
// fields set (prepare_launch).  A device that cannot co-schedule one such cluster (a MIG slice, or SMs taken by other
// work) gets EPNP_ERR_UNSUPPORTED; nothing is launched then.  launch = false: only that check (run_lm_amis_split makes
// it before its LM launch).  clusters [opt]: receives how many such clusters the device runs at once.
inline KArgs& kargs_of(KArgs& a) { return a; }
inline KArgs& kargs_of(SeededKArgs& s) { return s.k; }
inline int prepare_launch(GnBwArgs& g) { return prepare_launch(g.k); }
inline int prepare_launch(PoseBwArgs& g) { return prepare_launch(g.k); }
inline int prepare_launch(CamBwArgs& g) { return prepare_launch(g.k); }
inline int prepare_launch(GnCamBwArgs& g) { return prepare_launch(g.k); }
inline int prepare_launch(SeededKArgs& s) { return prepare_launch(s.k); }
inline int prepare_launch(EpnpInitArgs&) { return EPNP_OK; }
#if defined(EPNP_SIMT_EMUL) && !defined(SIMT_EMUL_HAS_CLUSTERS)
// The single-CTA emulator build (tests/simt_emul) cannot run a cluster: every launch is refused.
template <int T, class Kern, class Args>
int launch_cluster(Kern, Args&, int B, int smem_bytes, int, cudaStream_t, bool = true, int* = nullptr) {
    if (B == 0) return EPNP_OK;
    if ((size_t)smem_bytes > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    return EPNP_ERR_UNSUPPORTED;
}
#else
template <int T, class Kern, class Args>
int launch_cluster(Kern kern, Args& args, int B, int smem_bytes, int ctas, cudaStream_t stream, bool launch = true,
                   int* active = nullptr) {
    if (B == 0) return EPNP_OK;
    if ((size_t)smem_bytes > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    cudaError_t e = set_smem_attr(kern, smem_bytes, SmemAttr::size_and_carveout);
    if (e != cudaSuccess) return cuda_fail(e);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)ctas;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)B * (unsigned)ctas);
    cfg.blockDim = dim3(T);
    cfg.dynamicSmemBytes = (size_t)smem_bytes;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    e = cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg);
    if (e != cudaSuccess) return cuda_fail(e);
    if (clusters == 0) return EPNP_ERR_UNSUPPORTED;
    if (active) *active = clusters;
    if (!launch) return EPNP_OK;
    const int rc = prepare_launch(args);
    if (rc != EPNP_OK) return rc;
    e = cudaLaunchKernelEx(&cfg, kern, args, ctas);
    return e == cudaSuccess ? EPNP_OK : cuda_fail(e);
}
#endif

// Shared memory per CTA of a split launch; mc_samples = 0: the cost and GN-plus backward kernels.
int split_smem_bytes(int dof, int N, int ctas, int mc_samples, int mc_iter) {
    const int share = split_share(N, ctas);
    if (mc_samples == 0) return plan_cost_split(share).total_bytes;
    return by_dof(dof, [&](auto D) { return plan_amis_split<D>(share, mc_samples, mc_iter).a.total_bytes; });
}

// The automatic cluster size: the smallest C >= 2 whose largest rank share fits, 0 when even 8 do not.  A function of
// (N, M, I) only, so that an object's result does not depend on the batch it is solved in.
int split_min_ctas(int dof, int N, int mc_samples, int mc_iter) {
    for (int c = 2; c <= SPLIT_MAX_CTAS; ++c)
        if ((size_t)split_smem_bytes(dof, N, c, mc_samples, mc_iter) <= SMEM_LIMIT) return c;
    return 0;
}

// Cluster size of a split call: `requested` = 0 picks split_min_ctas; otherwise it must lie in [that minimum, 8].
// Returns C > 0, or a (negative) error code.
int split_ctas_for(int dof, int N, int mc_samples, int mc_iter, int requested) {
    const int c_min = split_min_ctas(dof, N, mc_samples, mc_iter);
    if (c_min == 0) return EPNP_ERR_TOO_MANY_POINTS;
    if (requested == 0) return c_min;
    if (requested < c_min || requested > SPLIT_MAX_CTAS) return EPNP_ERR_BAD_ARG;
    return requested;
}

unsigned long long* g_prof_buffer = nullptr;     // set by epnp_debug_set_phase_buffer (profiling build)

// Objects the device works on at once in a CTA-per-object kernel: SMs x resident CTAs per SM.  Used by the host-buffer
// entry points to cut the batch at whole waves.  `attr`: what the kernel's own launch sets.  0 when it cannot be
// determined.
template <int T, class Kern>
int resident_objects(Kern kern, int smem_bytes, SmemAttr attr = SmemAttr::size_and_carveout) {
    int sms = 0, occ = 0;
    if ((size_t)smem_bytes > SMEM_LIMIT) return 0;
    if (device_sms(&sms) != EPNP_OK) return 0;
    if (set_smem_attr(kern, smem_bytes, attr) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, T, smem_bytes) != cudaSuccess) return 0;
    return sms * occ;
}

// Fast mode takes the covariance, cost and cost_init from its Gauss-Newton steps' evaluations (each before its step):
// with lm_iter = 0 nothing evaluates, so none of the three has a value (the reference's has none either).  The calls
// that would return one refuse instead.
bool fast_mode_without_steps(const Params& p) { return p.fast_mode != 0 && p.lm_iter == 0; }

int check_amis_params(const Params& p) {
    if (p.mc_iter <= 0 || p.mc_iter > MAX_ITER || p.mc_samples <= 0 || p.mc_samples % p.mc_iter != 0) return EPNP_ERR_BAD_ARG;
    if (p.acg_mle_iter < 0) return EPNP_ERR_BAD_ARG;
    return EPNP_OK;
}

// The checks every AMIS call (epnp_amis_f32, the fused and the push calls) makes of its KArgs: the problem, the AMIS
// parameters, the sample outputs, and the noise tables, which come all three or not at all.
int check_amis_call(const KArgs& a) {
    if (check_common(a) != EPNP_OK || check_amis_params(a.p) != EPNP_OK) return EPNP_ERR_BAD_ARG;
    if (!a.pose_samples || !a.logw) return EPNP_ERR_BAD_ARG;
    const bool any = a.noise_n3 || a.noise_chi2 || a.noise_rot, all = a.noise_n3 && a.noise_chi2 && a.noise_rot;
    return any && !all ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

// The covariance of the fused calls travels from the LM to the AMIS kernel through a.pose_cov (caller's buffer) or,
// when the caller did not ask for it, through the first dof^2 floats of each object's -- not yet written -- sample rows.
int route_cov(KArgs& a) {
    const int dof = a.p.dof, D = dof == 6 ? 7 : 4;
    if (a.pose_cov) {
        a.cov_stride = dof * dof;
        return EPNP_OK;
    }
    if (a.p.mc_samples * D < dof * dof) return EPNP_ERR_BAD_ARG;
    a.pose_cov = a.pose_samples;
    a.cov_stride = a.p.mc_samples * D;
    return EPNP_OK;
}

// LM kernel, then AMIS kernel, on `stream`.  seed_ptr [opt]: the AMIS kernel reads its seed from there (launch_amis).
int run_lm_amis(KArgs& a, const PushArgs* push, cudaStream_t stream, const uint64_t* seed_ptr = nullptr) {
    int rc = route_cov(a);
    if (rc != EPNP_OK) return rc;
    if ((size_t)by_dof(a.p.dof, [&](auto D) { return amis_smem_bytes<D>(a.N, a.p.mc_samples); }) > SMEM_LIMIT)
        return EPNP_ERR_TOO_MANY_POINTS;        // before anything is launched
    rc = launch_lm_for_amis(a, stream);
    return rc != EPNP_OK ? rc : launch_amis(a, push, stream, seed_ptr);
}

// The launches of run_lm_amis_split on `args` (a KArgs, or a SeededKArgs for the seed-pointer kernel): a device that
// cannot run the cluster gets no LM launch either.
template <class Args>
int lm_amis_split_launches(Args& args, void (*kern)(const Args, const int), int ctas, int smem_bytes, cudaStream_t stream) {
    KArgs& a = kargs_of(args);
    int rc = launch_cluster<AMIS_T_DENSE>(kern, args, a.B, smem_bytes, ctas, stream, false);
    if (rc != EPNP_OK) return rc;
    rc = launch_lm_for_amis(a, stream);
    return rc != EPNP_OK ? rc : launch_cluster<AMIS_T_DENSE>(kern, args, a.B, smem_bytes, ctas, stream);
}

// run_lm_amis with the cluster-split AMIS kernel.  The LM half is the unstaged 8-warp LM kernel, which streams any N.
// seed_ptr [opt]: the AMIS kernel reads its seed from there (amis_split_seedptr_kernel).
int run_lm_amis_split(KArgs& a, int cluster_ctas, cudaStream_t stream, const uint64_t* seed_ptr = nullptr) {
    const int dof = a.p.dof;
    const int ctas = split_ctas_for(dof, a.N, a.p.mc_samples, a.p.mc_iter, cluster_ctas);
    if (ctas < 0) return ctas;                  // before anything is launched
    const int rc = route_cov(a);
    if (rc != EPNP_OK) return rc;
    const int smem_bytes = split_smem_bytes(dof, a.N, ctas, a.p.mc_samples, a.p.mc_iter);
    return by_dof(dof, [&](auto D) {
        if (!seed_ptr) return lm_amis_split_launches(a, amis_split_kernel<D>, ctas, smem_bytes, stream);
        SeededKArgs sa{a, seed_ptr};
        return lm_amis_split_launches(sa, amis_split_seedptr_kernel<D>, ctas, smem_bytes, stream);
    });
}

// What run_lm_amis_split would run B > 0 objects of N points on, checked without launching anything: returns the
// cluster size C, or the refusal it would give (negative); *wave = the objects the device solves at once (clusters of
// the AMIS split kernel it co-schedules).  For the host-buffer call, whose refusals come before its first copy.
int split_lm_amis_plan(const Params& p, int B, int N, int cluster_ctas, int* wave) {
    const int ctas = split_ctas_for(p.dof, N, p.mc_samples, p.mc_iter, cluster_ctas);
    if (ctas < 0) return ctas;
    KArgs unused{};                             // launch = false: launch_cluster does not read the kernel's arguments
    const int smem_bytes = split_smem_bytes(p.dof, N, ctas, p.mc_samples, p.mc_iter);
    const int rc = by_dof(p.dof, [&](auto D) {
        return launch_cluster<AMIS_T_DENSE>(amis_split_kernel<D>, unused, B, smem_bytes, ctas, nullptr, false, wave);
    });
    return rc != EPNP_OK ? rc : ctas;
}

}  // namespace

// ================================================================================================
extern "C" {

#ifdef EPNP_PHASE_TIMERS
// profiling build only (not declared in the public header): device buffer of PH_COUNT uint64 counters
void epnp_debug_set_phase_buffer(unsigned long long* dev_buf) { g_prof_buffer = dev_buf; }
#endif

int epnp_abi_version(void) { return EPNP_ABI_VERSION; }

int epnp_last_cuda_error(void) { return g_last_cuda_error; }

const char* epnp_error_string(int code) {
    switch (code) {
        case EPNP_OK: return "ok";
        case EPNP_ERR_BAD_ARG: return "bad argument";
        case EPNP_ERR_TOO_MANY_POINTS: return "correspondence set (and sample buffers) exceed 227 KB of shared memory";
        case EPNP_ERR_UNSUPPORTED: return "combination not supported by this build";
        case EPNP_ERR_CUDA: return "CUDA runtime error (see epnp_last_cuda_error)";
        case EPNP_ERR_NO_DEVICE: return "no CUDA device";
        default: return "unknown error";
    }
}

void epnp_default_params(EpnpParams* p, int dof) {
    p->dof = dof; p->lm_iter = 10; p->fast_mode = 0; p->z_min = 0.1f;
    p->min_lm_diagonal = 1e-6f; p->max_lm_diagonal = 1e32f; p->min_relative_decrease = 1e-3f;
    p->initial_radius = 30.0f; p->max_radius = 1e16f; p->eps = 1e-5f; p->huber_eps = 1e-10f;
    p->mc_samples = 512; p->mc_iter = 4; p->amis_eps = 1e-5f; p->acg_mle_iter = 3; p->acg_dispersion = 1e-3f;
}

int epnp_max_points(int dof, int mc_samples, int mc_iter) {
    (void)mc_iter;
    const bool amis = mc_samples > 0;
    int lo = 0, hi = 1 << 16;
    while (lo + 4 <= hi) {                   // largest multiple of 4 that fits
        const int mid = ((lo + hi) / 2) / 4 * 4;
        if (mid == lo) break;
        const int bytes = by_dof(dof, [&](auto D) {
            return amis ? amis_smem_bytes<D>(mid, mc_samples) : plan_obj<D>(mid).total_bytes;
        });
        if ((size_t)bytes <= SMEM_LIMIT) lo = mid; else hi = mid;
    }
    return lo;
}

int epnp_split_ctas(int dof, int N, int mc_samples, int mc_iter) {
    if ((dof != 4 && dof != 6) || N <= 0 || mc_samples < 0) return 0;
    if (mc_samples > 0 && (mc_iter <= 0 || mc_iter > MAX_ITER || mc_samples % mc_iter != 0)) return 0;
    return split_min_ctas(dof, N, mc_samples, mc_iter);
}

int epnp_max_points_split(int dof, int mc_samples, int mc_iter) {
    if (epnp_split_ctas(dof, 8, mc_samples, mc_iter) == 0) return 0;
    int lo = 8, hi = 1 << 16;               // rank shares (multiples of 8) that fit / do not fit
    while (hi - lo > 8) {
        const int mid = (lo + hi) / 2 / 8 * 8;
        if ((size_t)split_smem_bytes(dof, SPLIT_MAX_CTAS * mid, SPLIT_MAX_CTAS, mc_samples, mc_iter) <= SMEM_LIMIT) lo = mid;
        else hi = mid;
    }
    return SPLIT_MAX_CTAS * lo;
}

int epnp_adaptive_delta_f32(const float* x2d, const float* w2d, float relative_delta, float* delta, int B, int N,
                            void* stream) {
    if (!x2d || !w2d || !delta || B < 0 || N <= 0) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    return launch_plain(adaptive_delta_kernel, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, x2d, w2d, relative_delta,
                        delta, N);
}

int epnp_mc_epilogue_f32(const float* logw, const float* pose_samples, const float* pose_opt, const float* cost_target,
                         float* lse, float* loss, float* weights, float* score_te, int B, int M, int dof, void* stream) {
    if (!logw || B < 0 || M <= 0 || (dof != 4 && dof != 6)) return EPNP_ERR_BAD_ARG;
    if (!lse && !loss && !weights && !score_te) return EPNP_ERR_BAD_ARG;
    if (score_te && (!pose_samples || !pose_opt)) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    const auto run = [&](auto kern) {
        return launch_plain(kern, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, logw, pose_samples, pose_opt,
                            cost_target, lse, loss, weights, score_te, M);
    };
    return dof == 6 ? run(mc_epilogue_kernel<7>) : run(mc_epilogue_kernel<4>);
}

int epnp_mc_lse_backward_f32(const float* logw, const float* lse, const float* grad_lse, float* grad_logw, int B, int M,
                             void* stream) {
    if (!logw || !lse || !grad_lse || !grad_logw || B < 0 || M <= 0) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    return launch_plain(mc_lse_backward_kernel, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, logw, lse, grad_lse,
                        grad_logw, M);
}

// The checked KArgs of epnp_evaluate_cost_f32 and its split form, or the refusal.
static int cost_args(KArgs& a, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                     const float* lb, const float* ub, const float* delta, const float* poses, float* cost,
                     int S, int B, int N, int dof, float z_min) {
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = poses; a.cost_out = cost; a.S_eval = S;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    return (!poses || !cost || S < 0) ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

int epnp_evaluate_cost_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                           const float* lb, const float* ub, const float* delta, const float* poses, float* cost,
                           int S, int B, int N, int dof, float z_min, void* stream) {
    KArgs a;
    const int rc = cost_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, cost, S, B, N, dof, z_min);
    if (rc != EPNP_OK || S == 0) return rc;
    return by_dof(dof, [&](auto D) {
        return launch_cta_per_object(cost_kernel<D>, a, plan_obj<D>(N).total_bytes, (cudaStream_t)stream);
    });
}

int epnp_evaluate_cost_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                 const float* lb, const float* ub, const float* delta, const float* poses, float* cost,
                                 int S, int B, int N, int dof, float z_min, int cluster_ctas, void* stream) {
    KArgs a;
    const int rc = cost_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, cost, S, B, N, dof, z_min);
    if (rc != EPNP_OK) return rc;
    const int ctas = split_ctas_for(dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    if (S == 0) return EPNP_OK;
    const int smem_bytes = split_smem_bytes(dof, N, ctas, 0, 0);
    return by_dof(dof, [&](auto D) {
        return launch_cluster<COST_SPLIT_TILE>(cost_split_kernel<D>, a, B, smem_bytes, ctas, (cudaStream_t)stream);
    });
}

int epnp_evaluate_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose,
                      float* residual, float* jac, float* cost, int clip_jac,
                      int B, int N, int dof, float z_min, float huber_eps, void* stream) {
    KArgs a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = pose;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!pose) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    return by_dof(dof, [&](auto D) {
        return launch_plain(evaluate_full_kernel<D>, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, a, residual, jac,
                            cost, clip_jac, huber_eps);
    });
}

int epnp_lm_solve_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose_init,
                      float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                      int B, int N, const EpnpParams* p, void* stream) {
    if (!p) return EPNP_ERR_BAD_ARG;
    KArgs a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.pose_init = pose_init; a.pose_opt = pose_opt; a.pose_cov = pose_cov; a.cost = cost;
    a.pose_plus = pose_opt_plus; a.cost_init = cost_init; a.p = *p;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!pose_init || !pose_opt || p->lm_iter < 0) return EPNP_ERR_BAD_ARG;
    if (fast_mode_without_steps(*p) && (pose_cov || cost || cost_init)) return EPNP_ERR_BAD_ARG;
    a.cov_stride = p->dof * p->dof;
    return launch_lm(a, (cudaStream_t)stream);
}

int epnp_lm_solve_stacked_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                              const float* lb, const float* ub, const float* delta, const float* pose_init,
                              float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                              int S, int B, int N, const EpnpParams* p, void* stream) {
    if (!p) return EPNP_ERR_BAD_ARG;
    KArgs a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.pose_init = pose_init; a.pose_opt = pose_opt; a.pose_cov = pose_cov; a.cost = cost;
    a.pose_plus = pose_opt_plus; a.cost_init = cost_init; a.p = *p;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!pose_init || !pose_opt || p->lm_iter < 0 || S < 0 || (long long)S * B > 2147483647LL) return EPNP_ERR_BAD_ARG;
    if (fast_mode_without_steps(*p) && (pose_cov || cost || cost_init)) return EPNP_ERR_BAD_ARG;
    a.cov_stride = p->dof * p->dof;
    return launch_lm_stacked(a, S, (cudaStream_t)stream);
}

// The checked arguments of epnp_gn_plus_backward_f32 and its split form, or the refusal.
static int gn_bw_args(GnBwArgs& g, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose,
                      const float* grad_pose_plus, float* grad_x3d, float* grad_x2d, float* grad_w2d,
                      float* grad_delta, int B, int N, int dof, float z_min, float eps, float huber_eps) {
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = pose;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min; a.p.eps = eps; a.p.huber_eps = huber_eps;
    g.gplus = grad_pose_plus; g.gx3d = grad_x3d; g.gx2d = grad_x2d; g.gw2d = grad_w2d; g.gdelta = grad_delta;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    return (!pose || !grad_pose_plus) ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

int epnp_gn_plus_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                              const float* lb, const float* ub, const float* delta, const float* pose,
                              const float* grad_pose_plus, float* grad_x3d, float* grad_x2d, float* grad_w2d,
                              float* grad_delta, int B, int N, int dof, float z_min, float eps, float huber_eps,
                              void* stream) {
    GnBwArgs g{};
    const int rc = gn_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, grad_x3d, grad_x2d,
                              grad_w2d, grad_delta, B, N, dof, z_min, eps, huber_eps);
    if (rc != EPNP_OK || B == 0) return rc;
    return by_dof(dof, [&](auto D) {
        const int smem_bytes = plan_obj<D>(N).total_bytes;
        const int rc = prepare_resident(g.k, smem_bytes);
        if (rc != EPNP_OK) return rc;
        return launch_plain(gn_plus_backward_kernel<D>, B, NT, smem_bytes, SmemAttr::size, (cudaStream_t)stream, g);
    });
}

int epnp_gn_plus_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                    const float* lb, const float* ub, const float* delta, const float* pose,
                                    const float* grad_pose_plus, float* grad_x3d, float* grad_x2d, float* grad_w2d,
                                    float* grad_delta, int B, int N, int dof, float z_min, float eps, float huber_eps,
                                    int cluster_ctas, void* stream) {
    GnBwArgs g{};
    const int rc = gn_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, grad_x3d, grad_x2d,
                              grad_w2d, grad_delta, B, N, dof, z_min, eps, huber_eps);
    if (rc != EPNP_OK) return rc;
    const int ctas = split_ctas_for(dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    const int smem_bytes = split_smem_bytes(dof, N, ctas, 0, 0);
    return by_dof(dof, [&](auto D) {
        return launch_cluster<GNBW_SPLIT_T>(gn_plus_backward_split_kernel<D>, g, B, smem_bytes, ctas, (cudaStream_t)stream);
    });
}

// The outputs of the camera backward entry points: at least one, and a bound's gradient only with bounds.
static int camera_outputs_ok(const float* lb, const float* grad_cam, const float* grad_lb, const float* grad_ub) {
    if (!grad_cam && !grad_lb && !grad_ub) return EPNP_ERR_BAD_ARG;
    return ((grad_lb || grad_ub) && !lb) ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

// The checked arguments of epnp_gn_plus_camera_backward_f32 and its split form, or the refusal.
static int gn_cam_bw_args(GnCamBwArgs& g, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                          const float* lb, const float* ub, const float* delta, const float* pose,
                          const float* grad_pose_plus, float* grad_cam, float* grad_lb, float* grad_ub, int B, int N,
                          int dof, float z_min, float eps, float huber_eps) {
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = pose;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min; a.p.eps = eps; a.p.huber_eps = huber_eps;
    g.gplus = grad_pose_plus; g.gcam = grad_cam; g.glb = grad_lb; g.gub = grad_ub;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!pose || !grad_pose_plus) return EPNP_ERR_BAD_ARG;
    return camera_outputs_ok(lb, grad_cam, grad_lb, grad_ub);
}

int epnp_gn_plus_camera_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                     const float* lb, const float* ub, const float* delta, const float* pose,
                                     const float* grad_pose_plus, float* grad_cam, float* grad_lb, float* grad_ub,
                                     int B, int N, int dof, float z_min, float eps, float huber_eps, void* stream) {
    GnCamBwArgs g{};
    const int rc = gn_cam_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, grad_cam, grad_lb,
                                  grad_ub, B, N, dof, z_min, eps, huber_eps);
    if (rc != EPNP_OK || B == 0) return rc;
    return by_dof(dof, [&](auto D) {
        const int smem_bytes = plan_obj<D>(N).total_bytes;
        const int rc = prepare_resident(g.k, smem_bytes);
        if (rc != EPNP_OK) return rc;
        return launch_plain(gn_plus_camera_backward_kernel<D>, B, NT, smem_bytes, SmemAttr::size, (cudaStream_t)stream,
                            g);
    });
}

int epnp_gn_plus_camera_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                           const float* lb, const float* ub, const float* delta, const float* pose,
                                           const float* grad_pose_plus, float* grad_cam, float* grad_lb,
                                           float* grad_ub, int B, int N, int dof, float z_min, float eps,
                                           float huber_eps, int cluster_ctas, void* stream) {
    GnCamBwArgs g{};
    const int rc = gn_cam_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, grad_cam, grad_lb,
                                  grad_ub, B, N, dof, z_min, eps, huber_eps);
    if (rc != EPNP_OK) return rc;
    const int ctas = split_ctas_for(dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    const int smem_bytes = split_smem_bytes(dof, N, ctas, 0, 0);
    return by_dof(dof, [&](auto D) {
        return launch_cluster<GNBW_SPLIT_T>(gn_plus_camera_backward_split_kernel<D>, g, B, smem_bytes, ctas,
                                            (cudaStream_t)stream);
    });
}

int epnp_gn_plus_hvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                         const float* lb, const float* ub, const float* delta, const float* pose,
                         const float* grad_pose_plus, const float* t_x3d, const float* t_x2d, const float* t_w2d,
                         const float* t_delta, const float* t_cam, const float* t_lb, const float* t_ub,
                         float* h_x3d, float* h_x2d, float* h_w2d, float* h_delta, float* h_cam, float* h_lb,
                         float* h_ub, float* h_grad, int B, int N, int dof, float z_min, float eps, float huber_eps,
                         void* stream) {
    GnBwArgs gb{};
    const int rc = gn_bw_args(gb, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, nullptr, nullptr,
                              nullptr, nullptr, B, N, dof, z_min, eps, huber_eps);
    if (rc != EPNP_OK) return rc;
    if (!lb && (t_lb || t_ub || h_lb || h_ub)) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    if (N > epnp_max_points_split(dof, 0, 0)) return EPNP_ERR_TOO_MANY_POINTS;
    HvpArgs g{};
    g.k = gb.k;
    g.grad = grad_pose_plus;
    g.tx3d = t_x3d; g.tx2d = t_x2d; g.tw2d = t_w2d; g.tdelta = t_delta; g.tcam = t_cam; g.tlb = t_lb; g.tub = t_ub;
    g.hx3d = h_x3d; g.hx2d = h_x2d; g.hw2d = h_w2d; g.hdelta = h_delta; g.hcam = h_cam; g.hlb = h_lb; g.hub = h_ub;
    g.hgrad = h_grad;
    if (!(h_x3d || h_x2d || h_w2d || h_delta || h_cam || h_lb || h_ub || h_grad)) return EPNP_OK;
    return by_dof(dof, [&](auto D) {
        return launch_plain(gn_plus_hvp_kernel<D>, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, g);
    });
}

int epnp_rslm_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                  const float* lb, const float* ub, const float* delta, const int* inds, const float* start,
                  float* pose_best, float* cost_best, float* pose_all, float* cost_all,
                  int P, int n, int B, int N, const EpnpParams* p, void* stream) {
    if (!p) return EPNP_ERR_BAD_ARG;
    RslmArgs r{};
    r.k = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    r.k.p = *p;
    r.inds = inds; r.start = start; r.pose_best = pose_best; r.cost_best = cost_best;
    r.pose_all = pose_all; r.cost_all = cost_all; r.P = P; r.n = n;
    const int rc = check_common(r.k);
    if (rc != EPNP_OK) return rc;
    if (!inds || !start || !pose_best || !cost_best || P <= 0 || n <= 0 || p->lm_iter < 0) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    return by_dof(p->dof, [&](auto D) {
        const int smem_bytes = plan_obj<D>(N).total_bytes;
        const int rc = prepare_resident(r.k, smem_bytes);
        if (rc != EPNP_OK) return rc;
        return launch_plain(rslm_kernel<D>, B, NT, smem_bytes, SmemAttr::size, (cudaStream_t)stream, r);
    });
}

int epnp_rslm_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                        const float* lb, const float* ub, const float* delta, const int* inds, const float* start,
                        float* pose_best, float* cost_best, float* pose_all, float* cost_all,
                        int P, int n, int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    if (!p) return EPNP_ERR_BAD_ARG;
    RslmArgs r{};
    r.k = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    r.k.p = *p;
    r.inds = inds; r.start = start; r.pose_best = pose_best; r.cost_best = cost_best;
    r.pose_all = pose_all; r.cost_all = cost_all; r.P = P; r.n = n;
    const int rc = check_common(r.k);
    if (rc != EPNP_OK) return rc;
    if (!inds || !start || !pose_best || !cost_best || !pose_all || !cost_all || P <= 0 || n <= 0 || p->lm_iter < 0)
        return EPNP_ERR_BAD_ARG;
    const int ctas = split_ctas_for(p->dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    if (B == 0) return EPNP_OK;
    KArgs score = r.k;                          // cost_split_kernel on the P refined poses of every object
    score.poses = pose_all; score.cost_out = cost_all; score.S_eval = P;
    const int smem_bytes = split_smem_bytes(p->dof, N, ctas, 0, 0);
    const cudaStream_t s = (cudaStream_t)stream;
    const int rows = (int)(((size_t)P * B + NT - 1) / NT);
    return by_dof(p->dof, [&](auto D) {
        // a device that cannot run the scoring cluster gets no launch at all
        int rc = launch_cluster<COST_SPLIT_TILE>(cost_split_kernel<D>, score, B, smem_bytes, ctas, s, false);
        if (rc == EPNP_OK) rc = launch_plain(rslm_refine_kernel<D>, rows, NT, 0, SmemAttr::none, s, r);
        if (rc == EPNP_OK) rc = launch_cluster<COST_SPLIT_TILE>(cost_split_kernel<D>, score, B, smem_bytes, ctas, s);
        if (rc == EPNP_OK) rc = launch_plain(rslm_select_kernel<D>, (B + NT - 1) / NT, NT, 0, SmemAttr::none, s, r);
        return rc;
    });
}

// The draw kernel's shared memory: the weights (N rounded up to 4), n indices and floats per thread.  With its 2 KB of
// static shared memory it must fit SMEM_LIMIT.
static size_t rslm_draw_smem(int N, int n) {
    return (size_t)((N + 3) & ~3) * sizeof(float) + (size_t)n * NT * (sizeof(float) + sizeof(int));
}

// epnp_rslm_draw_f32 and, with seed_ptr != NULL, epnp_rslm_draw_seedptr_f32 (the seed then comes from *seed_ptr).
static int rslm_draw(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats, const float* t_init,
                     uint64_t seed, const uint64_t* seed_ptr, uint32_t obj_offset, int* inds, float* start, float* t_out,
                     int P, int n, int B, int N, int dof, float eps, void* stream) {
    if (!w2d || !inds || !start || (dof != 4 && dof != 6) || P <= 0 || n <= 0 || B < 0 || N <= 0 || n > N)
        return EPNP_ERR_BAD_ARG;
    if (!t_init && (!x3d || !x2d || !cam_mats)) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    const size_t smem = rslm_draw_smem(N, n);
    if (smem + 2048 > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    const RslmDrawArgs r{x3d, x2d, w2d, cam_mats, t_init, inds, start, t_out, seed, obj_offset, P, n, B, N, eps};
    const cudaStream_t s = (cudaStream_t)stream;
    return by_dof(dof, [&](auto D) {
        if (seed_ptr) return launch_plain(rslm_draw_seedptr_kernel<D>, B, NT, (int)smem, SmemAttr::size, s, r, seed_ptr);
        return launch_plain(rslm_draw_kernel<D>, B, NT, (int)smem, SmemAttr::size, s, r);
    });
}

int epnp_rslm_draw_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats, const float* t_init,
                       uint64_t seed, uint32_t obj_offset, int* inds, float* start, float* t_out,
                       int P, int n, int B, int N, int dof, float eps, void* stream) {
    return rslm_draw(x3d, x2d, w2d, cam_mats, t_init, seed, nullptr, obj_offset, inds, start, t_out, P, n, B, N, dof, eps,
                     stream);
}

int epnp_rslm_draw_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                               const float* t_init, const uint64_t* seed, uint32_t obj_offset, int* inds, float* start,
                               float* t_out, int P, int n, int B, int N, int dof, float eps, void* stream) {
    if (!seed) return EPNP_ERR_BAD_ARG;
    return rslm_draw(x3d, x2d, w2d, cam_mats, t_init, 0, seed, obj_offset, inds, start, t_out, P, n, B, N, dof, eps, stream);
}

int epnp_epnp_init_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats, float conf_quantile,
                       float* pose, int* n_sel, int B, int N, void* stream) {
    if (!x3d || !x2d || !cam_mats || !pose || B < 0 || N < 4) return EPNP_ERR_BAD_ARG;
    if (!(conf_quantile >= 0.0f && conf_quantile <= 1.0f)) return EPNP_ERR_BAD_ARG;
    if (N > epnp_max_points(6, 0, 0)) return EPNP_ERR_TOO_MANY_POINTS;
    if (w2d && epnp::min_selected(N, conf_quantile) < 4) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    const EpnpInitArgs a{x3d, x2d, w2d, cam_mats, pose, n_sel, N, conf_quantile};
    return launch_plain(epnp_init_kernel, B, NT, epnp_init_smem_bytes(N), SmemAttr::size, (cudaStream_t)stream, a);
}

int epnp_epnp_init_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                             float conf_quantile, float* pose, int* n_sel, int B, int N, int cluster_ctas, void* stream) {
    if (!x3d || !x2d || !cam_mats || !pose || B < 0 || N < 4) return EPNP_ERR_BAD_ARG;
    if (!(conf_quantile >= 0.0f && conf_quantile <= 1.0f)) return EPNP_ERR_BAD_ARG;
    if (w2d && epnp::min_selected(N, conf_quantile) < 4) return EPNP_ERR_BAD_ARG;
    const int ctas = split_ctas_for(6, N, 0, 0, cluster_ctas);     // the cost kernel's plan, which bounds this one's
    if (ctas < 0) return ctas;
    const int smem_bytes = epnp_split_smem_bytes(split_share(N, ctas));
    if ((size_t)smem_bytes > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    EpnpInitArgs a{x3d, x2d, w2d, cam_mats, pose, n_sel, N, conf_quantile};
    return launch_cluster<EPNP_SPLIT_T>(epnp_init_split_kernel, a, B, smem_bytes, ctas, (cudaStream_t)stream);
}

int epnp_amis_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                  const float* lb, const float* ub, const float* delta, const float* pose_opt, const float* pose_cov,
                  const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                  uint64_t seed, uint32_t obj_offset, float* pose_samples, float* logw, float* proposals,
                  int B, int N, const EpnpParams* p, void* stream) {
    if (!p) return EPNP_ERR_BAD_ARG;
    KArgs a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.pose_opt_in = pose_opt; a.pose_cov_in = pose_cov;
    a.noise_n3 = noise_normal; a.noise_chi2 = noise_chi2; a.noise_rot = noise_rot;
    a.seed = seed; a.obj_offset = obj_offset;
    a.pose_samples = pose_samples; a.logw = logw; a.proposals = proposals; a.p = *p;
    a.prof = g_prof_buffer;
    const int rc = check_amis_call(a);
    if (rc != EPNP_OK) return rc;
    if (!pose_opt || !pose_cov) return EPNP_ERR_BAD_ARG;
    a.cov_stride = p->dof * p->dof;
    return launch_amis(a, nullptr, (cudaStream_t)stream);
}

// The checked KArgs of the fused calls (resident and split, by-value and seed-pointer forms), or the refusal.
static int fused_args(KArgs& a, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose_init,
                      const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                      uint64_t seed, uint32_t obj_offset,
                      float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                      float* pose_samples, float* logw, float* proposals, int B, int N, const EpnpParams* p) {
    if (!p) return EPNP_ERR_BAD_ARG;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.pose_init = pose_init;
    a.noise_n3 = noise_normal; a.noise_chi2 = noise_chi2; a.noise_rot = noise_rot;
    a.seed = seed; a.obj_offset = obj_offset;
    a.pose_opt = pose_opt; a.pose_cov = pose_cov; a.cost = cost; a.pose_plus = pose_opt_plus; a.cost_init = cost_init;
    a.pose_samples = pose_samples; a.logw = logw; a.proposals = proposals; a.p = *p;
    a.prof = g_prof_buffer;
    const int rc = check_amis_call(a);
    if (rc != EPNP_OK) return rc;
    return (!pose_init || !pose_opt || p->lm_iter < 0 || fast_mode_without_steps(*p)) ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

int epnp_lm_amis_fused_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                           const float* lb, const float* ub, const float* delta, const float* pose_init,
                           const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                           uint64_t seed, uint32_t obj_offset,
                           float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                           float* pose_samples, float* logw, float* proposals,
                           int B, int N, const EpnpParams* p, void* stream) {
    KArgs a{};
    const int rc = fused_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, noise_normal, noise_chi2, noise_rot,
                              seed, obj_offset, pose_opt, pose_cov, cost, pose_opt_plus, cost_init, pose_samples, logw,
                              proposals, B, N, p);
    return rc != EPNP_OK ? rc : run_lm_amis(a, nullptr, (cudaStream_t)stream);
}

int epnp_lm_amis_fused_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                   const float* lb, const float* ub, const float* delta, const float* pose_init,
                                   const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                   const uint64_t* seed, uint32_t obj_offset,
                                   float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                                   float* pose_samples, float* logw, float* proposals,
                                   int B, int N, const EpnpParams* p, void* stream) {
    if (!seed) return EPNP_ERR_BAD_ARG;
    KArgs a{};
    const int rc = fused_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, noise_normal, noise_chi2, noise_rot,
                              0, obj_offset, pose_opt, pose_cov, cost, pose_opt_plus, cost_init, pose_samples, logw,
                              proposals, B, N, p);
    return rc != EPNP_OK ? rc : run_lm_amis(a, nullptr, (cudaStream_t)stream, seed);
}

int epnp_lm_amis_fused_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                 const float* lb, const float* ub, const float* delta, const float* pose_init,
                                 const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                 uint64_t seed, uint32_t obj_offset,
                                 float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus, float* cost_init,
                                 float* pose_samples, float* logw, float* proposals,
                                 int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    KArgs a{};
    const int rc = fused_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, noise_normal, noise_chi2, noise_rot,
                              seed, obj_offset, pose_opt, pose_cov, cost, pose_opt_plus, cost_init, pose_samples, logw,
                              proposals, B, N, p);
    return rc != EPNP_OK ? rc : run_lm_amis_split(a, cluster_ctas, (cudaStream_t)stream);
}

int epnp_lm_amis_fused_split_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                         const float* lb, const float* ub, const float* delta, const float* pose_init,
                                         const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                         const uint64_t* seed, uint32_t obj_offset,
                                         float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                                         float* cost_init, float* pose_samples, float* logw, float* proposals,
                                         int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    if (!seed) return EPNP_ERR_BAD_ARG;
    KArgs a{};
    const int rc = fused_args(a, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, noise_normal, noise_chi2, noise_rot,
                              0, obj_offset, pose_opt, pose_cov, cost, pose_opt_plus, cost_init, pose_samples, logw,
                              proposals, B, N, p);
    return rc != EPNP_OK ? rc : run_lm_amis_split(a, cluster_ctas, (cudaStream_t)stream, seed);
}

// The arguments of the push calls as the solve's KArgs and the peer table, or the refusal.
static int push_args(KArgs& a, PushArgs& push, const float* x3d, const float* x2d, const float* w2d,
                     const float* cam_mats, const float* lb, const float* ub, const float* delta, const float* pose_init,
                     uint64_t seed, uint32_t obj_offset,
                     float* pose_opt, float* pose_cov, float* cost, float* pose_samples, float* logw,
                     float* const* peer_logw, float* const* peer_pose, int n_peers, int B, int N, const EpnpParams* p) {
    if (!p) return EPNP_ERR_BAD_ARG;
    if (n_peers < 0 || n_peers > EPNP_MAX_PEERS || (n_peers > 0 && (!peer_logw || !peer_pose))) return EPNP_ERR_BAD_ARG;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.pose_init = pose_init;
    a.seed = seed; a.obj_offset = obj_offset;
    a.pose_opt = pose_opt; a.pose_cov = pose_cov; a.cost = cost;
    a.pose_samples = pose_samples; a.logw = logw; a.p = *p;
    a.prof = g_prof_buffer;
    const int rc = check_amis_call(a);
    if (rc != EPNP_OK) return rc;
    if (!pose_init || !pose_opt || p->lm_iter < 0 || fast_mode_without_steps(*p)) return EPNP_ERR_BAD_ARG;
    push = PushArgs{peer_logw, peer_pose, n_peers};
    return EPNP_OK;
}

int epnp_lm_amis_fused_push_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                const float* lb, const float* ub, const float* delta, const float* pose_init,
                                uint64_t seed, uint32_t obj_offset,
                                float* pose_opt, float* pose_cov, float* cost, float* pose_samples, float* logw,
                                float* const* peer_logw, float* const* peer_pose, int n_peers,
                                int B, int N, const EpnpParams* p, void* stream) {
    KArgs a{};
    PushArgs push{};
    const int rc = push_args(a, push, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, seed, obj_offset, pose_opt,
                             pose_cov, cost, pose_samples, logw, peer_logw, peer_pose, n_peers, B, N, p);
    return rc != EPNP_OK ? rc : run_lm_amis(a, &push, (cudaStream_t)stream);
}

int epnp_lm_amis_fused_split_push_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                      const float* lb, const float* ub, const float* delta, const float* pose_init,
                                      uint64_t seed, uint32_t obj_offset,
                                      float* pose_opt, float* pose_cov, float* cost, float* pose_samples, float* logw,
                                      float* const* peer_logw, float* const* peer_pose, int n_peers,
                                      int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    KArgs a{};
    PushArgs push{};
    int rc = push_args(a, push, x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, seed, obj_offset, pose_opt,
                       pose_cov, cost, pose_samples, logw, peer_logw, peer_pose, n_peers, B, N, p);
    if (rc != EPNP_OK) return rc;
    rc = run_lm_amis_split(a, cluster_ctas, (cudaStream_t)stream);
    if (rc != EPNP_OK || n_peers == 0 || B == 0) return rc;
    const size_t blocks = ((size_t)B * p->mc_samples + 4 * NT - 1) / (4 * NT);     // one float4 of logw per thread
    const int grid = blocks < 1024 ? (int)blocks : 1024;
    return launch_plain(push_split_kernel, grid, NT, 0, SmemAttr::none, (cudaStream_t)stream, logw, pose_opt, push,
                        (size_t)obj_offset, B, p->mc_samples, p->dof == 6 ? 7 : 4);
}

int epnp_cost_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                           const float* lb, const float* ub, const float* delta,
                           const float* poses_a, const float* grad_a, int PA,
                           const float* poses_b, const float* grad_b, int PB,
                           float* grad_x3d, float* grad_x2d, float* grad_w2d, float* grad_delta,
                           int B, int N, int dof, float z_min, void* stream) {
    if (!x3d || !x2d || !w2d || !cam_mats || !delta) return EPNP_ERR_BAD_ARG;
    if ((lb == nullptr) != (ub == nullptr)) return EPNP_ERR_BAD_ARG;
    if (B < 0 || N <= 0 || PA < 0 || PB < 0 || (dof != 4 && dof != 6)) return EPNP_ERR_BAD_ARG;
    if ((PA > 0 && (!poses_a || !grad_a)) || (PB > 0 && (!poses_b || !grad_b))) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    BwArgs a{};
    a.x3d = x3d; a.x2d = x2d; a.w2d = w2d; a.cam = cam_mats; a.lb = lb; a.ub = ub; a.delta = delta;
    a.poses_a = poses_a; a.grad_a = grad_a; a.poses_b = poses_b; a.grad_b = grad_b; a.PA = PA; a.PB = PB;
    a.gx3d = grad_x3d; a.gx2d = grad_x2d; a.gw2d = grad_w2d; a.gdelta = grad_delta;
    a.B = B; a.N = N; a.z_min = z_min;
    const int smem = (BW_POSE_TILE * 13 + 2 * NW * 32) * 4;
    int sms = 0;
    const int rc = device_sms(&sms);
    if (rc != EPNP_OK) return rc;
    const int grid = B < sms * 4 ? B : sms * 4;
    return by_dof(dof, [&](auto D) {
        return launch_plain(cost_backward_kernel<D>, grid, NT, smem, SmemAttr::size, (cudaStream_t)stream, a);
    });
}

int epnp_cost_hvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* poses, const float* grad, int P,
                      const float* t_x3d, const float* t_x2d, const float* t_w2d, const float* t_delta,
                      const float* t_pose, const float* t_cam, const float* t_lb, const float* t_ub,
                      float* h_x3d, float* h_x2d, float* h_w2d, float* h_delta, float* h_pose, float* h_grad,
                      float* h_cam, float* h_lb, float* h_ub, int B, int N, int dof, float z_min, void* stream) {
    HvpArgs g{};
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = poses;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (P < 0 || (P > 0 && (!poses || !grad))) return EPNP_ERR_BAD_ARG;
    if (!lb && (t_lb || t_ub || h_lb || h_ub)) return EPNP_ERR_BAD_ARG;
    if (B == 0) return EPNP_OK;
    if (N > epnp_max_points_split(dof, 0, 0)) return EPNP_ERR_TOO_MANY_POINTS;
    g.grad = grad; g.P = P;
    g.tx3d = t_x3d; g.tx2d = t_x2d; g.tw2d = t_w2d; g.tdelta = t_delta; g.tpose = t_pose; g.tcam = t_cam;
    g.tlb = t_lb; g.tub = t_ub;
    g.hx3d = h_x3d; g.hx2d = h_x2d; g.hw2d = h_w2d; g.hdelta = h_delta; g.hpose = h_pose; g.hgrad = h_grad;
    g.hcam = h_cam; g.hlb = h_lb; g.hub = h_ub;
    const bool points = h_x3d || h_x2d || h_w2d || h_delta || h_cam || h_lb || h_ub;
    const bool poses_out = P > 0 && (h_pose || h_grad);
    const int tiles = (P + NT - 1) / NT;
    return by_dof(dof, [&](auto D) {
        int r = EPNP_OK;
        if (points) r = launch_plain(cost_hvp_point_kernel<D>, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, g);
        if (r == EPNP_OK && poses_out)
            r = launch_plain(cost_hvp_pose_kernel<D>, B * tiles, NT, 0, SmemAttr::none, (cudaStream_t)stream, g, tiles);
        return r;
    });
}

// The checked arguments of epnp_cost_pose_backward_f32 and its split form, or the refusal.
static int pose_bw_args(PoseBwArgs& g, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                        const float* lb, const float* ub, const float* delta, const float* poses, const float* grad,
                        float* grad_pose, int P, int B, int N, int dof, float z_min) {
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = poses;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min;
    g.grad = grad; g.gpose = grad_pose; g.P = P;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    return (!poses || !grad || !grad_pose || P < 0) ? EPNP_ERR_BAD_ARG : EPNP_OK;
}

int epnp_cost_pose_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                const float* lb, const float* ub, const float* delta, const float* poses,
                                const float* grad, float* grad_pose, int P, int B, int N, int dof, float z_min,
                                void* stream) {
    PoseBwArgs g{};
    const int rc = pose_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, grad, grad_pose, P, B, N, dof, z_min);
    if (rc != EPNP_OK || P == 0 || B == 0) return rc;
    return by_dof(dof, [&](auto D) {
        const int smem_bytes = plan_obj<D>(N).total_bytes;
        const int rc = prepare_resident(g.k, smem_bytes);
        if (rc != EPNP_OK) return rc;
        return launch_plain(cost_pose_backward_kernel<D>, B, NT, smem_bytes, SmemAttr::size_and_carveout,
                            (cudaStream_t)stream, g);
    });
}

int epnp_cost_pose_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                      const float* lb, const float* ub, const float* delta, const float* poses,
                                      const float* grad, float* grad_pose, int P, int B, int N, int dof, float z_min,
                                      int cluster_ctas, void* stream) {
    PoseBwArgs g{};
    const int rc = pose_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, grad, grad_pose, P, B, N, dof, z_min);
    if (rc != EPNP_OK) return rc;
    const int ctas = split_ctas_for(dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    if (P == 0) return EPNP_OK;
    const int smem_bytes = split_smem_bytes(dof, N, ctas, 0, 0);
    return by_dof(dof, [&](auto D) {
        return launch_cluster<COST_SPLIT_TILE>(cost_pose_backward_split_kernel<D>, g, B, smem_bytes, ctas,
                                               (cudaStream_t)stream);
    });
}

// The checked arguments of epnp_cost_camera_backward_f32 and its split form, or the refusal.
static int cam_bw_args(CamBwArgs& g, const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                       const float* lb, const float* ub, const float* delta, const float* poses_a, const float* grad_a,
                       int PA, const float* poses_b, const float* grad_b, int PB, float* grad_cam, float* grad_lb,
                       float* grad_ub, int B, int N, int dof, float z_min) {
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min;
    g.poses_a = poses_a; g.grad_a = grad_a; g.poses_b = poses_b; g.grad_b = grad_b; g.PA = PA; g.PB = PB;
    g.gcam = grad_cam; g.glb = grad_lb; g.gub = grad_ub;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (PA < 0 || PB < 0 || (PA > 0 && (!poses_a || !grad_a)) || (PB > 0 && (!poses_b || !grad_b)))
        return EPNP_ERR_BAD_ARG;
    return camera_outputs_ok(lb, grad_cam, grad_lb, grad_ub);
}

int epnp_cost_camera_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                  const float* lb, const float* ub, const float* delta,
                                  const float* poses_a, const float* grad_a, int PA,
                                  const float* poses_b, const float* grad_b, int PB,
                                  float* grad_cam, float* grad_lb, float* grad_ub,
                                  int B, int N, int dof, float z_min, void* stream) {
    CamBwArgs g{};
    const int rc = cam_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses_a, grad_a, PA, poses_b, grad_b, PB,
                               grad_cam, grad_lb, grad_ub, B, N, dof, z_min);
    if (rc != EPNP_OK || B == 0) return rc;
    return by_dof(dof, [&](auto D) {
        const int smem_bytes = plan_obj<D>(N).total_bytes;
        const int rc = prepare_resident(g.k, smem_bytes);
        if (rc != EPNP_OK) return rc;
        return launch_plain(cost_camera_backward_kernel<D>, B, NT, smem_bytes, SmemAttr::size_and_carveout,
                            (cudaStream_t)stream, g);
    });
}

int epnp_cost_camera_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                        const float* lb, const float* ub, const float* delta,
                                        const float* poses_a, const float* grad_a, int PA,
                                        const float* poses_b, const float* grad_b, int PB,
                                        float* grad_cam, float* grad_lb, float* grad_ub,
                                        int B, int N, int dof, float z_min, int cluster_ctas, void* stream) {
    CamBwArgs g{};
    const int rc = cam_bw_args(g, x3d, x2d, w2d, cam_mats, lb, ub, delta, poses_a, grad_a, PA, poses_b, grad_b, PB,
                               grad_cam, grad_lb, grad_ub, B, N, dof, z_min);
    if (rc != EPNP_OK) return rc;
    const int ctas = split_ctas_for(dof, N, 0, 0, cluster_ctas);
    if (ctas < 0) return ctas;
    const int smem_bytes = split_smem_bytes(dof, N, ctas, 0, 0);
    return by_dof(dof, [&](auto D) {
        return launch_cluster<COST_SPLIT_TILE>(cost_camera_backward_split_kernel<D>, g, B, smem_bytes, ctas,
                                               (cudaStream_t)stream);
    });
}

int epnp_evaluate_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                               const float* lb, const float* ub, const float* delta, const float* poses,
                               const float* grad_residual, const float* grad_jac, const float* grad_cost,
                               float* grad_x3d, float* grad_x2d, float* grad_w2d, float* grad_delta, float* grad_pose,
                               float* grad_cam, float* grad_lb, float* grad_ub, int clip_jac, int S, int B, int N,
                               int dof, float z_min, float huber_eps, void* stream) {
    EvalBwArgs g{};
    KArgs& a = g.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = poses;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min; a.p.huber_eps = huber_eps;
    g.g_res = grad_residual; g.g_jac = grad_jac; g.g_cost = grad_cost;
    g.gx3d = grad_x3d; g.gx2d = grad_x2d; g.gw2d = grad_w2d; g.gdelta = grad_delta; g.gpose = grad_pose;
    g.gcam = grad_cam; g.glb = grad_lb; g.gub = grad_ub;
    g.S = S; g.clip = clip_jac;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!poses || S < 0 || (!grad_residual && !grad_jac && !grad_cost)) return EPNP_ERR_BAD_ARG;
    const bool other = grad_x3d || grad_x2d || grad_w2d || grad_delta || grad_pose;
    if (!other && !grad_cam && !grad_lb && !grad_ub) return EPNP_ERR_BAD_ARG;
    if ((grad_lb || grad_ub) && !lb) return EPNP_ERR_BAD_ARG;
    if (B == 0 || S == 0) return EPNP_OK;
    return by_dof(dof, [&](auto D) {
        return launch_plain(evaluate_backward_kernel<D>, B, NT, 0, SmemAttr::none, (cudaStream_t)stream, g);
    });
}

int epnp_evaluate_jvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                          const float* lb, const float* ub, const float* delta, const float* poses,
                          const float* t_x3d, const float* t_x2d, const float* t_w2d, const float* t_delta,
                          const float* t_pose, const float* t_cam, const float* t_lb, const float* t_ub,
                          float* d_residual, float* d_jac, float* d_cost, int clip_jac, int S, int B, int N, int dof,
                          float z_min, float huber_eps, void* stream) {
    JvpArgs g{};
    KArgs& a = g.h.k;
    a = problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta, B, N);
    a.poses = poses;
    epnp_default_params(&a.p, dof);
    a.p.z_min = z_min; a.p.huber_eps = huber_eps;
    const int rc = check_common(a);
    if (rc != EPNP_OK) return rc;
    if (!poses || S < 0 || (long long)S * B > 2147483647LL || (!d_residual && !d_jac && !d_cost)) return EPNP_ERR_BAD_ARG;
    if (!lb && (t_lb || t_ub)) return EPNP_ERR_BAD_ARG;
    if (B == 0 || S == 0) return EPNP_OK;
    g.h.P = S;
    g.h.tx3d = t_x3d; g.h.tx2d = t_x2d; g.h.tw2d = t_w2d; g.h.tdelta = t_delta; g.h.tpose = t_pose; g.h.tcam = t_cam;
    g.h.tlb = t_lb; g.h.tub = t_ub;
    g.dres = d_residual; g.djac = d_jac; g.dcost = d_cost; g.clip = clip_jac;
    const bool pose_major = !d_residual && !d_jac && S >= JVP_POSE_MAJOR_MIN_S;
    const int tiles = (S + NT - 1) / NT;
    return by_dof(dof, [&](auto D) {
        if (pose_major)
            return launch_plain(evaluate_jvp_cost_kernel<D>, B * tiles, NT, 0, SmemAttr::none, (cudaStream_t)stream, g,
                                tiles);
        return launch_plain(evaluate_jvp_kernel<D>, S * B, NT, 0, SmemAttr::none, (cudaStream_t)stream, g);
    });
}

}  // extern "C"

// ---- host-buffer entry points: chunked H2D -> solve -> D2H on two internal streams
namespace {

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct WsLayout {
    size_t x3d, x2d, w2d, cam, lb, ub, delta, pose_init, pose_opt, pose_cov, cost, samples, logw;
    size_t inds, start, pose_all, cost_all, cost_best;   // the RSLM initialiser's (P, B, .) and (B) scratch
    size_t P, n, total;                                  // P = n = 0 without it
};

// init [opt]: the initialiser of epnp_solve_host_f32; without it (the fused host calls) the layout ends at logw.
WsLayout ws_layout(int B, int N, const EpnpParams* p, const EpnpInit* init = nullptr) {
    const size_t D = (p->dof == 6) ? 7 : 4, dof = p->dof, M = p->mc_samples;
    const bool rslm = init && init->kind == EPNP_INIT_RSLM;
    WsLayout w; size_t o = 0;
    w.x3d = o; o += align256((size_t)B * N * 3 * 4);
    w.x2d = o; o += align256((size_t)B * N * 2 * 4);
    w.w2d = o; o += align256((size_t)B * N * 2 * 4);
    w.cam = o; o += align256((size_t)B * 9 * 4);
    w.lb = o; o += align256((size_t)B * 2 * 4);
    w.ub = o; o += align256((size_t)B * 2 * 4);
    w.delta = o; o += align256((size_t)B * 4);
    w.pose_init = o; o += align256((size_t)B * D * 4);
    w.pose_opt = o; o += align256((size_t)B * D * 4);
    w.pose_cov = o; o += align256((size_t)B * dof * dof * 4);
    w.cost = o; o += align256((size_t)B * 4);
    w.samples = o; o += align256((size_t)B * M * D * 4);
    w.logw = o; o += align256((size_t)B * M * 4);
    w.P = rslm && init->num_proposals > 0 ? (size_t)init->num_proposals : 0;
    w.n = rslm && init->num_points > 0 ? (size_t)init->num_points : 0;
    w.inds = o; o += align256(w.P * B * w.n * 4);
    w.start = o; o += align256(w.P * B * D * 4);
    w.pose_all = o; o += align256(w.P * B * D * 4);
    w.cost_all = o; o += align256(w.P * B * 4);
    w.cost_best = o; o += align256(rslm ? (size_t)B * 4 : 0);
    w.total = o;
    return w;
}

// Helper streams of the host-buffer entry points: one copy-in, two compute, one copy-out stream per host
// thread, created on first use and kept for the life of the thread (the only resource the library owns;
// creating and destroying four streams per call costs more than a whole chunk of work).
struct HostPipe {
    cudaStream_t in = nullptr, k[2] = {nullptr, nullptr}, out = nullptr;
    int device = -1;
    cudaError_t ensure() {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev == device && in) return cudaSuccess;
        if (in) { cudaStreamDestroy(in); cudaStreamDestroy(k[0]); cudaStreamDestroy(k[1]); cudaStreamDestroy(out); in = nullptr; }
        if ((e = cudaStreamCreateWithFlags(&in, cudaStreamNonBlocking)) != cudaSuccess) return e;
        if ((e = cudaStreamCreateWithFlags(&k[0], cudaStreamNonBlocking)) != cudaSuccess) return e;
        if ((e = cudaStreamCreateWithFlags(&k[1], cudaStreamNonBlocking)) != cudaSuccess) return e;
        if ((e = cudaStreamCreateWithFlags(&out, cudaStreamNonBlocking)) != cudaSuccess) return e;
        device = dev;
        return cudaSuccess;
    }
};
thread_local HostPipe g_pipe;

// The caller's host arrays of a host-buffer call.
struct HostBufs {
    const float *x3d, *x2d, *w2d, *cam, *lb, *ub, *delta, *pose_init;     // lb / ub, pose_init [opt]
    float *pose_opt, *pose_cov, *cost, *samples, *logw;                     // all but pose_opt [opt]
};

// One chunk's rows [b0, b0 + nb) of every workspace array, the global index of its first object and its stream.
struct Chunk {
    const float *x3d, *x2d, *w2d, *cam, *lb, *ub, *delta;
    float *pose_init, *pose_opt, *pose_cov, *cost, *samples, *logw;
    int* inds;
    float *start, *pose_all, *cost_all, *cost_best;
    uint32_t obj_offset;
    int nb;
    cudaStream_t stream;
};

Chunk chunk_at(char* ws, const WsLayout& w, int b0, int nb, int N, const EpnpParams* p, bool bounded,
                      uint32_t obj_offset, cudaStream_t stream) {
    const size_t D = (p->dof == 6) ? 7 : 4, dof = p->dof, M = p->mc_samples, b = (size_t)b0;
    const auto at = [&](size_t field, size_t per) { return (float*)(ws + field) + b * per; };
    Chunk c;
    c.x3d = at(w.x3d, (size_t)N * 3); c.x2d = at(w.x2d, (size_t)N * 2); c.w2d = at(w.w2d, (size_t)N * 2);
    c.cam = at(w.cam, 9); c.delta = at(w.delta, 1);
    c.lb = bounded ? at(w.lb, 2) : nullptr; c.ub = bounded ? at(w.ub, 2) : nullptr;
    c.pose_init = at(w.pose_init, D); c.pose_opt = at(w.pose_opt, D); c.pose_cov = at(w.pose_cov, dof * dof);
    c.cost = at(w.cost, 1); c.samples = at(w.samples, M * D); c.logw = at(w.logw, M);
    c.inds = (int*)at(w.inds, w.P * w.n); c.start = at(w.start, w.P * D); c.pose_all = at(w.pose_all, w.P * D);
    c.cost_all = at(w.cost_all, w.P); c.cost_best = at(w.cost_best, 1);
    c.obj_offset = obj_offset + (uint32_t)b0;
    c.nb = nb;
    c.stream = stream;
    return c;
}

// The argument checks both fused host-buffer calls make first: EPNP_OK or EPNP_ERR_BAD_ARG.
int check_host_args(const HostBufs& h, void* workspace, size_t workspace_bytes, int B, int N, const EpnpParams* p) {
    if (!p || !workspace || !h.x3d || !h.x2d || !h.w2d || !h.cam || !h.delta || !h.pose_init || !h.pose_opt || !h.logw)
        return EPNP_ERR_BAD_ARG;
    if ((h.lb == nullptr) != (h.ub == nullptr)) return EPNP_ERR_BAD_ARG;
    if (B < 0 || N <= 0) return EPNP_ERR_BAD_ARG;
    if (workspace_bytes < ws_layout(B, N, p).total) return EPNP_ERR_BAD_ARG;
    return EPNP_OK;
}

// LM + AMIS on one chunk: epnp_lm_amis_fused_f32, or its split form with cluster_ctas.
int lm_amis_chunk(const Chunk& c, uint64_t seed, int N, const EpnpParams* p, bool split, int cluster_ctas) {
    if (split)
        return epnp_lm_amis_fused_split_f32(c.x3d, c.x2d, c.w2d, c.cam, c.lb, c.ub, c.delta, c.pose_init, nullptr, nullptr,
                                            nullptr, seed, c.obj_offset, c.pose_opt, c.pose_cov, c.cost, nullptr, nullptr,
                                            c.samples, c.logw, nullptr, c.nb, N, p, cluster_ctas, c.stream);
    return epnp_lm_amis_fused_f32(c.x3d, c.x2d, c.w2d, c.cam, c.lb, c.ub, c.delta, c.pose_init, nullptr, nullptr, nullptr,
                                  seed, c.obj_offset, c.pose_opt, c.pose_cov, c.cost, nullptr, nullptr, c.samples, c.logw,
                                  nullptr, c.nb, N, p, c.stream);
}

// The chunked copy-in / solve / copy-out pipeline of the host-buffer calls, after their checks (B > 0): solve(chunk)
// enqueues a chunk's work on chunk.stream.  n_chunks = 0: cut the batch at whole waves of `wave` objects the device
// solves at once (a chunk of 1.7 waves costs 2), as few waves per chunk as the 64-chunk limit allows (one chunk when
// wave = 0); n_chunks >= 1: that many equal chunks.  h.pose_init and h.logw are copied only when given.
template <class Solve>
int host_pipeline(Solve solve, int wave, const HostBufs& h, void* workspace, const WsLayout& w,
                         uint32_t obj_offset, int n_chunks, int B, int N, const EpnpParams* p, void* stream_) {
    int chunk_objects = 0;
    if (n_chunks == 0) {
        if (wave > 0) {
            const int waves_per_chunk = (B + 64 * wave - 1) / (64 * wave);
            chunk_objects = wave * waves_per_chunk;
            n_chunks = (B + chunk_objects - 1) / chunk_objects;
        }
    }
    if (n_chunks < 1) n_chunks = 1;
    if (n_chunks > B) n_chunks = B;
    if (n_chunks > 64) n_chunks = 64;
    cudaStream_t stream = (cudaStream_t)stream_;
    char* ws = (char*)workspace;
    const size_t D = (p->dof == 6) ? 7 : 4, dof = p->dof, M = p->mc_samples;
    // Three-stage pipeline over object chunks: copy-in stream -> {compute 0, compute 1} -> copy-out stream, chained
    // by per-chunk events, so all H2D copies run back to back on one DMA engine, all D2H copies on the other, and
    // the solve of chunk c overlaps both (and the tail of chunk c-1 on the other compute stream).
    cudaError_t e = cudaSuccess;
    int rc = EPNP_OK;
    cudaEvent_t fork = nullptr, ev_in[64], ev_k[64], done[3] = {nullptr, nullptr, nullptr};
    for (int i = 0; i < 64; ++i) { ev_in[i] = nullptr; ev_k[i] = nullptr; }
#define EPNP_TRY(x) do { e = (x); if (e != cudaSuccess) { rc = cuda_fail(e); goto done; } } while (0)
    EPNP_TRY(g_pipe.ensure());
    EPNP_TRY(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
    EPNP_TRY(cudaEventRecord(fork, stream));
    EPNP_TRY(cudaStreamWaitEvent(g_pipe.in, fork, 0));
    EPNP_TRY(cudaStreamWaitEvent(g_pipe.k[0], fork, 0));
    EPNP_TRY(cudaStreamWaitEvent(g_pipe.k[1], fork, 0));
    EPNP_TRY(cudaStreamWaitEvent(g_pipe.out, fork, 0));
    for (int c = 0; c < n_chunks; ++c) {
        const int b0 = chunk_objects ? c * chunk_objects : (int)((long long)B * c / n_chunks);
        const int b1 = chunk_objects ? (b0 + chunk_objects < B ? b0 + chunk_objects : B) : (int)((long long)B * (c + 1) / n_chunks);
        const int nb = b1 - b0;
        if (nb <= 0) continue;
        cudaStream_t sk = g_pipe.k[c & 1];
#define H2D(field, host, per) EPNP_TRY(cudaMemcpyAsync(ws + w.field + (size_t)b0 * (per) * 4, (host) + (size_t)b0 * (per), (size_t)nb * (per) * 4, cudaMemcpyHostToDevice, g_pipe.in))
#define D2H(field, host, per) EPNP_TRY(cudaMemcpyAsync((host) + (size_t)b0 * (per), ws + w.field + (size_t)b0 * (per) * 4, (size_t)nb * (per) * 4, cudaMemcpyDeviceToHost, g_pipe.out))
        H2D(x3d, h.x3d, (size_t)N * 3); H2D(x2d, h.x2d, (size_t)N * 2); H2D(w2d, h.w2d, (size_t)N * 2);
        H2D(cam, h.cam, 9); H2D(delta, h.delta, 1);
        if (h.pose_init) H2D(pose_init, h.pose_init, D);
        if (h.lb) { H2D(lb, h.lb, 2); H2D(ub, h.ub, 2); }
        EPNP_TRY(cudaEventCreateWithFlags(&ev_in[c], cudaEventDisableTiming));
        EPNP_TRY(cudaEventRecord(ev_in[c], g_pipe.in));
        EPNP_TRY(cudaStreamWaitEvent(sk, ev_in[c], 0));
        rc = solve(chunk_at(ws, w, b0, nb, N, p, h.lb != nullptr, obj_offset, sk));
        if (rc != EPNP_OK) goto done;
        EPNP_TRY(cudaEventCreateWithFlags(&ev_k[c], cudaEventDisableTiming));
        EPNP_TRY(cudaEventRecord(ev_k[c], sk));
        EPNP_TRY(cudaStreamWaitEvent(g_pipe.out, ev_k[c], 0));
        D2H(pose_opt, h.pose_opt, D);
        if (h.logw) D2H(logw, h.logw, M);
        if (h.pose_cov) D2H(pose_cov, h.pose_cov, dof * dof);
        if (h.cost) D2H(cost, h.cost, 1);
        if (h.samples) D2H(samples, h.samples, M * D);
#undef H2D
#undef D2H
    }
    {   // join: the caller's stream waits for everything the helpers were given
        cudaStream_t all[3] = {g_pipe.out, g_pipe.k[0], g_pipe.k[1]};
        for (int i = 0; i < 3; ++i) {
            EPNP_TRY(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
            EPNP_TRY(cudaEventRecord(done[i], all[i]));
            EPNP_TRY(cudaStreamWaitEvent(stream, done[i], 0));
        }
    }
done:
#undef EPNP_TRY
    // events are released once recorded work has drained (cudaEventDestroy defers)
    for (int i = 0; i < 64; ++i) { if (ev_in[i]) cudaEventDestroy(ev_in[i]); if (ev_k[i]) cudaEventDestroy(ev_k[i]); }
    for (int i = 0; i < 3; ++i) if (done[i]) cudaEventDestroy(done[i]);
    if (fork) cudaEventDestroy(fork);
    return rc;
}

// ---- host-buffer solve from a given pose or from scratch (epnp_solve_host_f32, epnp_solve_split_host_f32)

// What the two calls compose on every chunk.
struct SolveSpec {
    const EpnpInit* init;                       // [opt]: NULL when the caller gives pose_init
    uint64_t seed;                              // the AMIS seed
    const EpnpParams* p;
    int N;
    bool split;
    int cluster_ctas;                           // as the caller gave it: 0 lets each split stage pick its own C
    bool want_cov, want_cost;                   // LM only: passed to epnp_lm_solve_f32 when the caller asked
};

// The refusals of the composed device calls that only a non-empty batch gets -- a resident launch's shared memory, a
// cluster the device cannot co-schedule -- checked without launching, and `wave`: the objects the heaviest stage
// (the AMIS kernel, else the initialiser's) solves at once, asked for when n_chunks = 0.
struct SolvePlan {
    int B;
    bool want_wave;
    int wave;
};

int plan_rslm(const SolveSpec& s, SolvePlan& plan) {
    const int dof = s.p->dof, N = s.N;
    int* wave = plan.want_wave ? &plan.wave : nullptr;
    if (rslm_draw_smem(N, s.init->num_points) + 2048 > SMEM_LIMIT) return EPNP_ERR_TOO_MANY_POINTS;
    return by_dof(dof, [&](auto D) {
        if (!s.split) {
            const int smem_bytes = plan_obj<D>(N).total_bytes;
            if ((size_t)smem_bytes > SMEM_LIMIT) return (int)EPNP_ERR_TOO_MANY_POINTS;
            if (wave) *wave = resident_objects<NT>(rslm_kernel<D>, smem_bytes, SmemAttr::size);
            return (int)EPNP_OK;
        }
        const int ctas = split_ctas_for(dof, N, 0, 0, s.cluster_ctas);
        KArgs unused{};                         // launch = false: launch_cluster does not read the kernel's arguments
        return launch_cluster<COST_SPLIT_TILE>(cost_split_kernel<D>, unused, plan.B, split_smem_bytes(dof, N, ctas, 0, 0),
                                               ctas, nullptr, false, wave);
    });
}

int plan_epnp(const SolveSpec& s, SolvePlan& plan) {
    int* wave = plan.want_wave ? &plan.wave : nullptr;
    if (!s.split) {
        if (wave) *wave = resident_objects<NT>(epnp_init_kernel, epnp_init_smem_bytes(s.N), SmemAttr::size);
        return EPNP_OK;
    }
    const int ctas = split_ctas_for(6, s.N, 0, 0, s.cluster_ctas);
    EpnpInitArgs unused{};
    return launch_cluster<EPNP_SPLIT_T>(epnp_init_split_kernel, unused, plan.B, epnp_split_smem_bytes(split_share(s.N, ctas)),
                                        ctas, nullptr, false, wave);
}

int plan_amis(const SolveSpec& s, SolvePlan& plan) {
    const EpnpParams& p = *s.p;
    if (s.split) {
        int wave = 0;
        const int ctas = split_lm_amis_plan(p, plan.B, s.N, s.cluster_ctas, &wave);
        if (plan.want_wave) plan.wave = wave;
        return ctas < 0 ? ctas : EPNP_OK;
    }
    if (plan.want_wave)
        plan.wave = by_dof(p.dof, [&](auto D) {
            return by_amis_threads(s.N, [&](auto T) {
                return resident_objects<T>(amis_kernel<D, T>, amis_smem_bytes<D>(s.N, p.mc_samples));
            });
        });
    return EPNP_OK;
}

// One chunk of the composed solve, stage by stage, each a public device call on chunk c.  With `plan` (c.nb = 0, a dry
// run that enqueues nothing) every call returns what it refuses for an empty batch, and, when plan->B > 0, the stage's
// plan adds what it refuses only for a non-empty one: the first refusal is the one the composition would meet.
int solve_chunk(const SolveSpec& s, const Chunk& c, SolvePlan* plan) {
    const EpnpInit* in = s.init;
    const EpnpParams* p = s.p;
    const bool check = plan && plan->B > 0;
    int rc = EPNP_OK;
    if (in && in->kind == EPNP_INIT_RSLM) {
        const int P = in->num_proposals, n = in->num_points;
        rc = epnp_rslm_draw_f32(c.x3d, c.x2d, c.w2d, c.cam, nullptr, in->seed, c.obj_offset, c.inds, c.start, nullptr, P,
                                n, c.nb, s.N, p->dof, in->rslm.eps, c.stream);
        if (rc != EPNP_OK) return rc;
        rc = s.split ? epnp_rslm_split_f32(c.x3d, c.x2d, c.w2d, c.cam, c.lb, c.ub, c.delta, c.inds, c.start, c.pose_init,
                                           c.cost_best, c.pose_all, c.cost_all, P, n, c.nb, s.N, &in->rslm,
                                           s.cluster_ctas, c.stream)
                     : epnp_rslm_f32(c.x3d, c.x2d, c.w2d, c.cam, c.lb, c.ub, c.delta, c.inds, c.start, c.pose_init,
                                     c.cost_best, nullptr, nullptr, P, n, c.nb, s.N, &in->rslm, c.stream);
        if (rc == EPNP_OK && check) rc = plan_rslm(s, *plan);
    } else if (in) {
        rc = s.split ? epnp_epnp_init_split_f32(c.x3d, c.x2d, c.w2d, c.cam, in->conf_quantile, c.pose_init, nullptr, c.nb,
                                                s.N, s.cluster_ctas, c.stream)
                     : epnp_epnp_init_f32(c.x3d, c.x2d, c.w2d, c.cam, in->conf_quantile, c.pose_init, nullptr, c.nb, s.N,
                                          c.stream);
        if (rc == EPNP_OK && check) rc = plan_epnp(s, *plan);
    }
    if (rc != EPNP_OK) return rc;
    if (p->mc_samples == 0)
        return epnp_lm_solve_f32(c.x3d, c.x2d, c.w2d, c.cam, c.lb, c.ub, c.delta, c.pose_init, c.pose_opt,
                                 s.want_cov ? c.pose_cov : nullptr, s.want_cost ? c.cost : nullptr, nullptr, nullptr,
                                 c.nb, s.N, p, c.stream);
    rc = lm_amis_chunk(c, s.seed, s.N, p, s.split, s.cluster_ctas);
    if (rc == EPNP_OK && check) rc = plan_amis(s, *plan);
    return rc;
}

// The argument checks of the two calls that no composed device call makes: EPNP_OK or EPNP_ERR_BAD_ARG.
int check_solve_host_args(const HostBufs& h, const EpnpInit* init, void* workspace, size_t workspace_bytes,
                                 int B, int N, const EpnpParams* p) {
    if (!p || !workspace || !h.x3d || !h.x2d || !h.w2d || !h.cam || !h.delta || !h.pose_opt) return EPNP_ERR_BAD_ARG;
    if ((h.lb == nullptr) != (h.ub == nullptr)) return EPNP_ERR_BAD_ARG;
    if (B < 0 || N <= 0 || p->mc_samples < 0) return EPNP_ERR_BAD_ARG;
    if ((h.pose_init == nullptr) == (init == nullptr)) return EPNP_ERR_BAD_ARG;        // exactly one start
    if (p->mc_samples == 0 ? (h.logw || h.samples) : !h.logw) return EPNP_ERR_BAD_ARG;
    if (init) {
        if (init->kind == EPNP_INIT_RSLM) {
            if (init->rslm.dof != p->dof) return EPNP_ERR_BAD_ARG;
        } else if (init->kind != EPNP_INIT_EPNP || p->dof != 6) {                  // EPnP gives 6DoF poses only
            return EPNP_ERR_BAD_ARG;
        }
    }
    if (workspace_bytes < ws_layout(B, N, p, init).total) return EPNP_ERR_BAD_ARG;
    return EPNP_OK;
}

int solve_host(const HostBufs& h, const EpnpInit* init, uint64_t seed, uint32_t obj_offset, void* workspace,
                      size_t workspace_bytes, int n_chunks, int B, int N, const EpnpParams* p, bool split,
                      int cluster_ctas, void* stream) {
    int rc = check_solve_host_args(h, init, workspace, workspace_bytes, B, N, p);
    if (rc != EPNP_OK) return rc;
    const WsLayout w = ws_layout(B, N, p, init);
    const SolveSpec s{init, seed, p, N, split, cluster_ctas, h.pose_cov != nullptr, h.cost != nullptr};
    SolvePlan plan{B, n_chunks == 0, 0};
    // every refusal before the first copy: the whole composition dry-run on an empty chunk
    rc = solve_chunk(s, chunk_at((char*)workspace, w, 0, 0, N, p, h.lb != nullptr, obj_offset, (cudaStream_t)stream),
                     &plan);
    if (rc != EPNP_OK || B == 0) return rc;
    return host_pipeline([&](const Chunk& c) { return solve_chunk(s, c, nullptr); }, plan.wave, h, workspace, w,
                         obj_offset, n_chunks, B, N, p, stream);
}

}  // namespace

extern "C" {

size_t epnp_fused_workspace_bytes(int B, int N, const EpnpParams* p) {
    if (!p || B < 0 || N <= 0) return 0;
    return ws_layout(B, N, p).total;
}

size_t epnp_solve_workspace_bytes(int B, int N, const EpnpParams* p, const EpnpInit* init) {
    if (!p || B < 0 || N <= 0) return 0;
    if (init && init->kind != EPNP_INIT_EPNP &&
        (init->kind != EPNP_INIT_RSLM || init->num_proposals <= 0 || init->num_points <= 0))
        return 0;
    return ws_layout(B, N, p, init).total;
}

int epnp_lm_amis_fused_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                                const float* cam_mats_host, const float* lb_host, const float* ub_host,
                                const float* delta_host, const float* pose_init_host,
                                uint64_t seed, uint32_t obj_offset,
                                float* pose_opt_host, float* pose_cov_host, float* cost_host,
                                float* pose_samples_host, float* logw_host,
                                void* workspace, size_t workspace_bytes, int n_chunks,
                                int B, int N, const EpnpParams* p, void* stream) {
    const HostBufs h{x3d_host, x2d_host, w2d_host, cam_mats_host, lb_host, ub_host, delta_host, pose_init_host,
                     pose_opt_host, pose_cov_host, cost_host, pose_samples_host, logw_host};
    const int rc = check_host_args(h, workspace, workspace_bytes, B, N, p);
    if (rc != EPNP_OK || B == 0) return rc;
    int wave = 0;                               // objects in flight: SMs x resident AMIS CTAs per SM
    if (n_chunks == 0) {
        if (check_amis_params(*p) != EPNP_OK) return EPNP_ERR_BAD_ARG;
        wave = by_dof(p->dof, [&](auto D) {
            return by_amis_threads(N, [&](auto T) {
                return resident_objects<T>(amis_kernel<D, T>, amis_smem_bytes<D>(N, p->mc_samples));
            });
        });
    }
    return host_pipeline([&](const Chunk& c) { return lm_amis_chunk(c, seed, N, p, false, 0); }, wave, h, workspace,
                         ws_layout(B, N, p), obj_offset, n_chunks, B, N, p, stream);
}

int epnp_lm_amis_fused_split_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                                      const float* cam_mats_host, const float* lb_host, const float* ub_host,
                                      const float* delta_host, const float* pose_init_host,
                                      uint64_t seed, uint32_t obj_offset,
                                      float* pose_opt_host, float* pose_cov_host, float* cost_host,
                                      float* pose_samples_host, float* logw_host,
                                      void* workspace, size_t workspace_bytes, int n_chunks,
                                      int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    const HostBufs h{x3d_host, x2d_host, w2d_host, cam_mats_host, lb_host, ub_host, delta_host, pose_init_host,
                     pose_opt_host, pose_cov_host, cost_host, pose_samples_host, logw_host};
    int rc = check_host_args(h, workspace, workspace_bytes, B, N, p);
    if (rc != EPNP_OK || B == 0) return rc;
    // every refusal of the chunk solves, made here, before the first copy is enqueued
    if ((p->dof != 4 && p->dof != 6) || check_amis_params(*p) != EPNP_OK || p->lm_iter < 0 || fast_mode_without_steps(*p))
        return EPNP_ERR_BAD_ARG;
    int wave = 0;                               // objects in flight: co-resident clusters
    const int ctas = split_lm_amis_plan(*p, B, N, cluster_ctas, &wave);
    if (ctas < 0) return ctas;
    return host_pipeline([&](const Chunk& c) { return lm_amis_chunk(c, seed, N, p, true, ctas); }, wave, h, workspace,
                         ws_layout(B, N, p), obj_offset, n_chunks, B, N, p, stream);
}

int epnp_solve_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                        const float* cam_mats_host, const float* lb_host, const float* ub_host,
                        const float* delta_host, const float* pose_init_host, const EpnpInit* init,
                        uint64_t seed, uint32_t obj_offset,
                        float* pose_opt_host, float* pose_cov_host, float* cost_host,
                        float* pose_samples_host, float* logw_host,
                        void* workspace, size_t workspace_bytes, int n_chunks,
                        int B, int N, const EpnpParams* p, void* stream) {
    const HostBufs h{x3d_host, x2d_host, w2d_host, cam_mats_host, lb_host, ub_host, delta_host, pose_init_host,
                     pose_opt_host, pose_cov_host, cost_host, pose_samples_host, logw_host};
    return solve_host(h, init, seed, obj_offset, workspace, workspace_bytes, n_chunks, B, N, p, false, 0, stream);
}

int epnp_solve_split_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                              const float* cam_mats_host, const float* lb_host, const float* ub_host,
                              const float* delta_host, const float* pose_init_host, const EpnpInit* init,
                              uint64_t seed, uint32_t obj_offset,
                              float* pose_opt_host, float* pose_cov_host, float* cost_host,
                              float* pose_samples_host, float* logw_host,
                              void* workspace, size_t workspace_bytes, int n_chunks,
                              int B, int N, const EpnpParams* p, int cluster_ctas, void* stream) {
    const HostBufs h{x3d_host, x2d_host, w2d_host, cam_mats_host, lb_host, ub_host, delta_host, pose_init_host,
                     pose_opt_host, pose_cov_host, cost_host, pose_samples_host, logw_host};
    return solve_host(h, init, seed, obj_offset, workspace, workspace_bytes, n_chunks, B, N, p, true, cluster_ctas,
                      stream);
}

}  // extern "C"
