// pnp_lm.cuh -- the Levenberg-Marquardt / Gauss-Newton pose solve (LMSolver.solve, levenberg_marquardt.py:80-241) as a
// WARP-PER-OBJECT kernel, and the CTA-wide normal-equation evaluation the backward kernel of the GN step still uses.
//
// Why one warp per object.  An LM iteration is: evaluate the 28 sums (21 J^T J + 6 J^T r + cost) over the N points at
// the candidate pose, then a short serial chain (6x6 damped Cholesky solve, SE(3) retraction, trust-region update).
// With a 128-thread CTA per object (round 1) each thread saw only N / 128 = 4 points between two block barriers and
// 127 threads idled through the serial chain: the phase was latency-bound (tools/split_probe.py times it).  With a
// warp per object a lane owns N / 32 = 16 points (long independent instruction
// streams), the reduction is 31 shuffles with no block barrier, the serial chain costs the same issue slots as before
// but 12-14 other warps of the SM -- other OBJECTS -- fill the scheduler meanwhile.  No __syncthreads anywhere.
//
// Data: the object's raw {x3d, x2d, w2d} arrays (28 N bytes) are pulled from HBM once by three cp.async.bulk copies
// into the warp's shared memory (lane l reads x3d[3 (l + 32 k) + c]: stride 3 floats, conflict-free; x2d / w2d as
// float2) and re-read from there by the K + 1 evaluations; for N above LM_STAGE_MAX_N (dense coordinate maps) the
// evaluations read global memory instead (L1 / L2 resident after the first pass).
//
// Long point sets: WARPS = 8 warps share one object -- warp w takes points 32 w + lane, 32 (w + 8) + lane, ... -- and their
// 28 partial sums meet in shared memory (one extra block barrier pair per evaluation): the dense 64 x 64 coordinate maps
// (N = 4096, typically a few hundred objects) would otherwise run one latency-bound warp per SM.  The warp count is a
// function of N only, so an object's result never depends on the batch it is solved in.
#pragma once
#include "pnp_device.cuh"

namespace {

constexpr int LM_STAGE_MAX_N = 640;     // 28 N bytes of shared memory per warp: 17.9 KB -> 12 resident warps per SM.  Below
                                        // that the K + 1 evaluations read shared memory instead of going back to L1 / L2

constexpr int LM_MAX_WARPS = 8;
template <int DOF, int WARPS> struct LmHead {
    uint64_t bar;
    float ev[32];                       // reduced evaluation: NV floats
    LMState<DOF> lm;
    float cov[DOF * DOF];
    float part[WARPS > 1 ? WARPS * 32 : 1];     // per-warp partial sums (WARPS > 1)
};

template <int WARPS> __device__ __forceinline__ void lm_group_sync() {
    if constexpr (WARPS == 1) __syncwarp(); else __syncthreads();
}

__host__ __device__ inline int lm_padded_points(int N) { return (N + 3) / 4 * 4; }
template <int DOF, int WARPS> __host__ __device__ inline int lm_head_bytes() { return (int)((sizeof(LmHead<DOF, WARPS>) + 127) / 128 * 128); }
template <int DOF, int WARPS> __host__ __device__ inline int lm_smem_bytes(int N, bool staged) {
    return lm_head_bytes<DOF, WARPS>() + (staged ? 28 * lm_padded_points(N) : 0);
}

// Normal equations at `pose` over the object's N points by the object's WARPS warps: result in ev[0..NV) (visible to
// every thread of the group on return).  Jacobian rows u / v in the two lanes of fp32x2 registers (27 V2 multiply-adds
// per point, two FFMA each on sm_90a).
template <int DOF, bool CLIP, int WARPS>
__device__ __forceinline__ void warp_normal_eq(const float* p3, const float* p2, const float* pw, int N, const float* pose,
                                               const Cam& cam, float delta, float huber_eps, float* ev, float* part) {
    constexpr int NP = Dim<DOF>::NA + DOF;
    const int lane = threadIdx.x & 31;
    float R[9], t[3];
    {
        float ps[Dim<DOF>::POSE];
#pragma unroll
        for (int i = 0; i < Dim<DOF>::POSE; ++i) ps[i] = pose[i];
        pose_to_rot<DOF>(ps, R);
        t[0] = ps[0]; t[1] = ps[1]; t[2] = ps[2];
    }
    V2 acc2[NP];
#pragma unroll
    for (int i = 0; i < NP; ++i) acc2[i] = v2splat(0.f);
    const V2 kuv[3] = {v2(cam.k[0], cam.k[3]), v2(cam.k[1], cam.k[4]), v2(cam.k[2], cam.k[5])};
    float cost = 0.f;
    const float2* uv2 = reinterpret_cast<const float2*>(p2);
    const float2* w2 = reinterpret_cast<const float2*>(pw);
    for (int n = threadIdx.x; n < N; n += 32 * WARPS) {
        const float X = p3[3 * n], Y = p3[3 * n + 1], Z = p3[3 * n + 2];
        const float2 uv = uv2[n], w = w2[n];
        point_normal_eq_rows<DOF, CLIP>(R, t, cam, kuv, delta, huber_eps, X, Y, Z, -uv.x, -uv.y, w.x, w.y, acc2, cost);
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < NP; ++i) acc[i] = acc2[i].x + acc2[i].y;
    acc[NP] = cost;
#pragma unroll
    for (int i = NP + 1; i < 32; ++i) acc[i] = 0.f;
    const float tot = warp_transpose_sum(acc);
    if constexpr (WARPS == 1) {
        ev[lane] = tot;
        __syncwarp();
    } else {
        part[(threadIdx.x >> 5) * 32 + lane] = tot;
        __syncthreads();
        if (threadIdx.x < 32) {
            float v = part[lane];
#pragma unroll
            for (int w = 1; w < WARPS; ++w) v += part[w * 32 + lane];
            ev[lane] = v;
        }
        __syncthreads();
    }
}

// One object per CTA of WARPS warps (blockDim.x = 32 WARPS, blockIdx.x = object).
template <int DOF, bool STAGED, int WARPS>
__global__ void __launch_bounds__(32 * WARPS) lm_warp_kernel(const KArgs a) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    LmHead<DOF, WARPS>& sh = *reinterpret_cast<LmHead<DOF, WARPS>*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE;
    const Params& p = a.p;
    const int lane = threadIdx.x, obj = blockIdx.x, N = a.N;     // `lane`: index within the object's group of 32 WARPS threads
    const float *p3, *p2, *pw;
    if constexpr (STAGED) {
        float* st = reinterpret_cast<float*>(smem_raw + lm_head_bytes<DOF, WARPS>());
        const int np = lm_padded_points(N);
        float *s3 = st, *s2 = st + 3 * np, *sw = st + 5 * np;
        const float* g3 = a.x3d + (size_t)obj * N * 3;
        const float* g2 = a.x2d + (size_t)obj * N * 2;
        const float* gw = a.w2d + (size_t)obj * N * 2;
        if (a.use_tma) {
            if (lane == 0) {
                mbar_init(&sh.bar, 1);
                fence_barrier_init();
                mbar_expect_tx(&sh.bar, (uint32_t)N * 28u);
                tma_load_1d(s3, g3, (uint32_t)N * 12u, &sh.bar);
                tma_load_1d(s2, g2, (uint32_t)N * 8u, &sh.bar);
                tma_load_1d(sw, gw, (uint32_t)N * 8u, &sh.bar);
            }
            lm_group_sync<WARPS>();
            mbar_wait(&sh.bar, 0u);
        } else {
            for (int i = lane; i < 3 * N; i += 32 * WARPS) s3[i] = __ldg(g3 + i);
            for (int i = lane; i < 2 * N; i += 32 * WARPS) { s2[i] = __ldg(g2 + i); sw[i] = __ldg(gw + i); }
            lm_group_sync<WARPS>();
        }
        p3 = s3; p2 = s2; pw = sw;
    } else {
        p3 = a.x3d + (size_t)obj * N * 3;
        p2 = a.x2d + (size_t)obj * N * 2;
        pw = a.w2d + (size_t)obj * N * 2;
    }
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < PD; ++i) sh.lm.pose[i] = __ldg(a.pose_init + (size_t)obj * PD + i);
        sh.lm.radius = p.initial_radius;
        sh.lm.shrink = 2.0f;
    }
    lm_group_sync<WARPS>();
    if (!p.fast_mode) {
        warp_normal_eq<DOF, true, WARPS>(p3, p2, pw, N, sh.lm.pose, cam, delta, p.huber_eps, sh.ev, sh.part);
        if (lane == 0) {
            lm_adopt<DOF>(sh.lm, sh.ev);
            if (a.cost_init) a.cost_init[obj] = sh.lm.cost;
            if (p.lm_iter > 0) lm_propose<DOF>(sh.lm, p);
        }
        lm_group_sync<WARPS>();
        for (int it = 0; it < p.lm_iter; ++it) {
            warp_normal_eq<DOF, true, WARPS>(p3, p2, pw, N, sh.lm.pose_new, cam, delta, p.huber_eps, sh.ev, sh.part);
            if (lane == 0) {
                lm_update<DOF>(sh.lm, sh.ev, p);
                if (it + 1 < p.lm_iter) lm_propose<DOF>(sh.lm, p);
            }
            lm_group_sync<WARPS>();
        }
    } else {
        for (int it = 0; it < p.lm_iter; ++it) {
            warp_normal_eq<DOF, false, WARPS>(p3, p2, pw, N, sh.lm.pose, cam, delta, p.huber_eps, sh.ev, sh.part);
            if (lane == 0) {
                lm_adopt<DOF>(sh.lm, sh.ev);                 // kept for covariance / cost (pre-step)
                if (it == 0 && a.cost_init) a.cost_init[obj] = sh.lm.cost;
                gn_advance<DOF>(sh.lm.pose, sh.ev, p.eps, sh.lm.pose);
            }
            lm_group_sync<WARPS>();
        }
    }
    if (lane < PD) a.pose_opt[(size_t)obj * PD + lane] = sh.lm.pose[lane];
    if (lane == 8 && a.cost) a.cost[obj] = sh.lm.cost;
    if (a.pose_cov) {
        if (lane < DOF) {                   // one covariance column per lane (fp64 Cholesky + one solve)
            float col[DOF];
            pose_covariance_column<DOF>(sh.lm.a, p.eps, lane, col);
#pragma unroll
            for (int i = 0; i < DOF; ++i) sh.cov[i * DOF + lane] = col[i];
        }
        lm_group_sync<WARPS>();
        for (int i = lane; i < DOF * DOF; i += 32 * WARPS) a.pose_cov[(size_t)obj * a.cov_stride + i] = sh.cov[i];
    }
    if (a.pose_plus) {      // y* (+) one undamped GN step, clip_jac always on (gn_step default)
        lm_group_sync<WARPS>();
        warp_normal_eq<DOF, true, WARPS>(p3, p2, pw, N, sh.lm.pose, cam, delta, p.huber_eps, sh.ev, sh.part);
        if (lane == 0) {
            float plus[PD];
            gn_advance<DOF>(sh.lm.pose, sh.ev, p.eps, plus);
#pragma unroll
            for (int i = 0; i < PD; ++i) a.pose_plus[(size_t)obj * PD + i] = plus[i];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// CTA-wide evaluation over the packed pair records (gn_plus_backward_kernel): 128 threads stride over the pairs,
// 28 partial sums per thread reduced by the transposed butterfly + one cross-warp pass; result in ev[0..NV).
template <int DOF, bool CLIP>
__device__ void eval_normal_eq(const float* pts, int N, const float* pose, const Cam& cam, float delta,
                               float huber_eps, float* red, float* ev) {
    constexpr int NV = Dim<DOF>::NV;
    float R[9], t[3];
    {
        float ps[Dim<DOF>::POSE];
#pragma unroll
        for (int i = 0; i < Dim<DOF>::POSE; ++i) ps[i] = pose[i];
        pose_to_rot<DOF>(ps, R);
        t[0] = ps[0]; t[1] = ps[1]; t[2] = ps[2];
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    const float4* p4 = reinterpret_cast<const float4*>(pts);
    const int npair = (N + 1) >> 1;
    for (int j = threadIdx.x; j < npair; j += NT) {
        const float4 q0 = p4[4 * j], q1 = p4[4 * j + 1], q2 = p4[4 * j + 2], q3 = p4[4 * j + 3];
        point_normal_eq<DOF, CLIP>(R, t, cam, delta, huber_eps, q0.x, q0.z, q1.x, -q1.z, -q2.x, q2.z, q3.x, acc);
        if (2 * j + 1 < N)
            point_normal_eq<DOF, CLIP>(R, t, cam, delta, huber_eps, q0.y, q0.w, q1.y, -q1.w, -q2.y, q2.w, q3.y, acc);
    }
    const float tot = warp_transpose_sum(acc);
    red[(threadIdx.x >> 5) * 32 + (threadIdx.x & 31)] = tot;
    __syncthreads();
    if (threadIdx.x < NV) {
        const int j = threadIdx.x;
        ev[j] = (red[j] + red[32 + j]) + (red[64 + j] + red[96 + j]);
    }
    __syncthreads();
}

}  // namespace
