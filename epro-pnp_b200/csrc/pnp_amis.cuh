// pnp_amis.cuh -- the adaptive-multiple-importance-sampling loop of EProPnPBase.monte_carlo_forward
// (epropnp.py:132-182; 6DoF proposals :288-342, 4DoF :199-260) as a CTA-PER-OBJECT kernel.  One loop, amis_loop, serves
// both pose families, the resident and the cluster-split kernels; the families differ only in the draw, the proposal
// density, the refit and the proposal dump.
//
//   * the object's correspondences are pulled from HBM once (TMA ring -> 64-byte pair records in shared memory);
//   * one thread owns one sample of an iteration: draws it (injected noise or Philox), sweeps all N points with the
//     pre-multiplied projection K[R|t] (points are shared-memory broadcasts, two points side by side in fp32x2
//     register pairs), evaluates the proposal densities it needs; the mixture density of a sample is kept as ONE
//     running log-sum-exp;
//   * a log-weight is -cost - (lse - log count): it is recomputed where needed instead of stored, and the staging ring
//     lives inside the (not yet written) sample buffer, so a CTA needs 36.1 KB at N = M = 512; five CTAs share an SM
//     (96 registers per thread);
//   * the proposal refit is four block reductions (transposed butterflies) + a short chain on one lane.
// The LM solution (pose, covariance) comes from global memory: lm_warp_kernel wrote it just before (same stream).
//
// Long point sets (N >= 2048, the dense 64 x 64 coordinate maps) leave room for one CTA per SM only; there the CTA has
// T = 512 threads: the cost sweep of a sample is cut into T / 128 = 4 point ranges swept by four threads (their partial
// costs meet in shared memory, summed in range order), every other pass simply strides over the samples with 512 threads.
#pragma once
#include "pnp_device.cuh"

namespace {

// Resident CTAs per SM the 128-thread kernel is compiled for.  Six fit in shared memory (36.1 KB at N = M = 512) at 80
// registers; ptxas then spills 76 bytes, none of it inside the sweep loops.  H100 SXM at a 400 W power limit (power-capped,
// SM clock 1575-1690 MHz), 4096 objects, 3 alternating runs each: amis_kernel 1.222 ms at five against 1.245 ms at six,
// 2.483 M against 2.420 M objects/s on the bench step, so five stay.  (Eight point pairs per sweep trip instead of four, same
// chains: 1.256 ms at five.)
constexpr int AMIS_CTAS_PER_SM = 5;

template <int DOF> struct ProposalOf;
template <> struct ProposalOf<6> { typedef Proposal6 type; };
template <> struct ProposalOf<4> { typedef Proposal4 type; };

constexpr int AMIS_T_DENSE = 512;          // threads per CTA for long point sets
constexpr int AMIS_DENSE_MIN_N = 2048;     // a function of N only: an object's result must not depend on its batch
constexpr int AMIS_CHUNK_DENSE = 512;      // points per TMA chunk there (one per thread and chunk)

template <int DOF, int T> struct AmisHead {
    uint64_t bar[2];
    float red[2 * (T / 32) * 32];           // two halves: consecutive reductions alternate, one barrier each
    float pose[8];                          // the LM solution ...
    float cov[DOF * DOF];                   // ... and its covariance
    float box[6];                           // bounding box of the object's points (point_box)
    typename ProposalOf<DOF>::type prop[MAX_ITER];
};

struct AmisPlan {        // offsets in floats from the start of dynamic smem
    int stage, pts, smp, cost, logp, cpart, total_bytes;
};

// The staging ring is dead once the object is packed and the sample buffer is not written before the AMIS loop, so the
// ring lives inside it whenever it fits.
template <int DOF, int T>
__host__ __device__ inline AmisPlan plan_amis(int N, int M) {
    AmisPlan s;
    int off = (int)((sizeof(AmisHead<DOF, T>) + 127) / 128 * 128 / 4);
    constexpr int ring = 2 * 7 * (T > NT ? AMIS_CHUNK_DENSE : CH);
    const bool alias = Dim<DOF>::POSE * M >= ring;
    s.stage = off; if (!alias) off += ring;
    s.pts = off; off += 16 * ((N + 1) / 2);        // 64 B per pair of points
    s.smp = off; off += Dim<DOF>::POSE * M;
    if (alias) s.stage = s.smp;
    s.cost = off; off += M;
    s.logp = off; off += M;                         // running log-sum-exp of the proposal densities, one per sample
    s.cpart = off; if (T > NT) off += (T / NT) * M; // partial costs of the point ranges (T / 128 sweeping threads per sample)
    s.total_bytes = off * 4;
    return s;
}

// running log-sum-exp over the proposals seen so far
struct RunningLse {
    float top, acc;
    __device__ __forceinline__ void start(float lp) { top = lp; acc = 1.f; }
    __device__ __forceinline__ void add(float lp) {
        if (lp > top) { acc = fmaf(acc, fast_exp(top - lp), 1.f); top = lp; }
        else acc += fast_exp(lp - top);
    }
    __device__ __forceinline__ float value() const { return top + fast_log(acc); }
};
__device__ __forceinline__ float log_add_exp(float a, float b) {
    const float hi = fmaxf(a, b), lo = fminf(a, b);
    return (lo == -CUDART_INF_F) ? hi : hi + fast_log1p(fast_exp(lo - hi));
}

// The 6DoF refit's block sums in the resident (T = NT) kernel: block_sum with the transposed butterfly unrolled one
// template instance per stage, so every stage's trip count is a constant and the W = 16 or 32 values stay in registers.
// In block_sum's warp_transpose_sum_w the stage count is a loop variable, the inner loops stay partly rolled and the
// values go through a local-memory copy indexed per lane (LDL / STL on the latency-bound refit chain).  Same adds in the
// same order, so the same bits.  T != NT keeps block_sum and its code, and so does the 4DoF refit: its 6-value sums do not reach local memory.
template <int W, int HALF> __device__ __forceinline__ void amis_transpose_stage(float (&v)[W], int lane) {
    constexpr int MASK = 32 * HALF / W;     // 16 at the first stage (HALF = W / 2), halving with HALF
    const bool up = (lane & MASK) != 0;
#pragma unroll
    for (int k = 0; k < HALF; ++k) {
        const float keep = up ? v[k + HALF] : v[k];
        const float send = up ? v[k] : v[k + HALF];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, MASK);
    }
    if constexpr (HALF > 1) amis_transpose_stage<W, HALF / 2>(v, lane);
}
template <int K, int T> __device__ __forceinline__ void amis_block_sum(float (&v)[K], float* red, int half) {
    if constexpr (T != NT) {
        block_sum<K, T>(v, red, half);
    } else {
        static_assert(K > 4 && K <= 32, "amis_block_sum: 5..32 values");
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        float* r = red + half * NT;
        constexpr int W = K <= 8 ? 8 : (K <= 16 ? 16 : 32);
        constexpr int SH = W == 8 ? 2 : (W == 16 ? 1 : 0);
        float w[W];
#pragma unroll
        for (int k = 0; k < W; ++k) w[k] = k < K ? v[k] : 0.f;
        amis_transpose_stage<W, W / 2>(w, lane);
        float tot = w[0];
#pragma unroll
        for (int o = 16 / W; o >= 1; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
        if ((lane & ((1 << SH) - 1)) == 0 && (lane >> SH) < K) r[warp * 32 + (lane >> SH)] = tot;
        __syncthreads();
        const float mine = lane < K ? sum_warp_partials<NT>(r, lane) : 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = __shfl_sync(0xffffffffu, mine, k);
    }
}

// One object's AMIS loop split over a thread-block cluster (amis_split_kernel): this CTA is rank `rank` of `ctas` and
// holds `npair` pair records of the object.  xbuf: 2 S floats of this CTA's shared memory, the per-sample partial costs
// of its point range in the half of the current iteration's parity.
struct SplitCtx {
    float* xbuf;
    int rank, ctas, npair;
};

__device__ __forceinline__ float proposal_logpdf(const Proposal6& pr, const float* q) { return proposal_logpdf6(pr, q); }
__device__ __forceinline__ float proposal_logpdf(const Proposal4& pr, const float* q) { return proposal_logpdf4(pr, q); }

// ------------------------------------------------------------------------------------------------
// The AMIS loop of one object, either pose family.  sh.prop[0] holds the first proposal (the kernel fitted it to the LM
// solution).  Where the families differ, each keeps the form its kernels were validated with (a common form, such as
// the 6DoF register copy of a sample in the 4DoF sweep, compiles them differently).  4DoF (EProPnP4DoF,
// epropnp.py:199-260): the yaw proposal is 0.75 von Mises + 0.25 uniform, and injected noise_rot (B, M) holds the yaw
// draws themselves (the reference samples them with numpy on the host, distributions.py:61-72, so there is no base
// noise to replay).
// SPLIT: the cluster form (sc describes the CTA's share); every rank draws the same samples and, after the exchange of
// the partial costs, holds the same costs, so each runs the same refits; rank 0 alone writes the outputs.
template <int DOF, int T, bool SPLIT>
__device__ void amis_loop(const KArgs& a, AmisHead<DOF, T>& sh, const float* pts4, float* smp, float* cst, float* logp,
                          float* cpart, const Cam& cam, float delta, int obj, const SplitCtx sc = SplitCtx{}) {
    constexpr int PARTS = T / NT;           // threads sweeping one sample (1: the thread that drew it)
    constexpr int PD = Dim<DOF>::POSE;
    const Params& p = a.p;
    const int tid = threadIdx.x;
    const int M = p.mc_samples, I = p.mc_iter, S = M / I;
    const bool injected = a.noise_n3 != nullptr;
    const int st = serial_thread<T>(a);
    float* const logw_out = a.logw + (size_t)obj * M;
    PH_DECL;

    for (int i = 0; i < I; ++i) {
        // ---- draw, cost, densities of the new samples (one sample per thread and pass; T > 128: the first 128 threads
        // draw, then T / 128 threads sweep one point range each of every sample)
        for (int s = tid; s < S; s += NT) {
            if (PARTS > 1 && tid >= NT) break;
            const int m = i * S + s;
            float n3[3], n4[4], chi2, q[PD];        // n4: the rotation's base noise (6DoF)
            if (injected) {
                const size_t g = (size_t)obj * M + m;
                n3[0] = __ldg(a.noise_n3 + g * 3); n3[1] = __ldg(a.noise_n3 + g * 3 + 1); n3[2] = __ldg(a.noise_n3 + g * 3 + 2);
                chi2 = __ldg(a.noise_chi2 + g);
                if constexpr (DOF == 6) {
                    n4[0] = __ldg(a.noise_rot + g * 4); n4[1] = __ldg(a.noise_rot + g * 4 + 1);
                    n4[2] = __ldg(a.noise_rot + g * 4 + 2); n4[3] = __ldg(a.noise_rot + g * 4 + 3);
                } else {
                    q[3] = __ldg(a.noise_rot + g);
                }
            } else if constexpr (DOF == 6) {
                draw_base_noise(a.seed, a.obj_offset + (uint32_t)obj, (uint32_t)m, n3, chi2, n4);
            } else {
                draw_base_noise_t(a.seed, a.obj_offset + (uint32_t)obj, (uint32_t)m, n3, chi2);
                q[3] = draw_yaw(a.seed, a.obj_offset + (uint32_t)obj, (uint32_t)m, s, S, sh.prop[i].mode, sh.prop[i].kappa);
            }
            if constexpr (DOF == 6) proposal_draw6(sh.prop[i], n3, chi2, n4, q);
            else draw_translation(sh.prop[i].mu, sh.prop[i].lt, n3, chi2, q);
#pragma unroll
            for (int k = 0; k < PD; ++k) smp[m * PD + k] = q[k];
            if constexpr (PARTS == 1) cst[m] = pose_cost_pairs<DOF>(pts4, 0, (a.N + 1) >> 1, q, cam, delta, sh.box);
            RunningLse l;
            l.start(proposal_logpdf(sh.prop[0], q));
            for (int j = 1; j <= i; ++j) l.add(proposal_logpdf(sh.prop[j], q));
            logp[m] = l.value();
        }
        if constexpr (PARTS > 1) {
            __syncthreads();
            const int part = tid / NT, npair = SPLIT ? sc.npair : (a.N + 1) >> 1;
            const int j0 = (int)((long long)npair * part / PARTS) & ~3, j1 = part + 1 == PARTS ? npair : ((int)((long long)npair * (part + 1) / PARTS) & ~3);
            for (int s = tid % NT; s < S; s += NT) {
                const int m = i * S + s;
                if constexpr (DOF == 6) {
                    float q[7];
#pragma unroll
                    for (int k = 0; k < 7; ++k) q[k] = smp[m * 7 + k];
                    cpart[part * M + m] = pose_cost_pairs<6>(pts4, j0, j1, q, cam, delta, sh.box);
                } else {
                    cpart[part * M + m] = pose_cost_pairs<4>(pts4, j0, j1, smp + m * 4, cam, delta, sh.box);
                }
            }
            __syncthreads();
            for (int s = tid; s < S; s += T) {
                const int m = i * S + s;
                float c = cpart[m];
#pragma unroll
                for (int r = 1; r < PARTS; ++r) c += cpart[r * M + m];
                if constexpr (SPLIT) sc.xbuf[(i & 1) * S + s] = c;
                else cst[m] = c;
            }
            if constexpr (SPLIT) {
                // One cluster barrier per iteration: the half (i & 1) of xbuf is written again at iteration i + 2, after
                // the barrier of iteration i + 1, which every rank reaches only once its reads below are done.
                cluster_sync();
                for (int s = tid; s < S; s += T) cst[i * S + s] = sum_ranks(sc.xbuf + (i & 1) * S + s, sc.ctas);
            }
        }
        PH_MARK(a, PH_DRAW_SWEEP);
        // ---- the new proposal on all earlier samples
        for (int m = tid; m < i * S; m += T) {
            if constexpr (DOF == 6) {
                float q[7];
#pragma unroll
                for (int k = 0; k < 7; ++k) q[k] = smp[m * 7 + k];
                logp[m] = log_add_exp(logp[m], proposal_logpdf6(sh.prop[i], q));
            } else {
                logp[m] = log_add_exp(logp[m], proposal_logpdf4(sh.prop[i], smp + m * 4));
            }
        }
        __syncthreads();
        PH_MARK(a, PH_LOGP_OLD);
        // ---- log-weights of all samples so far: -cost - log(mixture density)
        const int n = (i + 1) * S;
        const float log_cnt = logf((float)(i + 1));
        auto logweight = [&](int m) { return -cst[m] - (logp[m] - log_cnt); };
        if (i == I - 1) {
            if (!SPLIT || sc.rank == 0)
                for (int m = tid; m < M; m += T) { logw_out[m] = logweight(m); SPLIT_AUDIT_STORES(1); }
            PH_MARK(a, PH_OUTPUT);
            break;
        }
        float mx = -CUDART_INF_F;
        for (int m = tid; m < n; m += T) mx = fmaxf(mx, logweight(m));
        PH_MARK(a, PH_WEIGHTS);
        // ---- refit proposal i+1 to the weighted samples (estimate_params; 6DoF epropnp.py:317-342, 4DoF :232-260).
        // One block reduction, one barrier each:
        //   A  max of the log-weights
        //   B  e = exp(lw - max): sum e, sum e t; 6DoF: and ACG fixed-point iteration 1 (Lambda_0 = I, so
        //      M = q.q) -- the normalisation of the weights cancels in Lambda; 4DoF: and sum e sin, sum e cos
        //   C  translation covariance about the mean (6DoF: + ACG iteration 2)
        //   D+ 6DoF: remaining ACG iterations
        mx = block_max<T>(mx, sh.red, 0);
        // the refit's results live to the end of the iteration: scoped to the 6DoF branch, they change that family's
        // 512-thread code
        float lam10[10];                    // 6DoF: the ACG scatter
        float mean[3], inv_sum;
        float tc[6];
        if constexpr (DOF == 6) {
            {
                float acc[15];
#pragma unroll
                for (int r = 0; r < 15; ++r) acc[r] = 0.f;
                for (int m = tid; m < n; m += T) {
                    const float e = fast_exp(logweight(m) - mx);
                    const float* s7 = smp + m * 7;
                    acc[0] += e;
                    acc[1] = fmaf(e, s7[0], acc[1]); acc[2] = fmaf(e, s7[1], acc[2]); acc[3] = fmaf(e, s7[2], acc[3]);
                    const float* q = s7 + 3;
                    const float mq = fmaxf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3], p.amis_eps);
                    const float wm = e / mq;
                    acc[4] += wm;
                    int idx = 5;
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = r; c < 4; ++c) { acc[idx] = fmaf(wm * q[r], q[c], acc[idx]); ++idx; }
                }
                amis_block_sum<15, T>(acc, sh.red, 1);
                inv_sum = 1.0f / acc[0];
                mean[0] = acc[1] * inv_sum; mean[1] = acc[2] * inv_sum; mean[2] = acc[3] * inv_sum;
                const float inv0 = 1.0f / acc[4];
#pragma unroll
                for (int r = 0; r < 10; ++r) lam10[r] = acc[5 + r] * inv0;
                lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
            }
            if (p.acg_mle_iter == 0) {          // degenerate configuration: Lambda stays the identity
#pragma unroll
                for (int r = 0; r < 10; ++r) lam10[r] = 0.f;
                lam10[0] = lam10[4] = lam10[7] = lam10[9] = 1.f;
            }
            {
                const bool more = p.acg_mle_iter >= 2;
                float lam_inv[16];
                if (more) acg_scatter_inverse(lam10, lam_inv);
                float acc[17];
#pragma unroll
                for (int r = 0; r < 17; ++r) acc[r] = 0.f;
                for (int m = tid; m < n; m += T) {
                    const float w = fast_exp(logweight(m) - mx) * inv_sum;       // normalised softmax weight
                    const float* s7 = smp + m * 7;
                    const float d0 = s7[0] - mean[0], d1 = s7[1] - mean[1], d2 = s7[2] - mean[2];
                    acc[11] = fmaf(w * d0, d0, acc[11]); acc[12] = fmaf(w * d0, d1, acc[12]); acc[13] = fmaf(w * d0, d2, acc[13]);
                    acc[14] = fmaf(w * d1, d1, acc[14]); acc[15] = fmaf(w * d1, d2, acc[15]); acc[16] = fmaf(w * d2, d2, acc[16]);
                    if (more) {
                        const float* q = s7 + 3;
                        const float wm = w / fmaxf(quad4(lam_inv, q), p.amis_eps);
                        acc[0] += wm;
                        int idx = 1;
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int c = r; c < 4; ++c) { acc[idx] = fmaf(wm * q[r], q[c], acc[idx]); ++idx; }
                    }
                }
                amis_block_sum<17, T>(acc, sh.red, 0);
#pragma unroll
                for (int r = 0; r < 6; ++r) tc[r] = acc[11 + r];
                if (more) {
                    const float inv0 = 1.0f / acc[0];
#pragma unroll
                    for (int r = 0; r < 10; ++r) lam10[r] = acc[1 + r] * inv0;
                    lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
                }
            }
            for (int itr = 2; itr < p.acg_mle_iter; ++itr) {
                float lam_inv[16];
                acg_scatter_inverse(lam10, lam_inv);
                float acc[11];
#pragma unroll
                for (int r = 0; r < 11; ++r) acc[r] = 0.f;
                for (int m = tid; m < n; m += T) {
                    const float* q = smp + m * 7 + 3;
                    const float wm = fast_exp(logweight(m) - mx) * inv_sum / fmaxf(quad4(lam_inv, q), p.amis_eps);
                    acc[0] += wm;
                    int idx = 1;
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = r; c < 4; ++c) { acc[idx] = fmaf(wm * q[r], q[c], acc[idx]); ++idx; }
                }
                amis_block_sum<11, T>(acc, sh.red, (itr + 1) & 1);
                const float inv0 = 1.0f / acc[0];
#pragma unroll
                for (int r = 0; r < 10; ++r) lam10[r] = acc[1 + r] * inv0;
                lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
            }
            PH_MARK(a, PH_REFIT_SUMS);
            if (tid == st) refit_finish6(mean, tc, lam10, p.acg_dispersion, sh.prop[i + 1]);
        } else {
            float accB[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int m = tid; m < n; m += T) {
                const float e = fast_exp(logweight(m) - mx);
                const float* s4 = smp + m * 4;
                float sn, cs;
                sincosf(s4[3], &sn, &cs);
                accB[0] += e;
                accB[1] = fmaf(e, s4[0], accB[1]); accB[2] = fmaf(e, s4[1], accB[2]); accB[3] = fmaf(e, s4[2], accB[3]);
                accB[4] = fmaf(e, sn, accB[4]); accB[5] = fmaf(e, cs, accB[5]);
            }
            block_sum<6, T>(accB, sh.red, 1);
            inv_sum = 1.0f / accB[0];
            mean[0] = accB[1] * inv_sum; mean[1] = accB[2] * inv_sum; mean[2] = accB[3] * inv_sum;
#pragma unroll
            for (int r = 0; r < 6; ++r) tc[r] = 0.f;
            for (int m = tid; m < n; m += T) {
                const float w = fast_exp(logweight(m) - mx) * inv_sum;
                const float* s4 = smp + m * 4;
                const float d0 = s4[0] - mean[0], d1 = s4[1] - mean[1], d2 = s4[2] - mean[2];
                tc[0] = fmaf(w * d0, d0, tc[0]); tc[1] = fmaf(w * d0, d1, tc[1]); tc[2] = fmaf(w * d0, d2, tc[2]);
                tc[3] = fmaf(w * d1, d1, tc[3]); tc[4] = fmaf(w * d1, d2, tc[4]); tc[5] = fmaf(w * d2, d2, tc[5]);
            }
            block_sum<6, T>(tc, sh.red, 0);
            PH_MARK(a, PH_REFIT_SUMS);
            if (tid == st) refit_finish4(mean, tc, accB[4] * inv_sum, accB[5] * inv_sum, p.amis_eps, sh.prop[i + 1]);
        }
        PH_MARK(a, PH_REFIT_FINISH);
        __syncthreads();
    }
    if (a.proposals && tid < I && (!SPLIT || sc.rank == 0)) {   // (B, I, 19): mu3, Lt6, then Lr10 or mode, kappa, 0...
        float* o = a.proposals + ((size_t)obj * I + tid) * PROP_FLOATS;
        SPLIT_AUDIT_STORES(PROP_FLOATS);
        const typename ProposalOf<DOF>::type& pr = sh.prop[tid];
        o[0] = pr.mu[0]; o[1] = pr.mu[1]; o[2] = pr.mu[2];
#pragma unroll
        for (int r = 0; r < 6; ++r) o[3 + r] = pr.lt[r];
        if constexpr (DOF == 6) {
#pragma unroll
            for (int r = 0; r < 10; ++r) o[9 + r] = pr.lr[r];
        } else {
            o[9] = pr.mode; o[10] = pr.kappa;
#pragma unroll
            for (int r = 11; r < PROP_FLOATS; ++r) o[r] = 0.f;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Optional epilogue of the multi-GPU path: when an object is finished, its CTA also stores the object's pose and its M
// log-weights into row (obj_offset + obj) of the full-batch result buffers of up to EPNP_MAX_PEERS other GPUs (pointers
// into their memory, mapped through CUDA IPC): plain st.global over NVLink, 2 KB + 28 B per object and peer, issued
// object by object underneath the other CTAs' math.  No gather kernel and no copy afterwards; the caller only needs a
// rendezvous before reading (sharded.PushGather).  The peers' buffer addresses come as two DEVICE arrays of pointers
// (like a batched-BLAS pointer array): the kernel takes 20 bytes of parameters for the feature, not a 136-byte table.
constexpr int EPNP_MAX_PEERS = 8;
struct PushArgs {
    float* const* logw;                     // device array [n]: (B_total, M) buffer of each peer
    float* const* pose;                     // device array [n]: (B_total, D) buffer of each peer
    int n;
};

// dst[0, n) = src[0, n) by the T threads of the CTA: float4 runs where n and both addresses allow, single floats otherwise.
template <int T>
__device__ __forceinline__ void block_copy(float* dst, const float* src, int n) {
    const int tid = threadIdx.x;
    if ((n & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
        for (int q = tid; q < n / 4; q += T) reinterpret_cast<float4*>(dst)[q] = reinterpret_cast<const float4*>(src)[q];
    } else {
        for (int m = tid; m < n; m += T) dst[m] = src[m];
    }
}

// The push epilogue of one object: its M log-weights (as this CTA wrote them to global memory) and its pose go to row
// `row` of every peer's buffers.  Not inlined: it must not take part in the main body's register allocation (inlined,
// it would weigh on every caller, pushing or not).
template <int T>
__device__ __noinline__ void push_rows(const float* src, const float* pose, size_t row, int M, int PD,
                                       float* const* peer_logw, float* const* peer_pose, int n) {
    const int tid = threadIdx.x;
    for (int r = 0; r < n; ++r) {
        block_copy<T>(peer_logw[r] + row * M, src, M);
        if (tid < PD) peer_pose[r][row * PD + tid] = pose[tid];
    }
}

// The serial thread's part of the set-up: the LM solution and its covariance from global memory, and the first proposal
// fitted to them (EProPnP*.initial_fit: fp64 factorizations, ~12 k cycles on one lane).  The covariance is read BEFORE
// this object's sample rows are written: the fused entry point may have parked it there (cov_stride = M * D); plain
// loads, that memory is written later in this launch.
template <int DOF, int T>
__device__ __forceinline__ void amis_initial_fit(const KArgs& a, AmisHead<DOF, T>& sh, int obj) {
    constexpr int PD = Dim<DOF>::POSE;
#pragma unroll
    for (int i = 0; i < PD; ++i) sh.pose[i] = a.pose_opt_in[(size_t)obj * PD + i];
#pragma unroll
    for (int i = 0; i < DOF * DOF; ++i) sh.cov[i] = a.pose_cov_in[(size_t)obj * a.cov_stride + i];
    if constexpr (DOF == 6) initial_fit6(sh.pose, sh.cov, a.p.acg_dispersion, sh.prop[0]);
    else initial_fit4(sh.pose, sh.cov, a.p.amis_eps, sh.prop[0]);
}

// One object per CTA of T threads (blockIdx.x = object).  The body of amis_kernel and amis_seedptr_kernel.
template <int DOF, int T>
__device__ __forceinline__ void amis_body(const KArgs& a, const PushArgs& push) {
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    AmisHead<DOF, T>& sh = *reinterpret_cast<AmisHead<DOF, T>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE;
    const int M = a.p.mc_samples;
    const AmisPlan pl = plan_amis<DOF, T>(a.N, M);
    const int st = serial_thread<T>(a);
    (void)st;
    float* pts4 = dyn + pl.pts;
    const int obj = blockIdx.x, tid = threadIdx.x;
    PH_DECL;
    // Set-up, two things at once: the serial warp's lane 0 fits the first proposal, the other warps meanwhile pull the
    // object's correspondences through the TMA ring and pack them (named barrier 1 among themselves).
    const int serial_warp = st >> 5;
    if ((tid >> 5) == serial_warp) {
        if (tid == st) amis_initial_fit(a, sh, obj);
    } else {
        LoaderT<(T > NT ? AMIS_CHUNK_DENSE : CH)> ld(a, sh.bar, dyn + pl.stage);
        ld.template load_object<T>(obj, pts4, serial_warp);
    }
    __syncthreads();
    point_box<T>(pts4, a.N, sh.red + (T / 32) * 32, sh.box);     // the second half of `red`: the AMIS loop starts on the first
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    PH_MARK(a, PH_LOAD);
    amis_loop<DOF, T, false>(a, sh, pts4, dyn + pl.smp, dyn + pl.cost, dyn + pl.logp, dyn + pl.cpart, cam, delta, obj);
    // The samples leave as one contiguous run per object: `smp` holds them in the output's (M, PD) layout, complete since
    // the AMIS loop's last barrier.  (The covariance the fused call may have parked in these rows was read at set-up.)
    block_copy<T>(a.pose_samples + (size_t)obj * M * PD, dyn + pl.smp, M * PD);
    // In-kernel gather (push.n > 0, uniform for the launch).  A run-time branch of ONE kernel, not a second instantiation:
    // a sharded run must be bit-identical to the single-GPU run, and two instantiations are two compilations -- as
    // template variants the push / plain pair need not agree bit for bit, since each compilation allocates registers
    // and orders the arithmetic on its own.
    if (push.n > 0) {
        __syncthreads();                                        // the CTA's own global stores are visible to all its threads
        push_rows<T>(a.logw + (size_t)obj * M, sh.pose, (size_t)a.obj_offset + (size_t)obj, M, PD, push.logw, push.pose, push.n);
    }
}

template <int DOF, int T>
__global__ void __launch_bounds__(T, T == NT ? AMIS_CTAS_PER_SM : 1) amis_kernel(const KArgs a, const PushArgs push) {
    amis_body<DOF, T>(a, push);
}

// amis_kernel with the Philox seed read from device memory at entry, so that a CUDA graph replaying the launch draws
// from whatever seed the graph (or the caller) wrote there last, instead of the one it was captured with.
template <int DOF, int T>
__global__ void __launch_bounds__(T, T == NT ? AMIS_CTAS_PER_SM : 1)
    amis_seedptr_kernel(const KArgs a, const PushArgs push, const uint64_t* seed) {
    KArgs s = a;
    s.seed = *seed;
    amis_body<DOF, T>(s, push);
}

// ------------------------------------------------------------------------------------------------
// Objects whose points do not fit one SM: one object per thread-block CLUSTER of `ctas` CTAs (grid = B * ctas), rank r
// holding the contiguous point range [r share, (r + 1) share) (split_share).  Every rank runs the whole AMIS control
// flow of amis_kernel<DOF, 512> on the same samples -- Philox keyed by (seed, obj_offset + object, m), or the same
// injected noise -- and sweeps only its own range, in the dense kernel's four point ranges.  Per iteration the ranks
// exchange their per-sample partial costs through distributed shared memory and add them (sum_ranks), so all ranks
// hold bit-identical costs and log-densities and compute the refits redundantly (no proposal broadcast).  The result
// depends on ctas, never on B, the shard or obj_offset.
constexpr int SPLIT_MAX_CTAS = 8;                   // the portable cluster size

// Points per rank: ceil(N / C) rounded up to a multiple of 8, so every range starts where a bulk copy may start; the
// last rank's range is the remainder (shorter, or empty when C is larger than N needs).
__host__ __device__ inline int split_share(int N, int C) { return ((N + C - 1) / C + 7) / 8 * 8; }

struct AmisSplitPlan {
    AmisPlan a;
    int xbuf;                                       // 2 S floats: the partial costs exchanged per iteration
};
// plan_amis<DOF, 512> for a rank holding `share` points, with the 128-point staging ring (inside the sample buffer
// whenever it fits) instead of the 512-point one: the points are what has to fit.
template <int DOF>
__host__ __device__ inline AmisSplitPlan plan_amis_split(int share, int M, int I) {
    constexpr int T = AMIS_T_DENSE;
    AmisSplitPlan s;
    int off = (int)((sizeof(AmisHead<DOF, T>) + 127) / 128 * 128 / 4);
    constexpr int ring = 2 * STAGE_FLOATS;
    const bool alias = Dim<DOF>::POSE * M >= ring;
    s.a.stage = off; if (!alias) off += ring;
    s.a.pts = off; off += 16 * ((share + 1) / 2);
    s.a.smp = off; off += Dim<DOF>::POSE * M;
    if (alias) s.a.stage = s.a.smp;
    s.a.cost = off; off += M;
    s.a.logp = off; off += M;
    s.a.cpart = off; off += (T / NT) * M;
    s.xbuf = off; off += 2 * (M / I);
    s.a.total_bytes = off * 4;
    return s;
}

template <int DOF>
__device__ __forceinline__ void amis_split_body(const KArgs& a, const int ctas) {
    constexpr int T = AMIS_T_DENSE;
    EPNP_DYN_SMEM(unsigned char, smem_raw, 128);
    AmisHead<DOF, T>& sh = *reinterpret_cast<AmisHead<DOF, T>*>(smem_raw);
    float* dyn = reinterpret_cast<float*>(smem_raw);
    constexpr int PD = Dim<DOF>::POSE;
    const int M = a.p.mc_samples;
    const int share = split_share(a.N, ctas);
    const AmisSplitPlan pl = plan_amis_split<DOF>(share, M, a.p.mc_iter);
    const int rank = cluster_rank(), obj = blockIdx.x / ctas, tid = threadIdx.x;
    const int p0 = min(a.N, rank * share), p1 = min(a.N, p0 + share);
    const int st = serial_thread<T>(a);
    float* pts4 = dyn + pl.a.pts;
    PH_DECL;
    // Set-up as in amis_kernel, the loader taking this rank's range only.
    // Ordering rule 1: the fused entry point may have parked the covariance in this object's sample rows
    // (cov_stride = M * D).  Every rank reads it here, before its first cluster barrier (AMIS iteration 0), and rank 0
    // writes the sample rows only after the AMIS loop: no rank can read a row that rank 0 has overwritten.
    const int serial_warp = st >> 5;
    if ((tid >> 5) == serial_warp) {
        if (tid == st) amis_initial_fit(a, sh, obj);
    } else {
        LoaderT<CH> ld(a, sh.bar, dyn + pl.a.stage);
        ld.template load_range<T>(obj, pts4, p0, p1, serial_warp);
    }
    __syncthreads();
    // the rank's own bounding box: the sweep without the depth clamp gives the same bits as the clamped one, so which of
    // the two a rank runs cannot change a result
    point_box<T>(pts4, p1 - p0, sh.red + (T / 32) * 32, sh.box);
    const Cam cam = load_cam(a, obj);
    const float delta = __ldg(a.delta + obj);
    PH_MARK(a, PH_LOAD);
    const SplitCtx sc{dyn + pl.xbuf, rank, ctas, (p1 - p0 + 1) >> 1};
    amis_loop<DOF, T, true>(a, sh, pts4, dyn + pl.a.smp, dyn + pl.a.cost, dyn + pl.a.logp, dyn + pl.a.cpart, cam, delta, obj, sc);
#ifdef EPNP_SPLIT_AUDIT
    cluster_sync();                         // every rank's state is final
    for (int m = tid; m < M; m += T) {
        const float* own[3] = {dyn + pl.a.cost + m, dyn + pl.a.logp + m, dyn + pl.a.smp + m * PD};
        for (int k = 0; k < 2 + PD; ++k) {
            const float* x = k < 2 ? own[k] : own[2] + (k - 2);
            if (__float_as_uint(dsmem_ld(x, 0)) != __float_as_uint(*x)) SPLIT_AUDIT_MISMATCH();
        }
    }
#endif
    if (rank == 0) {
        block_copy<T>(a.pose_samples + (size_t)obj * M * PD, dyn + pl.a.smp, M * PD);
        SPLIT_AUDIT_STORES(tid == 0 ? M * PD : 0);
    }
    // Ordering rule 2: a CTA's shared memory disappears when it exits; this barrier keeps every CTA of the cluster alive
    // until no rank can still read its partial costs of the last iteration.
    cluster_sync();
}

template <int DOF>
__global__ void __launch_bounds__(AMIS_T_DENSE, 1) amis_split_kernel(const KArgs a, const int ctas) {
    amis_split_body<DOF>(a, ctas);
}

// amis_split_kernel with the seed read from device memory at entry (as amis_seedptr_kernel).
struct SeededKArgs {
    KArgs k;
    const uint64_t* seed;
};

template <int DOF>
__global__ void __launch_bounds__(AMIS_T_DENSE, 1) amis_split_seedptr_kernel(const SeededKArgs sa, const int ctas) {
    KArgs s = sa.k;
    s.seed = *sa.seed;
    amis_split_body<DOF>(s, ctas);
}

}  // namespace
