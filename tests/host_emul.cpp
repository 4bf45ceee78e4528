// host_emul.cpp -- TEST-ONLY serial driver around epro-pnp_b200/csrc/pnp_math.cuh compiled with g++.
// It lets the CPU test-suite (-m "not gpu") exercise the exact scalar code the sm_90a kernels inline
// (per-point math, LM state machine, small Cholesky algebra, proposal draw/density, refit formulas)
// against the golden vectors, without a GPU.  It is NOT a product path and is not shipped in the
// library: the library has no CPU fallback.  The loops here mirror pnp_kernels.cu's control flow with
// the parallel reductions replaced by plain sums.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../epro-pnp_b200/csrc/pnp_math.cuh"

using namespace pnp;

namespace {

Cam make_cam(const float* cam, const float* lb, const float* ub, int b, float z_min) {
    Cam c;
    for (int i = 0; i < 9; ++i) c.k[i] = cam[b * 9 + i];
    c.z_min = z_min;
    c.bounded = (lb && ub) ? 1 : 0;
    if (c.bounded) { c.lbx = lb[2 * b]; c.lby = lb[2 * b + 1]; c.ubx = ub[2 * b]; c.uby = ub[2 * b + 1]; }
    else { c.lbx = c.lby = -INFINITY; c.ubx = c.uby = INFINITY; }
    return c;
}

template <int DOF>
void eval_ne(const float* x3d, const float* x2d, const float* w2d, int N, const float* pose, const Cam& cam,
             float delta, float heps, bool clip, float* ev) {
    float R[9];
    pose_to_rot<DOF>(pose, R);
    float acc[32];
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int n = 0; n < N; ++n) {
        if (clip) point_normal_eq<DOF, true>(R, pose, cam, delta, heps, x3d[3 * n], x3d[3 * n + 1], x3d[3 * n + 2],
                                              x2d[2 * n], x2d[2 * n + 1], w2d[2 * n], w2d[2 * n + 1], acc);
        else point_normal_eq<DOF, false>(R, pose, cam, delta, heps, x3d[3 * n], x3d[3 * n + 1], x3d[3 * n + 2],
                                          x2d[2 * n], x2d[2 * n + 1], w2d[2 * n], w2d[2 * n + 1], acc);
    }
    for (int i = 0; i < Dim<DOF>::NV; ++i) ev[i] = acc[i];
}

template <int DOF>
float pose_cost_host(const float* x3d, const float* x2d, const float* w2d, int N, const float* pose, const Cam& cam,
                     float delta) {
    float R[9], P[12];
    pose_to_rot<DOF>(pose, R);
    make_proj(cam.k, R, pose, P);
    const float half_d2 = 0.5f * delta * delta;
    float c = 0.f;
    for (int n = 0; n < N; ++n) {
        if (cam.bounded)
            c += point_cost<true>(P, cam, delta, half_d2, x3d[3 * n], x3d[3 * n + 1], x3d[3 * n + 2], x2d[2 * n],
                                  x2d[2 * n + 1], w2d[2 * n], w2d[2 * n + 1], ExactRcp(), ExactSqrt());
        else
            c += point_cost<false>(P, cam, delta, half_d2, x3d[3 * n], x3d[3 * n + 1], x3d[3 * n + 2], x2d[2 * n],
                                   x2d[2 * n + 1], w2d[2 * n], w2d[2 * n + 1], ExactRcp(), ExactSqrt());
    }
    return c;
}

// The row-packed (two-lane) normal equations of the LM kernel: the same template, evaluated with the scalar host
// fall-backs of pnp::V2.
template <int DOF>
void eval_ne_rows(const float* x3d, const float* x2d, const float* w2d, int N, const float* pose, const Cam& cam,
                  float delta, float heps, bool clip, float* ev) {
    constexpr int NP = Dim<DOF>::NA + DOF;
    float R[9];
    pose_to_rot<DOF>(pose, R);
    V2 acc2[NP];
    for (int i = 0; i < NP; ++i) acc2[i] = v2splat(0.f);
    const V2 kuv[3] = {v2(cam.k[0], cam.k[3]), v2(cam.k[1], cam.k[4]), v2(cam.k[2], cam.k[5])};
    float cost = 0.f;
    for (int n = 0; n < N; ++n) {
        if (clip) point_normal_eq_rows<DOF, true>(R, pose, cam, kuv, delta, heps, x3d[3 * n], x3d[3 * n + 1],
                                                   x3d[3 * n + 2], -x2d[2 * n], -x2d[2 * n + 1], w2d[2 * n],
                                                   w2d[2 * n + 1], acc2, cost);
        else point_normal_eq_rows<DOF, false>(R, pose, cam, kuv, delta, heps, x3d[3 * n], x3d[3 * n + 1],
                                               x3d[3 * n + 2], -x2d[2 * n], -x2d[2 * n + 1], w2d[2 * n],
                                               w2d[2 * n + 1], acc2, cost);
    }
    for (int i = 0; i < NP; ++i) ev[i] = acc2[i].x + acc2[i].y;
    ev[NP] = cost;
}

template <int DOF>
void lm_object(const float* x3d, const float* x2d, const float* w2d, int N, const Cam& cam, float delta,
               const float* pose_init, const EpnpParams& p, float* pose_opt, float* cov, float* cost,
               float* pose_plus, float* cost_init) {
    constexpr int PD = Dim<DOF>::POSE;
    LMState<DOF> s;
    float ev[32];
    for (int i = 0; i < PD; ++i) s.pose[i] = pose_init[i];
    s.radius = p.initial_radius;
    s.shrink = 2.0f;
    if (!p.fast_mode) {
        eval_ne<DOF>(x3d, x2d, w2d, N, s.pose, cam, delta, p.huber_eps, true, ev);
        lm_adopt<DOF>(s, ev);
        if (cost_init) *cost_init = s.cost;
        if (p.lm_iter > 0) lm_propose<DOF>(s, p);
        for (int it = 0; it < p.lm_iter; ++it) {
            eval_ne<DOF>(x3d, x2d, w2d, N, s.pose_new, cam, delta, p.huber_eps, true, ev);
            lm_update<DOF>(s, ev, p);
            if (it + 1 < p.lm_iter) lm_propose<DOF>(s, p);
        }
    } else {
        for (int it = 0; it < p.lm_iter; ++it) {
            eval_ne<DOF>(x3d, x2d, w2d, N, s.pose, cam, delta, p.huber_eps, false, ev);
            lm_adopt<DOF>(s, ev);
            if (it == 0 && cost_init) *cost_init = s.cost;
            gn_advance<DOF>(s.pose, ev, p.eps, s.pose);
        }
    }
    for (int i = 0; i < PD; ++i) pose_opt[i] = s.pose[i];
    if (cost) *cost = s.cost;
    if (cov) pose_covariance<DOF>(s.a, p.eps, cov);
    if (pose_plus) {
        eval_ne<DOF>(x3d, x2d, w2d, N, s.pose, cam, delta, p.huber_eps, true, ev);
        gn_advance<DOF>(s.pose, ev, p.eps, pose_plus);
    }
}

void amis_object6(const float* x3d, const float* x2d, const float* w2d, int N, const Cam& cam, float delta,
                  const float* pose_opt, const float* cov, const float* n3, const float* c2, const float* n4,
                  uint64_t seed, uint32_t obj, const EpnpParams& p, float* samples, float* logw, float* props) {
    const int M = p.mc_samples, I = p.mc_iter, S = M / I;
    std::vector<Proposal6> prop(I);
    std::vector<float> cst(M), logp((size_t)I * M), lw(M);
    initial_fit6(pose_opt, cov, p.acg_dispersion, prop[0]);
    for (int i = 0; i < I; ++i) {
        for (int s = 0; s < S; ++s) {
            const int m = i * S + s;
            float a3[3], a4[4], chi2;
            if (n3) { memcpy(a3, n3 + 3 * m, 12); chi2 = c2[m]; memcpy(a4, n4 + 4 * m, 16); }
            else draw_base_noise(seed, obj, (uint32_t)m, a3, chi2, a4);
            float* q = samples + 7 * m;
            proposal_draw6(prop[i], a3, chi2, a4, q);
            cst[m] = pose_cost_host<6>(x3d, x2d, w2d, N, q, cam, delta);
            for (int j = 0; j <= i; ++j) logp[(size_t)j * M + m] = proposal_logpdf6(prop[j], q);
        }
        for (int m = 0; m < i * S; ++m) logp[(size_t)i * M + m] = proposal_logpdf6(prop[i], samples + 7 * m);
        const int n = (i + 1) * S;
        const float log_cnt = logf((float)(i + 1));
        float mx = -INFINITY;
        for (int m = 0; m < n; ++m) {
            float top = logp[m];
            for (int j = 1; j <= i; ++j) top = fmaxf(top, logp[(size_t)j * M + m]);
            float acc = 0.f;
            for (int j = 0; j <= i; ++j) acc += expf(logp[(size_t)j * M + m] - top);
            lw[m] = -cst[m] - ((top + logf(acc)) - log_cnt);
            mx = fmaxf(mx, lw[m]);
        }
        if (i == I - 1) { for (int m = 0; m < M; ++m) logw[m] = lw[m]; break; }
        // pass B: e = exp(lw - max); sum e, sum e t, ACG iteration 1 (Lambda_0 = I)
        float accB[15];
        for (int r = 0; r < 15; ++r) accB[r] = 0.f;
        for (int m = 0; m < n; ++m) {
            const float e = expf(lw[m] - mx);
            lw[m] = e;
            const float* s7 = samples + 7 * m;
            accB[0] += e;
            for (int k = 0; k < 3; ++k) accB[1 + k] = fmaf(e, s7[k], accB[1 + k]);
            const float* q = s7 + 3;
            const float mq = fmaxf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3], p.amis_eps);
            const float wm = e / mq;
            accB[4] += wm;
            int idx = 5;
            for (int r = 0; r < 4; ++r)
                for (int c = r; c < 4; ++c) { accB[idx] = fmaf(wm * q[r], q[c], accB[idx]); ++idx; }
        }
        const float inv_sum = 1.0f / accB[0];
        float mean[3] = {accB[1] * inv_sum, accB[2] * inv_sum, accB[3] * inv_sum};
        float lam10[10], tc[6], lam_inv[16];
        {
            const float inv0 = 1.0f / accB[4];
            for (int r = 0; r < 10; ++r) lam10[r] = accB[5 + r] * inv0;
            lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
        }
        if (p.acg_mle_iter == 0) { for (int r = 0; r < 10; ++r) lam10[r] = 0.f; lam10[0] = lam10[4] = lam10[7] = lam10[9] = 1.f; }
        // pass C: covariance about the mean (+ ACG iteration 2)
        {
            const bool more = p.acg_mle_iter >= 2;
            if (more) acg_scatter_inverse(lam10, lam_inv);
            float acc[17];
            for (int r = 0; r < 17; ++r) acc[r] = 0.f;
            for (int m = 0; m < n; ++m) {
                const float w = lw[m] * inv_sum;
                lw[m] = w;
                const float* s7 = samples + 7 * m;
                const float d0 = s7[0] - mean[0], d1 = s7[1] - mean[1], d2 = s7[2] - mean[2];
                acc[11] = fmaf(w * d0, d0, acc[11]); acc[12] = fmaf(w * d0, d1, acc[12]); acc[13] = fmaf(w * d0, d2, acc[13]);
                acc[14] = fmaf(w * d1, d1, acc[14]); acc[15] = fmaf(w * d1, d2, acc[15]); acc[16] = fmaf(w * d2, d2, acc[16]);
                if (more) {
                    const float* q = s7 + 3;
                    const float wm = w / fmaxf(quad4(lam_inv, q), p.amis_eps);
                    acc[0] += wm;
                    int idx = 1;
                    for (int r = 0; r < 4; ++r)
                        for (int c = r; c < 4; ++c) { acc[idx] = fmaf(wm * q[r], q[c], acc[idx]); ++idx; }
                }
            }
            for (int r = 0; r < 6; ++r) tc[r] = acc[11 + r];
            if (more) {
                const float inv0 = 1.0f / acc[0];
                for (int r = 0; r < 10; ++r) lam10[r] = acc[1 + r] * inv0;
                lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
            }
        }
        for (int itr = 2; itr < p.acg_mle_iter; ++itr) {
            acg_scatter_inverse(lam10, lam_inv);
            float acc[11];
            for (int r = 0; r < 11; ++r) acc[r] = 0.f;
            for (int m = 0; m < n; ++m) {
                const float* q = samples + 7 * m + 3;
                const float wm = lw[m] / fmaxf(quad4(lam_inv, q), p.amis_eps);
                acc[0] += wm;
                int idx = 1;
                for (int r = 0; r < 4; ++r)
                    for (int c = r; c < 4; ++c) { acc[idx] = fmaf(wm * q[r], q[c], acc[idx]); ++idx; }
            }
            const float inv0 = 1.0f / acc[0];
            for (int r = 0; r < 10; ++r) lam10[r] = acc[1 + r] * inv0;
            lam10[0] += p.amis_eps; lam10[4] += p.amis_eps; lam10[7] += p.amis_eps; lam10[9] += p.amis_eps;
        }
        refit_finish6(mean, tc, lam10, p.acg_dispersion, prop[i + 1]);
    }
    if (props) {
        for (int i = 0; i < I; ++i) {
            float* o = props + i * 19;
            for (int r = 0; r < 3; ++r) o[r] = prop[i].mu[r];
            for (int r = 0; r < 6; ++r) o[3 + r] = prop[i].lt[r];
            for (int r = 0; r < 10; ++r) o[9 + r] = prop[i].lr[r];
        }
    }
}

void amis_object4(const float* x3d, const float* x2d, const float* w2d, int N, const Cam& cam, float delta,
                  const float* pose_opt, const float* cov, const float* n3, const float* c2, const float* yaw,
                  uint64_t seed, uint32_t obj, const EpnpParams& p, float* samples, float* logw, float* props) {
    const int M = p.mc_samples, I = p.mc_iter, S = M / I;
    std::vector<Proposal4> prop(I);
    std::vector<float> cst(M), logp((size_t)I * M), lw(M);
    initial_fit4(pose_opt, cov, p.amis_eps, prop[0]);
    for (int i = 0; i < I; ++i) {
        for (int s = 0; s < S; ++s) {
            const int m = i * S + s;
            float a3[3], chi2;
            float* q = samples + 4 * m;
            if (n3) { memcpy(a3, n3 + 3 * m, 12); chi2 = c2[m]; q[3] = yaw[m]; }
            else { draw_base_noise_t(seed, obj, (uint32_t)m, a3, chi2); q[3] = draw_yaw(seed, obj, (uint32_t)m, s, S, prop[i].mode, prop[i].kappa); }
            draw_translation(prop[i].mu, prop[i].lt, a3, chi2, q);
            cst[m] = pose_cost_host<4>(x3d, x2d, w2d, N, q, cam, delta);
            for (int j = 0; j <= i; ++j) logp[(size_t)j * M + m] = proposal_logpdf4(prop[j], q);
        }
        for (int m = 0; m < i * S; ++m) logp[(size_t)i * M + m] = proposal_logpdf4(prop[i], samples + 4 * m);
        const int n = (i + 1) * S;
        const float log_cnt = logf((float)(i + 1));
        float mx = -INFINITY;
        for (int m = 0; m < n; ++m) {
            float top = logp[m];
            for (int j = 1; j <= i; ++j) top = fmaxf(top, logp[(size_t)j * M + m]);
            float acc = 0.f;
            for (int j = 0; j <= i; ++j) acc += expf(logp[(size_t)j * M + m] - top);
            lw[m] = -cst[m] - ((top + logf(acc)) - log_cnt);
            mx = fmaxf(mx, lw[m]);
        }
        if (i == I - 1) { for (int m = 0; m < M; ++m) logw[m] = lw[m]; break; }
        float accB[6] = {0, 0, 0, 0, 0, 0};
        for (int m = 0; m < n; ++m) {
            const float e = expf(lw[m] - mx);
            lw[m] = e;
            const float* s4 = samples + 4 * m;
            accB[0] += e;
            for (int k = 0; k < 3; ++k) accB[1 + k] = fmaf(e, s4[k], accB[1 + k]);
            accB[4] = fmaf(e, sinf(s4[3]), accB[4]); accB[5] = fmaf(e, cosf(s4[3]), accB[5]);
        }
        const float inv_sum = 1.0f / accB[0];
        const float mean[3] = {accB[1] * inv_sum, accB[2] * inv_sum, accB[3] * inv_sum};
        float tc[6] = {0, 0, 0, 0, 0, 0};
        for (int m = 0; m < n; ++m) {
            const float w = lw[m] * inv_sum;
            const float* s4 = samples + 4 * m;
            const float d0 = s4[0] - mean[0], d1 = s4[1] - mean[1], d2 = s4[2] - mean[2];
            tc[0] = fmaf(w * d0, d0, tc[0]); tc[1] = fmaf(w * d0, d1, tc[1]); tc[2] = fmaf(w * d0, d2, tc[2]);
            tc[3] = fmaf(w * d1, d1, tc[3]); tc[4] = fmaf(w * d1, d2, tc[4]); tc[5] = fmaf(w * d2, d2, tc[5]);
        }
        refit_finish4(mean, tc, accB[4] * inv_sum, accB[5] * inv_sum, p.amis_eps, prop[i + 1]);
    }
    if (props) {
        for (int i = 0; i < I; ++i) {
            float* o = props + i * 19;
            for (int r = 0; r < 19; ++r) o[r] = 0.f;
            for (int r = 0; r < 3; ++r) o[r] = prop[i].mu[r];
            for (int r = 0; r < 6; ++r) o[3 + r] = prop[i].lt[r];
            o[9] = prop[i].mode; o[10] = prop[i].kappa;
        }
    }
}

}  // namespace

extern "C" {

// normal equations (NV floats per object) at one pose per object
int emul_normal_eq(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb,
                   const float* ub, const float* delta, const float* pose, float* out, int clip, int B, int N,
                   int dof, float z_min, float heps) {
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, z_min);
        const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
        if (dof == 6) eval_ne<6>(p3, p2, pw, N, pose + b * 7, c, delta[b], heps, clip != 0, out + b * Dim<6>::NV);
        else eval_ne<4>(p3, p2, pw, N, pose + b * 4, c, delta[b], heps, clip != 0, out + b * Dim<4>::NV);
    }
    return 0;
}

int emul_residual_jac(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb,
                      const float* ub, const float* delta, const float* pose, float* res, float* jac, float* cost,
                      int clip, int B, int N, int dof, float z_min, float heps) {
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, z_min);
        float R[9];
        const int PD = dof == 6 ? 7 : 4;
        if (dof == 6) pose_to_rot<6>(pose + b * PD, R); else pose_to_rot<4>(pose + b * PD, R);
        float cs = 0.f;
        for (int n = 0; n < N; ++n) {
            const size_t g = (size_t)b * N + n;
            if (dof == 6)
                cs += point_residual_jac<6>(R, pose + b * PD, c, delta[b], heps, clip != 0, x3d[g * 3], x3d[g * 3 + 1],
                                            x3d[g * 3 + 2], x2d[g * 2], x2d[g * 2 + 1], w2d[g * 2], w2d[g * 2 + 1],
                                            res + g * 2, jac + g * 12);
            else
                cs += point_residual_jac<4>(R, pose + b * PD, c, delta[b], heps, clip != 0, x3d[g * 3], x3d[g * 3 + 1],
                                            x3d[g * 3 + 2], x2d[g * 2], x2d[g * 2 + 1], w2d[g * 2], w2d[g * 2 + 1],
                                            res + g * 2, jac + g * 8);
        }
        cost[b] = cs;
    }
    return 0;
}

int emul_cost(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb, const float* ub,
              const float* delta, const float* poses, float* cost, int S, int B, int N, int dof, float z_min) {
    const int PD = dof == 6 ? 7 : 4;
    for (int s = 0; s < S; ++s)
        for (int b = 0; b < B; ++b) {
            const Cam c = make_cam(cam, lb, ub, b, z_min);
            const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
            const float* pose = poses + ((size_t)s * B + b) * PD;
            cost[(size_t)s * B + b] = dof == 6 ? pose_cost_host<6>(p3, p2, pw, N, pose, c, delta[b])
                                               : pose_cost_host<4>(p3, p2, pw, N, pose, c, delta[b]);
        }
    return 0;
}

int emul_normal_eq_rows(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb,
                        const float* ub, const float* delta, const float* pose, float* out, int clip, int B, int N,
                        int dof, float z_min, float heps) {
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, z_min);
        const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
        if (dof == 6) eval_ne_rows<6>(p3, p2, pw, N, pose + b * 7, c, delta[b], heps, clip != 0, out + b * Dim<6>::NV);
        else eval_ne_rows<4>(p3, p2, pw, N, pose + b * 4, c, delta[b], heps, clip != 0, out + b * Dim<4>::NV);
    }
    return 0;
}


int emul_lm(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb, const float* ub,
            const float* delta, const float* pose_init, float* pose_opt, float* cov, float* cost, float* pose_plus,
            float* cost_init, int B, int N, const EpnpParams* p) {
    const int dof = p->dof, PD = dof == 6 ? 7 : 4;
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, p->z_min);
        const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
        if (dof == 6)
            lm_object<6>(p3, p2, pw, N, c, delta[b], pose_init + b * PD, *p, pose_opt + b * PD, cov ? cov + b * 36 : nullptr,
                         cost ? cost + b : nullptr, pose_plus ? pose_plus + b * PD : nullptr, cost_init ? cost_init + b : nullptr);
        else
            lm_object<4>(p3, p2, pw, N, c, delta[b], pose_init + b * PD, *p, pose_opt + b * PD, cov ? cov + b * 16 : nullptr,
                         cost ? cost + b : nullptr, pose_plus ? pose_plus + b * PD : nullptr, cost_init ? cost_init + b : nullptr);
    }
    return 0;
}

// noise object-major: n3 (B,M,3), c2 (B,M), n4 (B,M,4) or all NULL (Philox)
int emul_amis6(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb, const float* ub,
               const float* delta, const float* pose_opt, const float* cov, const float* n3, const float* c2,
               const float* n4, uint64_t seed, uint32_t obj_offset, float* samples, float* logw, float* props, int B,
               int N, const EpnpParams* p) {
    const int M = p->mc_samples, I = p->mc_iter;
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, p->z_min);
        const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
        amis_object6(p3, p2, pw, N, c, delta[b], pose_opt + b * 7, cov + b * 36, n3 ? n3 + (size_t)b * M * 3 : nullptr,
                     c2 ? c2 + (size_t)b * M : nullptr, n4 ? n4 + (size_t)b * M * 4 : nullptr, seed, obj_offset + b, *p,
                     samples + (size_t)b * M * 7, logw + (size_t)b * M, props ? props + (size_t)b * I * 19 : nullptr);
    }
    return 0;
}

// 4DoF: n3 (B,M,3), c2 (B,M), yaw draws (B,M) or all NULL (Philox + Best-Fisher)
int emul_amis4(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb, const float* ub,
               const float* delta, const float* pose_opt, const float* cov, const float* n3, const float* c2,
               const float* yaw, uint64_t seed, uint32_t obj_offset, float* samples, float* logw, float* props, int B,
               int N, const EpnpParams* p) {
    const int M = p->mc_samples, I = p->mc_iter;
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, p->z_min);
        const float *p3 = x3d + (size_t)b * N * 3, *p2 = x2d + (size_t)b * N * 2, *pw = w2d + (size_t)b * N * 2;
        amis_object4(p3, p2, pw, N, c, delta[b], pose_opt + b * 4, cov + b * 16, n3 ? n3 + (size_t)b * M * 3 : nullptr,
                     c2 ? c2 + (size_t)b * M : nullptr, yaw ? yaw + (size_t)b * M : nullptr, seed, obj_offset + b, *p,
                     samples + (size_t)b * M * 4, logw + (size_t)b * M, props ? props + (size_t)b * I * 19 : nullptr);
    }
    return 0;
}

// reverse mode of the cost: poses (B, P, D), grads (B, P) -> gx3d (B,N,3), gx2d (B,N,2), gw2d (B,N,2), gdelta (B)
int emul_cost_backward(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* lb,
                       const float* ub, const float* delta, const float* poses, const float* grads, float* gx3d,
                       float* gx2d, float* gw2d, float* gdelta, int P, int B, int N, int dof, float z_min) {
    const int PD = dof == 6 ? 7 : 4;
    for (int b = 0; b < B; ++b) {
        const Cam c = make_cam(cam, lb, ub, b, z_min);
        float gd = 0.f;
        for (int n = 0; n < N; ++n) {
            const size_t q = (size_t)b * N + n;
            float g[7] = {0, 0, 0, 0, 0, 0, 0};
            for (int p = 0; p < P; ++p) {
                const float* pose = poses + ((size_t)b * P + p) * PD;
                float R[9], Pj[12];
                if (dof == 6) pose_to_rot<6>(pose, R); else pose_to_rot<4>(pose, R);
                make_proj(c.k, R, pose, Pj);
                const float gj = grads[(size_t)b * P + p];
                gd += c.bounded
                    ? point_cost_backward<true>(Pj, c, delta[b], gj, x3d[q * 3], x3d[q * 3 + 1], x3d[q * 3 + 2], x2d[q * 2],
                                                x2d[q * 2 + 1], w2d[q * 2], w2d[q * 2 + 1], g, ExactRcp())
                    : point_cost_backward<false>(Pj, c, delta[b], gj, x3d[q * 3], x3d[q * 3 + 1], x3d[q * 3 + 2], x2d[q * 2],
                                                 x2d[q * 2 + 1], w2d[q * 2], w2d[q * 2 + 1], g, ExactRcp());
            }
            gx3d[q * 3] = g[0]; gx3d[q * 3 + 1] = g[1]; gx3d[q * 3 + 2] = g[2];
            gx2d[q * 2] = g[3]; gx2d[q * 2 + 1] = g[4]; gw2d[q * 2] = g[5]; gw2d[q * 2 + 1] = g[6];
        }
        gdelta[b] = gd;
    }
    return 0;
}

// yaw draws of the production sampler, for statistical tests
// Tail of a proposal refit from given statistics (refit_finish6 / refit_finish4): out[0..3) mu, [3..9) L_t, then
// dof 6: [9..19) L_r; dof 4: [9] mode, [10] kappa.  Exercises the not-positive-definite fallbacks of the device code.
int emul_refit_finish(int dof, const float* mean, const float* tc6, const float* lam10_or_sincos, float* out) {
    if (dof == 6) {
        Proposal6 p;
        refit_finish6(mean, tc6, lam10_or_sincos, 1e-3f, p);
        for (int i = 0; i < 3; ++i) out[i] = p.mu[i];
        for (int i = 0; i < 6; ++i) out[3 + i] = p.lt[i];
        for (int i = 0; i < 10; ++i) out[9 + i] = p.lr[i];
    } else {
        Proposal4 p;
        refit_finish4(mean, tc6, lam10_or_sincos[0], lam10_or_sincos[1], 1e-5f, p);
        for (int i = 0; i < 3; ++i) out[i] = p.mu[i];
        for (int i = 0; i < 6; ++i) out[3 + i] = p.lt[i];
        out[9] = p.mode; out[10] = p.kappa;
    }
    return 0;
}

int emul_yaw(uint64_t seed, uint32_t obj, int count, int S, float mode, float kappa, float* out) {
    for (int m = 0; m < count; ++m) out[m] = draw_yaw(seed, obj, (uint32_t)m, m % S, S, mode, kappa);
    return 0;
}

// base noise of the production RNG, for statistical tests: out (count, 8) = n3, chi2, n4
int emul_base_noise(uint64_t seed, uint32_t obj, int count, float* out) {
    for (int m = 0; m < count; ++m) draw_base_noise(seed, obj, (uint32_t)m, out + 8 * m, out[8 * m + 3], out + 8 * m + 4);
    return 0;
}

}  // extern "C"
