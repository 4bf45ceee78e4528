// epnp_host.cpp -- TEST-ONLY serial driver around epro-pnp_b200/csrc/pnp_epnp.cuh compiled with g++ (the sibling of
// host_emul.cpp for the EPnP initialiser).  It runs the selection rule and the per-object EPnP math the kernel uses,
// with the kernel's parallel parts (order statistics, compaction, per-point sums) replaced by a sort and plain loops,
// so the CPU suite can check them against np.quantile and cv2.  Not a product path: the library has no CPU fallback.
#include <algorithm>
#include <cmath>
#include <vector>

#include "../epro-pnp_b200/csrc/pnp_epnp.cuh"

using namespace pnp::epnp;

extern "C" {

// mask[i] = conf_i >= np.quantile(conf, q) for one row; returns the number kept, or -1 when a confidence is NaN
int epnp_host_select(const float* w2d, int N, float q, unsigned char* mask) {
    std::vector<uint32_t> keys(N);
    std::vector<float> conf(N);
    for (int i = 0; i < N; ++i) {
        conf[i] = (w2d[2 * i] + w2d[2 * i + 1]) * 0.5f;
        if (conf[i] != conf[i]) return -1;
        keys[i] = conf_key(conf[i]);
    }
    std::sort(keys.begin(), keys.end());
    const QuantileRank r = quantile_rank(N, q);
    const float thr = quantile_threshold(key_conf(keys[r.k]), key_conf(keys[r.k1]), r.g);
    int n = 0;
    for (int i = 0; i < N; ++i) {
        mask[i] = conf[i] >= thr;
        n += mask[i];
    }
    return n;
}

int epnp_host_min_selected(int N, float q) { return min_selected(N, q); }

// EPnP on the points with mask[i] != 0 (all when mask is NULL): pose = [x y z w i j k]; err[3] = the candidates' mean
// pixel reprojection errors
void epnp_host_solve(const float* x3d, const float* x2d, const float* K, const unsigned char* mask, int N, float* pose,
                     double* err) {
    std::vector<int> idx;
    for (int i = 0; i < N; ++i)
        if (!mask || mask[i]) idx.push_back(i);
    const int n = (int)idx.size();
    const Intrinsics in = intrinsics(K);
    double c0[3] = {0.0, 0.0, 0.0}, S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i : idx)
        for (int c = 0; c < 3; ++c) c0[c] += x3d[3 * i + c];
    for (int c = 0; c < 3; ++c) c0[c] /= n;
    for (int i : idx) {
        const double d[3] = {x3d[3 * i] - c0[0], x3d[3 * i + 1] - c0[1], x3d[3 * i + 2] - c0[2]};
        S[0] += d[0] * d[0]; S[1] += d[0] * d[1]; S[2] += d[0] * d[2];
        S[3] += d[1] * d[1]; S[4] += d[1] * d[2]; S[5] += d[2] * d[2];
    }
    Control cp;
    control_points(c0, S, n, cp);
    double acc[NSUM];
    for (int k = 0; k < NSUM; ++k) acc[k] = 0.0;
    for (int i : idx) accumulate_point(cp, in, x3d[3 * i], x3d[3 * i + 1], x3d[3 * i + 2], x2d[2 * i], x2d[2 * i + 1], acc);
    double al0[4];
    barycentric(cp, x3d[3 * idx[0]], x3d[3 * idx[0] + 1], x3d[3 * idx[0] + 2], al0);
    Candidate cand[3];
    solve_candidates(acc, cp, in, al0, n, cand);
    double e[3] = {0.0, 0.0, 0.0};
    for (int c = 0; c < 3; ++c)
        for (int i : idx) e[c] += reproj_error(cand[c], in, x3d[3 * i], x3d[3 * i + 1], x3d[3 * i + 2], x2d[2 * i], x2d[2 * i + 1]);
    write_pose(cand[pick_candidate(e)], pose);
    for (int c = 0; c < 3; ++c) err[c] = e[c] / n;
}

}  // extern "C"
