// pnp_epnp.cuh -- per-object math of the EPnP initialiser (epnp_epnp_init_f32): the confidence-quantile point selection
// and EPnP (Lepetit, Moreno-Noguer & Fua, "EPnP: an accurate O(n) solution to the PnP problem", IJCV 2009) in fp64.
// It replaces the per-object host loop of the reference's 6DoF test (EPro-PnP-6DoF/lib/test.py:178-194): conf =
// w2d.mean(-1), keep conf >= np.quantile(conf, q), cv2.solvePnP(..., flags=SOLVEPNP_EPNP), Rodrigues -> quaternion.
//
// Like pnp_math.cuh, everything is __host__ __device__ and allocation-free, so tests/epnp_host.cpp builds the same code
// with g++.  The kernels (pnp_kernels.cu, epnp_init_kernel and epnp_init_split_kernel) supply the parallel parts: the
// order statistics of the confidences, the compaction of the selected points and the per-point sums; the serial parts
// are here.  The out-of-line functions (EPNP_HD_COLD) take a SITE tag: ptxas fits an out-of-line function to all of
// its callers, so each kernel instantiates its own copies (epnp_init_kernel SITE 0, epnp_init_split_kernel SITE 1) and
// a new caller cannot change an existing kernel's code.
//
// Conventions, fixed by experiment against cv2 (OpenCV 4.13), which the reference calls:
//   * pixel coordinates with fu = K[0][0], fv = K[1][1], uc = K[0][2], vc = K[1][2]: with fu != fv the normalised-
//     coordinate formulation differs from cv2 by ~2e-5 rad, the pixel one agrees to fp64 rounding; K[0][1] is not read;
//   * control points: the centroid, and the centroid + sqrt(lambda_i / n) e_i along the principal axes of the points;
//   * every symmetric eigenproblem is solved as an SVD by cyclic one-sided (Hestenes) Jacobi sweeps, whose rotations
//     fix the sign of each axis.  The EPnP result depends on those signs at the 1e-3 level on noisy data (the distance
//     constraints do not, the least-squares fit of the null space does), so the sign convention is part of the parity;
//   * the three beta approximations (N = 1, 2, 3 in the paper), each refined by 5 Gauss-Newton steps; the camera-frame
//     control points are negated when the FIRST selected point comes out behind the camera;
//   * R, t from the orthogonal Procrustes fit as cv2 forms it: R = U V^T of the cross-covariance H, and when that is a
//     reflection (det H < 0) its third row negated -- not the optimal rotation, but what cv2 returns, and on noisy or
//     outlier-laden objects it decides the winning candidate.  Computed in Horn's quaternion form, which yields the
//     quaternion directly: R = Horn(H) for det H >= 0, else diag(-1, -1, 1) Horn(-H), since U V^T = -Horn(-H) then;
//   * the candidate with the smallest mean pixel reprojection error wins (ties go to the earlier one).
// The camera's bounds (lb / ub) and z_min play no part: cv2's EPnP has neither.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define EPNP_HD __host__ __device__ __forceinline__
#define EPNP_HD_COLD __host__ __device__ __noinline__
#else
#define EPNP_HD inline
#define EPNP_HD_COLD inline
#endif

namespace pnp {
namespace epnp {

// ------------------------------------------------------------------------------------------------
// Point selection: conf_i = (w2d[i, 0] + w2d[i, 1]) / 2 in fp32, kept when conf_i >= np.quantile(conf, q).

// Order-preserving integer image of an fp32 key (-0 folded onto +0, as a comparison sees them).  NaN is handled apart.
EPNP_HD uint32_t conf_key(float c) {
    uint32_t u;
    memcpy(&u, &c, 4);
    if (u == 0x80000000u) u = 0u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
EPNP_HD float key_conf(uint32_t k) {
    const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float c;
    memcpy(&c, &u, 4);
    return c;
}

// NumPy 2.x np.quantile(x, q) (method 'linear') of a float32 row works in float32: h = (N - 1) q, k = floor(h),
// g = h - k, then interpolates between the order statistics s[k] and s[min(k + 1, N - 1)].
struct QuantileRank { int k, k1; float g; };
EPNP_HD QuantileRank quantile_rank(int N, float q) {
    const float h = (float)(N - 1) * q;
    const float fk = floorf(h);
    QuantileRank r;
    r.k = (int)fk;
    r.k1 = r.k + 1 < N - 1 ? r.k + 1 : N - 1;
    r.g = h - fk;
    return r;
}
// fp32 product, correctly rounded whatever the compiler's contraction setting: the fp64 product of two floats is exact
EPNP_HD float mul_rn(float a, float b) { return (float)((double)a * (double)b); }
// threshold from a = s[k], b = s[k1] (NumPy's _lerp: from the nearer end, every operation rounded to fp32)
EPNP_HD float quantile_threshold(float a, float b, float g) {
    const float d = b - a;
    return g >= 0.5f ? b - mul_rn(d, 1.0f - g) : a + mul_rn(d, g);
}
// fewest points any row of N confidences can keep at quantile q: s[k1..N-1] always pass, s[k] too when g == 0
EPNP_HD int min_selected(int N, float q) {
    const QuantileRank r = quantile_rank(N, q);
    return N - r.k - (r.g > 0.0f ? 1 : 0);
}

// ------------------------------------------------------------------------------------------------
// Small dense fp64 algebra (once per object)

EPNP_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// SVD of a symmetric n x n matrix by cyclic one-sided Jacobi sweeps over its rows: the rows are rotated pairwise until
// they are mutually orthogonal (at most max(n, 30) sweeps, so a NaN input ends too), then sorted by descending norm
// (stable) and normalised.  On return A's rows are the left singular vectors and w the singular values.  Each rotation
// is the one of angle at most pi/4 that orthogonalises the pair -- this choice is what fixes the vectors' signs.
template <int n, int SITE = 0>
EPNP_HD_COLD void jacobi_svd_rows(double (&A)[n][n], double (&w)[n]) {
    const double tol = 10.0 * 2.220446049250313e-16;
    for (int i = 0; i < n; ++i) {
        double s = 0.0;
        for (int k = 0; k < n; ++k) s += A[i][k] * A[i][k];
        w[i] = s;
    }
    const int sweeps = n > 30 ? n : 30;
    for (int it = 0; it < sweeps; ++it) {
        bool changed = false;
        for (int i = 0; i < n - 1; ++i) {
            for (int j = i + 1; j < n; ++j) {
                const double a = w[i], b = w[j];
                double p = 0.0;
                for (int k = 0; k < n; ++k) p += A[i][k] * A[j][k];
                if (fabs(p) <= tol * sqrt(a * b)) continue;
                p *= 2.0;
                const double beta = a - b, gamma = hypot(p, beta);
                double c, s;
                if (beta < 0.0) {
                    s = sqrt((gamma - beta) * 0.5 / gamma);
                    c = p / (gamma * s * 2.0);
                } else {
                    c = sqrt((gamma + beta) / (gamma * 2.0));
                    s = p / (gamma * c * 2.0);
                }
                double na = 0.0, nb = 0.0;
                for (int k = 0; k < n; ++k) {
                    const double t0 = c * A[i][k] + s * A[j][k];
                    const double t1 = -s * A[i][k] + c * A[j][k];
                    A[i][k] = t0;
                    A[j][k] = t1;
                    na += t0 * t0;
                    nb += t1 * t1;
                }
                w[i] = na;
                w[j] = nb;
                changed = true;
            }
        }
        if (!changed) break;
    }
    for (int i = 0; i < n; ++i) {
        double s = 0.0;
        for (int k = 0; k < n; ++k) s += A[i][k] * A[i][k];
        w[i] = sqrt(s);
    }
    for (int i = 0; i < n - 1; ++i) {
        int m = i;
        for (int k = i + 1; k < n; ++k)
            if (w[m] < w[k]) m = k;
        if (m != i) {
            const double t = w[i]; w[i] = w[m]; w[m] = t;
            for (int k = 0; k < n; ++k) { const double x = A[i][k]; A[i][k] = A[m][k]; A[m][k] = x; }
        }
    }
    for (int i = 0; i < n; ++i) {
        const double s = w[i] > 0.0 ? 1.0 / w[i] : 0.0;
        for (int k = 0; k < n; ++k) A[i][k] *= s;
    }
}

// Least-squares solution of the M x N system A x = b (M >= N) by Householder QR.  A and b are overwritten.  A column
// that is zero below the diagonal gives x = 0 in that component.
template <int M, int N, int SITE = 0>
EPNP_HD_COLD void lstsq(double (&A)[M][N], double (&b)[M], double (&x)[N]) {
    for (int k = 0; k < N; ++k) {
        double nrm = 0.0;
        for (int i = k; i < M; ++i) nrm += A[i][k] * A[i][k];
        nrm = sqrt(nrm);
        if (!(nrm > 0.0)) continue;
        const double alpha = A[k][k] > 0.0 ? -nrm : nrm;
        double v[M];
        for (int i = 0; i < M; ++i) v[i] = i < k ? 0.0 : A[i][k];
        v[k] -= alpha;
        double vv = 0.0;
        for (int i = k; i < M; ++i) vv += v[i] * v[i];
        if (!(vv > 0.0)) continue;
        for (int j = k + 1; j < N; ++j) {
            double s = 0.0;
            for (int i = k; i < M; ++i) s += v[i] * A[i][j];
            s = 2.0 * s / vv;
            for (int i = k; i < M; ++i) A[i][j] -= s * v[i];
        }
        double s = 0.0;
        for (int i = k; i < M; ++i) s += v[i] * b[i];
        s = 2.0 * s / vv;
        for (int i = k; i < M; ++i) b[i] -= s * v[i];
        A[k][k] = alpha;
        for (int i = k + 1; i < M; ++i) A[i][k] = 0.0;
    }
    for (int k = N - 1; k >= 0; --k) {
        double s = b[k];
        for (int j = k + 1; j < N; ++j) s -= A[k][j] * x[j];
        x[k] = A[k][k] != 0.0 ? s / A[k][k] : 0.0;
    }
}

// ------------------------------------------------------------------------------------------------
// EPnP

struct Intrinsics { double fu, fv, uc, vc; };
EPNP_HD Intrinsics intrinsics(const float* K) {
    Intrinsics c;
    c.fu = K[0]; c.fv = K[4]; c.uc = K[2]; c.vc = K[5];
    return c;
}

// World control points and the map to barycentric coordinates: alpha_{1..3} = axis_i . (p - c_0), alpha_0 = 1 - sum.
struct Control {
    double c[4][3];
    double axis[3][3];          // e_i / sqrt(lambda_i / n)
};

// c0: centroid of the n selected points; S: their centred scatter (xx xy xz yy yz zz)
template <int SITE = 0>
EPNP_HD_COLD void control_points(const double (&c0)[3], const double (&S)[6], int n, Control& cp) {
    double A[3][3] = {{S[0], S[1], S[2]}, {S[1], S[3], S[4]}, {S[2], S[4], S[5]}};
    double w[3];
    jacobi_svd_rows<3, SITE>(A, w);
    for (int j = 0; j < 3; ++j) cp.c[0][j] = c0[j];
    for (int i = 0; i < 3; ++i) {
        const double k = sqrt(w[i] / n);
        for (int j = 0; j < 3; ++j) {
            cp.c[i + 1][j] = c0[j] + k * A[i][j];
            cp.axis[i][j] = A[i][j] / k;
        }
    }
}

EPNP_HD void barycentric(const Control& cp, double x, double y, double z, double (&al)[4]) {
    const double d[3] = {x - cp.c[0][0], y - cp.c[0][1], z - cp.c[0][2]};
    al[1] = dot3(cp.axis[0], d);
    al[2] = dot3(cp.axis[1], d);
    al[3] = dot3(cp.axis[2], d);
    al[0] = 1.0 - al[1] - al[2] - al[3];
}

// Per-point sums everything after the control points needs (one pass):
//   [0, 40)   M^T M of the 2n x 12 system, factored: M^T M = sum_i (alpha alpha^T) (x) [[fu^2 0 fu du] [0 fv^2 fv dv]
//             [fu du fv dv du^2 + dv^2]] with du = uc - u, dv = vc - v; per alpha pair (j <= k): sum of alpha_j alpha_k
//             times {1, du, dv, du^2 + dv^2}
//   [40, 52)  sum_i alpha_ij (p_i - c_0)    (the Procrustes cross-covariance is linear in the camera control points)
//   [52, 56)  sum_i alpha_ij
constexpr int NSUM = 56;
EPNP_HD void accumulate_point(const Control& cp, const Intrinsics& in, double x, double y, double z, double u, double v,
                              double (&acc)[NSUM]) {
    double al[4];
    barycentric(cp, x, y, z, al);
    const double du = in.uc - u, dv = in.vc - v, dq = du * du + dv * dv;
    int p = 0;
    for (int j = 0; j < 4; ++j) {
        for (int k = j; k < 4; ++k, ++p) {
            const double aa = al[j] * al[k];
            acc[4 * p] += aa;
            acc[4 * p + 1] += aa * du;
            acc[4 * p + 2] += aa * dv;
            acc[4 * p + 3] += aa * dq;
        }
    }
    const double d[3] = {x - cp.c[0][0], y - cp.c[0][1], z - cp.c[0][2]};
    for (int j = 0; j < 4; ++j) {
        for (int c = 0; c < 3; ++c) acc[40 + 3 * j + c] += al[j] * d[c];
        acc[52 + j] += al[j];
    }
}

// One EPnP candidate: unit quaternion [w, i, j, k] (w >= 0), rotation and translation.
struct Candidate { double q[4], R[9], t[3]; };

EPNP_HD void quat_rot(const double (&q)[4], double (&R)[9]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = w * w + x * x - y * y - z * z; R[1] = 2.0 * (x * y - w * z);         R[2] = 2.0 * (x * z + w * y);
    R[3] = 2.0 * (x * y + w * z);         R[4] = w * w - x * x + y * y - z * z; R[5] = 2.0 * (y * z - w * x);
    R[6] = 2.0 * (x * z - w * y);         R[7] = 2.0 * (y * z + w * x);         R[8] = w * w - x * x - y * y + z * z;
}

// R, t from the camera-frame control points ccs: pc_i = sum_j alpha_ij ccs_j.  Horn: q maximises q^T N(S) q with
// S_ab = sum_i (p_i - c_0)_a pc_{i,b}; N is shifted by a Gershgorin bound so that its top eigenvector is its top
// singular vector.  det S < 0 (the best orthogonal fit is a reflection): q of diag(-1, -1, 1) Horn(-S), see the top.
template <int SITE = 0>
EPNP_HD_COLD void procrustes(const double (&ccs)[4][3], const double (&acc)[NSUM], int n, const double (&c0)[3], Candidate& out) {
    double S[3][3], pc0[3];
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) {
            double s = 0.0;
            for (int j = 0; j < 4; ++j) s += acc[40 + 3 * j + a] * ccs[j][b];
            S[a][b] = s;
        }
        double s = 0.0;
        for (int j = 0; j < 4; ++j) s += acc[52 + j] * ccs[j][a];
        pc0[a] = s / n;
    }
    const double det = S[0][0] * (S[1][1] * S[2][2] - S[1][2] * S[2][1]) - S[0][1] * (S[1][0] * S[2][2] - S[1][2] * S[2][0]) +
                       S[0][2] * (S[1][0] * S[2][1] - S[1][1] * S[2][0]);
    const bool reflect = det < 0.0;
    if (reflect)
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) S[a][b] = -S[a][b];
    double Nm[4][4] = {
        {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0]},
        {S[1][2] - S[2][1], S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2]},
        {S[2][0] - S[0][2], S[0][1] + S[1][0], -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1]},
        {S[0][1] - S[1][0], S[2][0] + S[0][2], S[1][2] + S[2][1], -S[0][0] - S[1][1] + S[2][2]}};
    double shift = 0.0;
    for (int i = 0; i < 4; ++i) {
        double r = 0.0;
        for (int j = 0; j < 4; ++j) r += fabs(Nm[i][j]);
        shift = r > shift ? r : shift;
    }
    for (int i = 0; i < 4; ++i) Nm[i][i] += shift;
    double w[4];
    jacobi_svd_rows<4, SITE>(Nm, w);
    double q[4] = {Nm[0][0], Nm[0][1], Nm[0][2], Nm[0][3]};
    if (reflect) {                      // (0, 0, 0, 1) * q: a half turn about z after Horn(-S)
        const double h[4] = {-q[3], -q[2], q[1], q[0]};
        for (int i = 0; i < 4; ++i) q[i] = h[i];
    }
    const double nq = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double sg = q[0] < 0.0 ? -1.0 / nq : 1.0 / nq;
    for (int i = 0; i < 4; ++i) out.q[i] = q[i] * sg;
    quat_rot(out.q, out.R);
    for (int a = 0; a < 3; ++a) out.t[a] = pc0[a] - (out.R[3 * a] * c0[0] + out.R[3 * a + 1] * c0[1] + out.R[3 * a + 2] * c0[2]);
}

// The three candidates from the per-point sums.  al_first: barycentric coordinates of the first selected point.
template <int SITE = 0>
EPNP_HD_COLD void solve_candidates(const double (&acc)[NSUM], const Control& cp, const Intrinsics& in, const double (&al_first)[4],
                                   int n, Candidate (&cand)[3]) {
    // M^T M (12 x 12), block (j, k) from the factored sums
    double A[12][12];
    {
        int p = 0;
        for (int j = 0; j < 4; ++j) {
            for (int k = j; k < 4; ++k, ++p) {
                const double s1 = acc[4 * p], su = acc[4 * p + 1], sv = acc[4 * p + 2], sq = acc[4 * p + 3];
                const double blk[3][3] = {{in.fu * in.fu * s1, 0.0, in.fu * su},
                                          {0.0, in.fv * in.fv * s1, in.fv * sv},
                                          {in.fu * su, in.fv * sv, sq}};
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) {
                        A[3 * j + r][3 * k + c] = blk[r][c];
                        A[3 * k + c][3 * j + r] = blk[r][c];
                    }
            }
        }
    }
    double w[12];
    jacobi_svd_rows<12, SITE>(A, w);
    // null-space basis: v_i = the singular vector of the (i+1)-th smallest singular value
    const double* v[4] = {A[11], A[10], A[9], A[8]};
    // L (6 x 10) and rho over the control-point pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3); betas ordered
    // [b11 b12 b22 b13 b23 b33 b14 b24 b34 b44]
    const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
    double L[6][10], rho[6];
    for (int r = 0; r < 6; ++r) {
        double dv[4][3];
        for (int i = 0; i < 4; ++i)
            for (int c = 0; c < 3; ++c) dv[i][c] = v[i][3 * pa[r] + c] - v[i][3 * pb[r] + c];
        L[r][0] = dot3(dv[0], dv[0]);
        L[r][1] = 2.0 * dot3(dv[0], dv[1]);
        L[r][2] = dot3(dv[1], dv[1]);
        L[r][3] = 2.0 * dot3(dv[0], dv[2]);
        L[r][4] = 2.0 * dot3(dv[1], dv[2]);
        L[r][5] = dot3(dv[2], dv[2]);
        L[r][6] = 2.0 * dot3(dv[0], dv[3]);
        L[r][7] = 2.0 * dot3(dv[1], dv[3]);
        L[r][8] = 2.0 * dot3(dv[2], dv[3]);
        L[r][9] = dot3(dv[3], dv[3]);
        double d[3];
        for (int c = 0; c < 3; ++c) d[c] = cp.c[pa[r]][c] - cp.c[pb[r]][c];
        rho[r] = dot3(d, d);
    }
    double betas[3][4];
    {   // N = 1 (paper): [b11 b12 b13 b14] from columns 0 1 3 6
        double M4[6][4], r4[6], x[4];
        for (int r = 0; r < 6; ++r) { M4[r][0] = L[r][0]; M4[r][1] = L[r][1]; M4[r][2] = L[r][3]; M4[r][3] = L[r][6]; r4[r] = rho[r]; }
        lstsq<6, 4, SITE>(M4, r4, x);
        const double b0 = sqrt(fabs(x[0])), sg = x[0] < 0.0 ? -1.0 : 1.0;
        betas[0][0] = b0;
        for (int i = 1; i < 4; ++i) betas[0][i] = sg * x[i] / b0;
    }
    {   // N = 2: [b11 b12 b22] from columns 0 1 2
        double M3[6][3], r3[6], x[3];
        for (int r = 0; r < 6; ++r) { for (int c = 0; c < 3; ++c) M3[r][c] = L[r][c]; r3[r] = rho[r]; }
        lstsq<6, 3, SITE>(M3, r3, x);
        double b0, b1;
        if (x[0] < 0.0) { b0 = sqrt(-x[0]); b1 = x[2] < 0.0 ? sqrt(-x[2]) : 0.0; }
        else { b0 = sqrt(x[0]); b1 = x[2] > 0.0 ? sqrt(x[2]) : 0.0; }
        if (x[1] < 0.0) b0 = -b0;
        betas[1][0] = b0; betas[1][1] = b1; betas[1][2] = 0.0; betas[1][3] = 0.0;
    }
    {   // N = 3: [b11 b12 b22 b13 b23] from columns 0..4
        double M5[6][5], r5[6], x[5];
        for (int r = 0; r < 6; ++r) { for (int c = 0; c < 5; ++c) M5[r][c] = L[r][c]; r5[r] = rho[r]; }
        lstsq<6, 5, SITE>(M5, r5, x);
        double b0, b1;
        if (x[0] < 0.0) { b0 = sqrt(-x[0]); b1 = x[2] < 0.0 ? sqrt(-x[2]) : 0.0; }
        else { b0 = sqrt(x[0]); b1 = x[2] > 0.0 ? sqrt(x[2]) : 0.0; }
        if (x[1] < 0.0) b0 = -b0;
        betas[2][0] = b0; betas[2][1] = b1; betas[2][2] = x[3] / b0; betas[2][3] = 0.0;
    }
    const int bi[10] = {0, 0, 1, 0, 1, 2, 0, 1, 2, 3}, bj[10] = {0, 1, 1, 2, 2, 2, 3, 3, 3, 3};
    for (int c = 0; c < 3; ++c) {
        double* be = betas[c];
        for (int it = 0; it < 5; ++it) {        // Gauss-Newton on sum_r (L_r . bb(be) - rho_r)^2
            double J[6][4], res[6], dx[4];
            for (int r = 0; r < 6; ++r) {
                const double* l = L[r];
                J[r][0] = 2.0 * l[0] * be[0] + l[1] * be[1] + l[3] * be[2] + l[6] * be[3];
                J[r][1] = l[1] * be[0] + 2.0 * l[2] * be[1] + l[4] * be[2] + l[7] * be[3];
                J[r][2] = l[3] * be[0] + l[4] * be[1] + 2.0 * l[5] * be[2] + l[8] * be[3];
                J[r][3] = l[6] * be[0] + l[7] * be[1] + l[8] * be[2] + 2.0 * l[9] * be[3];
                double s = 0.0;
                for (int m = 0; m < 10; ++m) s += l[m] * be[bi[m]] * be[bj[m]];
                res[r] = rho[r] - s;
            }
            lstsq<6, 4, SITE>(J, res, dx);
            for (int i = 0; i < 4; ++i) be[i] += dx[i];
        }
        double ccs[4][3];
        for (int j = 0; j < 4; ++j)
            for (int k = 0; k < 3; ++k)
                ccs[j][k] = be[0] * v[0][3 * j + k] + be[1] * v[1][3 * j + k] + be[2] * v[2][3 * j + k] + be[3] * v[3][3 * j + k];
        const double z0 = al_first[0] * ccs[0][2] + al_first[1] * ccs[1][2] + al_first[2] * ccs[2][2] + al_first[3] * ccs[3][2];
        if (z0 < 0.0)
            for (int j = 0; j < 4; ++j)
                for (int k = 0; k < 3; ++k) ccs[j][k] = -ccs[j][k];
        procrustes<SITE>(ccs, acc, n, cp.c[0], cand[c]);
    }
}

// pixel reprojection error of one point under a candidate
EPNP_HD double reproj_error(const Candidate& c, const Intrinsics& in, double x, double y, double z, double u, double v) {
    const double X = c.R[0] * x + c.R[1] * y + c.R[2] * z + c.t[0];
    const double Y = c.R[3] * x + c.R[4] * y + c.R[5] * z + c.t[1];
    const double Z = c.R[6] * x + c.R[7] * y + c.R[8] * z + c.t[2];
    const double eu = u - (in.uc + in.fu * X / Z), ev = v - (in.vc + in.fv * Y / Z);
    return sqrt(eu * eu + ev * ev);
}

// the winner among the candidates by summed reprojection error (the earlier one on ties); pose = [x y z w i j k]
EPNP_HD int pick_candidate(const double (&err)[3]) {
    int best = 0;
    if (err[1] < err[best]) best = 1;
    if (err[2] < err[best]) best = 2;
    return best;
}
EPNP_HD void write_pose(const Candidate& c, float* pose) {
    for (int i = 0; i < 3; ++i) pose[i] = (float)c.t[i];
    for (int i = 0; i < 4; ++i) pose[3 + i] = (float)c.q[i];
}

}  // namespace epnp
}  // namespace pnp
