/* epropnp_b200.h -- C ABI of libepropnp_b200.so: the EPro-PnP hot path (batched LM / GN pose solve
 * and the AMIS Monte-Carlo loop) as hand-written sm_90a CUDA.
 *
 * The reference (tjiiv-cprg/EPro-PnP) has NO native interface for this path: it is ~10^3 PyTorch
 * op launches behind Python classes.  This header is therefore the FFI a maintainer would bind
 * underneath those classes; each entry point names the reference code it replaces (file:line under
 * epropnp/ of the reference).  The Python mirror of the reference surface that calls it lives in
 * epro-pnp_b200/epropnp/ ; INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous row-major fp32 unless the name ends in _host;
 *   - the caller owns and allocates every buffer; the library allocates no memory, is re-entrant, and only enqueues work
 *     on `stream` (a cudaStream_t passed as void*).  Per-host-thread state, exactly two items: the cudaError_t of the
 *     last failed call (epnp_last_cuda_error) and the four helper streams of the host-buffer calls, created on that
 *     thread's first host-buffer call and kept for its lifetime;
 *   - return value: EPNP_OK or a negative EPNP_ERR_* code (never throws, never aborts);
 *     CUDA launch errors come back as EPNP_ERR_CUDA (epnp_last_cuda_error() has the cudaError_t);
 *   - B = objects, N = correspondences per object, D = 7 (dof 6: x y z w i j k) or 4 (dof 4:
 *     x y z yaw), M = mc_samples, I = mc_iter, S = M / I;
 *   - nullable arguments are marked [opt];
 *   - AMIS outputs are OBJECT-MAJOR: pose_samples (B, M, D), logw (B, M).  The reference returns
 *     (M, B, D) / (M, B); the Python layer hands out transposed views.
 */
#ifndef EPROPNP_B200_H
#define EPROPNP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EPNP_ABI_VERSION 2   /* 2: epnp_rslm_draw_f32 added; the push entry point takes DEVICE arrays of peer pointers */

enum {
    EPNP_OK = 0,
    EPNP_ERR_BAD_ARG = -1,       /* null pointer, non-positive size, dof not in {4,6}, M % I != 0 ...  */
    EPNP_ERR_TOO_MANY_POINTS = -2, /* N (and M) do not fit the 227 KB shared memory of one SM       */
    EPNP_ERR_UNSUPPORTED = -3,   /* combination not supported by this build                            */
    EPNP_ERR_CUDA = -4,          /* a CUDA runtime call failed, see epnp_last_cuda_error()             */
    EPNP_ERR_NO_DEVICE = -5      /* no sm_90 device is current                                         */
};

/* Hyper-parameters of the solve.  Defaults (epnp_default_params) are the reference's constructor
 * defaults: LMSolver.__init__ levenberg_marquardt.py:31-53, HuberPnPCost.__init__ cost_fun.py:25-28,
 * PerspectiveCamera.__init__ camera.py:35-43, EProPnPBase/6DoF.__init__ epropnp.py:47-62,273-280. */
typedef struct EpnpParams {
    int32_t dof;                    /* 4 or 6                                                   */
    int32_t lm_iter;                /* LMSolver.num_iter                                        */
    int32_t fast_mode;              /* 1: Gauss-Newton, no trust region, no clip_jac            */
    float   z_min;                  /* PerspectiveCamera.z_min                                  */
    float   min_lm_diagonal;
    float   max_lm_diagonal;
    float   min_relative_decrease;
    float   initial_radius;         /* initial_trust_region_radius                              */
    float   max_radius;             /* max_trust_region_radius                                  */
    float   eps;                    /* LMSolver.eps                                             */
    float   huber_eps;              /* HuberPnPCost.eps                                         */
    int32_t mc_samples;             /* EProPnPBase.mc_samples  (M)                              */
    int32_t mc_iter;                /* EProPnPBase.num_iter    (I)                              */
    float   amis_eps;               /* EProPnPBase.eps                                          */
    int32_t acg_mle_iter;           /* EProPnP6DoF.acg_mle_iter                                 */
    float   acg_dispersion;         /* EProPnP6DoF.acg_dispersion                               */
} EpnpParams;

int         epnp_abi_version(void);
const char* epnp_error_string(int code);
int         epnp_last_cuda_error(void);             /* cudaError_t of the last EPNP_ERR_CUDA    */
void        epnp_default_params(EpnpParams* p, int dof);
/* Largest N one object may have (correspondences are resident in shared memory); mc_samples = 0
 * for the LM-only entry points. */
int         epnp_max_points(int dof, int mc_samples, int mc_iter);

/* Cluster-split entry points (epnp_lm_amis_fused_split_f32, epnp_evaluate_cost_split_f32): for N above
 * epnp_max_points, one object is spread over a thread-block cluster of C = 2..8 CTAs on C SMs; CTA r holds the r-th
 * range of ceil(N / C) points (rounded up to a multiple of 8) and the ranks' partial costs are added over distributed
 * shared memory in rank order.
 *   epnp_split_ctas: the C those calls choose automatically -- the smallest C >= 2 whose largest share fits one SM's
 *     shared memory; 0 when even 8 CTAs are too few (or the arguments are invalid).  A function of (dof, N, M, I) only;
 *     mc_samples = 0 gives the plan of both epnp_evaluate_cost_split_f32 and epnp_gn_plus_backward_split_f32.
 *   epnp_max_points_split: the largest N any C can take (a multiple of 64). */
int         epnp_split_ctas(int dof, int N, int mc_samples, int mc_iter);
int         epnp_max_points_split(int dof, int mc_samples, int mc_iter);

/* AdaptiveHuberPnPCost.set_param (cost_fun.py:123-126):
 *   delta[b] = mean(w2d[b]) * sqrt(sum_xy var_unbiased(x2d[b])) * relative_delta               */
int epnp_adaptive_delta_f32(const float* x2d, const float* w2d, float relative_delta,
                            float* delta /*(B)*/, int B, int N, void* stream);

/* evaluate_pnp(..., out_cost=True) for a stack of poses (common.py:67-100 through camera.py:21-30
 * `project_b` and cost_fun.py:52-59): poses (S, B, D) -> cost (S, B).  S may be 1.
 * lb/ub: [opt] (B, 2) clamp bounds of the projection (both or neither).                        */
int epnp_evaluate_cost_f32(const float* x3d /*(B,N,3)*/, const float* x2d /*(B,N,2)*/,
                           const float* w2d /*(B,N,2)*/, const float* cam_mats /*(B,3,3)*/,
                           const float* lb, const float* ub, const float* delta /*(B)*/,
                           const float* poses, float* cost,
                           int S, int B, int N, int dof, float z_min, void* stream);

/* epnp_evaluate_cost_f32 for objects of up to epnp_max_points_split(dof, 0, 0) points: one cluster of C CTAs per
 * object.  cluster_ctas = 0 takes C = epnp_split_ctas(dof, N, 0, 0); a caller may ask for any C from that minimum to
 * 8 (EPNP_ERR_BAD_ARG outside it, EPNP_ERR_TOO_MANY_POINTS when no C fits).  The costs depend on C (it sets the order
 * in which the ranks' partial sums are added) and never on B.  EPNP_ERR_UNSUPPORTED when the device cannot run one
 * cluster of that size (cudaOccupancyMaxActiveClusters = 0, e.g. a MIG slice); nothing is launched then.          */
int epnp_evaluate_cost_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                 const float* lb, const float* ub, const float* delta, const float* poses, float* cost,
                                 int S, int B, int N, int dof, float z_min, int cluster_ctas, void* stream);

/* evaluate_pnp(..., out_jacobian, out_residual, out_cost) at one pose per object (common.py:67-100,
 * camera.py:10-18,64-143, cost_fun.py:33-89): pose (B, D) ->
 * residual [opt] (B, 2N), jac [opt] (B, 2N, dof), cost [opt] (B).                              */
int epnp_evaluate_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose,
                      float* residual, float* jac, float* cost, int clip_jac,
                      int B, int N, int dof, float z_min, float huber_eps, void* stream);

/* Backward of epnp_evaluate_f32's outputs at S stacked poses (S, B, D): the vector-Jacobian product with any of the
 * upstream gradients grad_residual (S, B, 2N), grad_jac (S, B, 2N, dof) and grad_cost (S, B) (at least one; a null one
 * counts as zero), differentiated as the reference's autograd differentiates evaluate_pnp(out_residual, out_jacobian,
 * out_cost): no tangent through a depth clamped at z_min, a coordinate clamped at a bound takes that bound's tangent,
 * the clip mask is constant, the Huber scale keeps its branches and huber_eps, the Jacobian's rows are differentiated
 * as written with K's first two rows, and the rotation with respect to the raw pose components.  Outputs, each optional
 * but at least one:
 *   grad_x3d (B, N, 3), grad_x2d / grad_w2d (B, N, 2), grad_delta (B)   summed over the S poses
 *   grad_pose (S, B, D)
 *   grad_cam (B, 3, 3), grad_lb / grad_ub (B, 2)                         summed over the S poses; bounds' only with bounds
 * One CTA per object over the points in global memory: any N.  Fixed-order reductions, no atomics: an object's results
 * depend on nothing else in the batch.  B = 0 or S = 0 writes nothing.                                           */
int epnp_evaluate_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                               const float* lb, const float* ub, const float* delta, const float* poses,
                               const float* grad_residual, const float* grad_jac, const float* grad_cost,
                               float* grad_x3d, float* grad_x2d, float* grad_w2d, float* grad_delta, float* grad_pose,
                               float* grad_cam, float* grad_lb, float* grad_ub, int clip_jac, int S, int B, int N,
                               int dof, float z_min, float huber_eps, void* stream);

/* Forward mode of epnp_evaluate_f32's outputs at S stacked poses (S, B, D): the Jacobian-vector product with one
 * tangent, the transpose of epnp_evaluate_backward_f32 (<g, J v> = <J^T g, v>) with its gates.  Tangent [opt, NULL =
 * zero]: t_x3d (B,N,3), t_x2d / t_w2d (B,N,2), t_delta (B), t_pose (S,B,D) (raw components, through the forward's
 * rotation), t_cam (B,3,3), t_lb / t_ub (B,2).  Outputs, each optional but at least one:
 *   d_residual (S, B, 2N), d_jac (S, B, 2N, dof), d_cost (S, B)
 * Two launches: point-major (one CTA per pose and object, the points streamed from global memory: any N; d_cost one
 * fixed-order block sum) and, for d_cost alone at S >= 64 poses, pose-major (thread per pose, the points staged through
 * shared memory).  No atomics: results are bit-identical from run to run.  Refusals as epnp_evaluate_backward_f32
 * (S < 0, S * B above INT_MAX, no output) and t_lb / t_ub without bounds: EPNP_ERR_BAD_ARG.  B = 0 or S = 0 writes
 * nothing.                                                                                                       */
int epnp_evaluate_jvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                          const float* lb, const float* ub, const float* delta, const float* poses,
                          const float* t_x3d, const float* t_x2d, const float* t_w2d, const float* t_delta,
                          const float* t_pose, const float* t_cam, const float* t_lb, const float* t_ub,
                          float* d_residual, float* d_jac, float* d_cost, int clip_jac, int S, int B, int N, int dof,
                          float z_min, float huber_eps, void* stream);

/* Backward of the derivative-regularisation branch: pose_opt_plus = pose (+) gn_step(pose) with the pose detached
 * (LMSolver.forward :66-68, gn_step :243-253, pose_add :255-265, evaluated with autograd on in the reference:
 * camera.py:119-129, cost_fun.py:52-84).  Given dL/d pose_opt_plus (B, D), writes dL/d x3d (B, N, 3), dL/d x2d
 * (B, N, 2), dL/d w2d (B, N, 2) and dL/d delta (B) (each optional).  The forward value is what
 * epnp_lm_solve_f32 returns in pose_opt_plus (lm_iter = 0 evaluates the step at pose_init).                      */
int epnp_gn_plus_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                              const float* lb, const float* ub, const float* delta, const float* pose,
                              const float* grad_pose_plus, float* grad_x3d, float* grad_x2d, float* grad_w2d,
                              float* grad_delta, int B, int N, int dof, float z_min, float eps, float huber_eps,
                              void* stream);

/* epnp_gn_plus_backward_f32 for objects of up to epnp_max_points_split(dof, 0, 0) points (the dense coordinate maps of
 * training): one cluster of C CTAs per object, each rank holding one range of the points; the ranks' normal equations
 * and grad_delta partials are added over distributed shared memory in rank order, and each rank writes the gradient rows
 * of its own points.  cluster_ctas = 0 takes C = epnp_split_ctas(dof, N, 0, 0); a caller may ask for any C from that
 * minimum to 8 (EPNP_ERR_BAD_ARG outside it, EPNP_ERR_TOO_MANY_POINTS when no C fits).  The gradients depend on C (the
 * order of the sums over ranks) and never on B or the object's position in the batch.  EPNP_ERR_UNSUPPORTED when the
 * device cannot run one cluster of that size; nothing is launched then.  Each output stays optional.               */
int epnp_gn_plus_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                    const float* lb, const float* ub, const float* delta, const float* pose,
                                    const float* grad_pose_plus, float* grad_x3d, float* grad_x2d, float* grad_w2d,
                                    float* grad_delta, int B, int N, int dof, float z_min, float eps, float huber_eps,
                                    int cluster_ctas, void* stream);

/* Everything RSLMSolver.solve does before its solves (levenberg_marquardt.py:283-324) in one launch:
 *   the centre-based translation guess (center_based_init, :283-298: mean ray direction times the ratio of the 3D spread
 *     to the ray spread), computed per object unless t_init (B, 3) is given; written to t_out [opt] (B, 3);
 *   inds (P, B, n) int32: per (proposal, object) n distinct correspondence indices drawn WITHOUT replacement with
 *     probabilities proportional to mean(w2d, -1) -- torch.multinomial(mean_weight, num_points) (:306-309), by the
 *     same exponential race (the n smallest E_i / w_i, E_i ~ Exp(1)); a weight <= 0 is never drawn while a positive
 *     one is left (the reference raises when fewer than n are positive; here the subset is completed in index order);
 *   start (P, B, D): that translation (:314) + a uniformly random orientation: normalised Gaussian quaternion,
 *     (1,0,0,0) when its norm < eps (:319-324), or a yaw uniform on [0, 2 pi) (:316-317).
 * x3d / x2d / cam_mats may be NULL when t_init is given.
 * Philox-4x32-10 keyed by (seed; obj_offset + object, proposal): a batch shard draws what the whole batch would.   */
int epnp_rslm_draw_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                       const float* t_init, uint64_t seed, uint32_t obj_offset,
                       int* inds, float* start, float* t_out,
                       int P, int n, int B, int N, int dof, float eps, void* stream);

/* CUDA-graph capture.  A by-value seed is baked into a captured launch, so every replay of a graph would draw the
 * same samples.  The *_seedptr_f32 forms below take the seed as `const uint64_t* seed`, a DEVICE address the kernel
 * reads when it starts; a graph that writes a new seed there (e.g. torch.randint on the device, inside the graph)
 * draws new samples at every replay.  Arguments, checks and results are otherwise those of the by-value call: given
 * the value *seed, the outputs equal the by-value call's bit for bit.  EPNP_ERR_BAD_ARG also for seed == NULL.
 * These and the other device-buffer calls only enqueue kernels on `stream`, so they may be captured.  Not capturable,
 * and without a seed-pointer form: the host-buffer calls (epnp_lm_amis_fused_host_f32 and its split form run their
 * own helper streams and events) and the push calls (epnp_lm_amis_fused_push_f32 and its split form write into
 * IPC-mapped peer buffers that the ranks hand over outside the stream, around an all-reduce).                      */
int epnp_rslm_draw_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                               const float* t_init, const uint64_t* seed, uint32_t obj_offset,
                               int* inds, float* start, float* t_out,
                               int P, int n, int B, int N, int dof, float eps, void* stream);

/* RSLMSolver.solve after the hypotheses are drawn (levenberg_marquardt.py:300-353): for every object, P starting
 * poses, each refined by LM / GN on its own n sampled correspondences, scored on all N correspondences, cheapest
 * kept.  Replaces the reference's gather of (P*B, n, .) mini-problems, the P-fold repeated camera / cost objects,
 * the solve of P*B tiny problems and the stacked evaluate_pnp (:326-352).
 *   inds (P, B, n) int32: sampled correspondence indices WITHIN the object (the torch.multinomial draw, :310-312)
 *   start (P, B, D): starting poses (centre-based translation + random orientation, :314-324)
 *   pose_best (B, D), cost_best (B); pose_all [opt] (P, B, D), cost_all [opt] (P, B)                          */
int epnp_rslm_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                  const float* lb, const float* ub, const float* delta, const int* inds, const float* start,
                  float* pose_best, float* cost_best, float* pose_all, float* cost_all,
                  int P, int n, int B, int N, const EpnpParams* p, void* stream);

/* epnp_rslm_f32 for objects of up to epnp_max_points_split(dof, 0, 0) points, as three launches on `stream`: one
 * thread per (hypothesis, object) refines the hypothesis on its n correspondences, read from the object's rows in
 * global memory (pose_all: bit-identical to epnp_rslm_f32's for the same inds / start); epnp_evaluate_cost_split_f32's
 * kernel scores the P poses on all N points on the object's cluster (cost_all: bit-identical to that call on pose_all
 * with the same C and params->z_min); one thread per object keeps the cheapest (torch.min's order: a NaN cost wins,
 * then the smaller cost, then the earlier hypothesis) in pose_best / cost_best.  The costs, and so a winner between
 * nearly equal hypotheses, depend on C (the order of the ranks' partial sums), never on B.
 *   pose_all (P, B, D) and cost_all (P, B) are REQUIRED: they carry the results from one launch to the next.
 *   cluster_ctas as epnp_evaluate_cost_split_f32's (0: epnp_split_ctas(dof, N, 0, 0); EPNP_ERR_BAD_ARG outside [that
 *   minimum, 8]; EPNP_ERR_TOO_MANY_POINTS when no C fits, for any B).  EPNP_ERR_UNSUPPORTED when the device cannot
 *   run one cluster of that size; nothing is launched then.                                                       */
int epnp_rslm_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                        const float* lb, const float* ub, const float* delta, const int* inds, const float* start,
                        float* pose_best, float* cost_best, float* pose_all, float* cost_all,
                        int P, int n, int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);

/* EPnP initialisation of the 6DoF test-time solve (EPro-PnP-6DoF/lib/test.py:178-194): per object,
 *   conf_i = (w2d[i,0] + w2d[i,1]) / 2, the points with conf_i >= np.quantile(conf, conf_quantile) (NumPy 2.x
 *   'linear', evaluated in fp32 as NumPy does for a float32 row; ties kept) -> cv2.solvePnP(..., SOLVEPNP_EPNP)
 *   (pixel coordinates, fu = K00, fv = K11, uc = K02, vc = K12; K01 is not read) -> pose (B, 7) = [x y z w i j k],
 *   the quaternion normalised with w >= 0.  EPnP runs in fp64.  w2d [opt]: NULL keeps every point.
 *   n_sel [opt] (B) int32: points kept per object.  The camera bounds and z_min of the other entry points do not
 *   apply (cv2's EPnP has none).  An object with a NaN confidence gets a NaN pose and n_sel = 0; degenerate (coplanar,
 *   collinear) kept points give a finite or NaN pose; neither affects other objects.
 *   EPNP_ERR_BAD_ARG: N < 4, conf_quantile outside [0, 1], or fewer than 4 points kept by construction
 *   (N - floor((N-1) q) - (fractional part > 0) < 4 with w2d given; cv2 refuses those); EPNP_ERR_TOO_MANY_POINTS:
 *   N > epnp_max_points(6, 0, 0). */
int epnp_epnp_init_f32(const float* x3d, const float* x2d, const float* w2d /*[opt] NULL = all points*/,
                       const float* cam_mats, float conf_quantile, float* pose /*(B,7)*/, int* n_sel /*[opt]*/,
                       int B, int N, void* stream);

/* epnp_epnp_init_f32 for objects of up to epnp_max_points_split(6, 0, 0) points (the dense coordinate maps of the 6DoF
 * test loop): one cluster of C CTAs per object, each rank holding one range of the points.  The radix-select counts,
 * the kept counts and the fp64 sums are added over distributed shared memory in rank order, so every rank solves the
 * same EPnP problem; rank 0 writes pose and n_sel.  The kept set is exactly that of epnp_epnp_init_f32 (the counts
 * are integers) for every C; the pose depends on C (the order of the fp64 sums over ranks) and never on B or the
 * object's position in the batch.  cluster_ctas = 0 takes C = epnp_split_ctas(6, N, 0, 0); a caller may ask for any C
 * from that minimum to 8 (EPNP_ERR_BAD_ARG outside it, EPNP_ERR_TOO_MANY_POINTS when no C fits).  EPNP_ERR_UNSUPPORTED
 * when the device cannot run one cluster of that size; nothing is launched then.  The other arguments, checks and the
 * NaN / degenerate-object semantics are those of epnp_epnp_init_f32.                                                 */
int epnp_epnp_init_split_f32(const float* x3d, const float* x2d, const float* w2d /*[opt] NULL = all points*/,
                             const float* cam_mats, float conf_quantile, float* pose /*(B,7)*/, int* n_sel /*[opt]*/,
                             int B, int N, int cluster_ctas, void* stream);

/* LMSolver.solve with a given pose_init (levenberg_marquardt.py:80-190, _lm_iter :192-241, GN
 * fast mode :136-152) plus, when pose_opt_plus != NULL, the extra Gauss-Newton step of
 * LMSolver.forward (:66-68, gn_step :243-253, pose_add :255-265).
 *   pose_opt (B, D); pose_cov [opt] (B, dof, dof) = inverse(J^T J + eps I); cost [opt] (B);
 *   cost_init [opt] (B) = cost at pose_init (what monte_carlo_forward returns, epropnp.py:121-124)
 * In fast mode pose_cov, cost and cost_init come from the evaluation before a Gauss-Newton step, so fast_mode != 0
 * with lm_iter = 0 returns EPNP_ERR_BAD_ARG (for any B) when any of the three is requested; pose_opt alone (= pose_init)
 * and pose_opt_plus stay allowed.  The fused calls (resident, split, seed-pointer, push and host-buffer forms) always
 * compute the covariance and refuse that combination outright.                                                     */
int epnp_lm_solve_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* pose_init,
                      float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                      float* cost_init, int B, int N, const EpnpParams* p, void* stream);

/* The AMIS loop of EProPnPBase.monte_carlo_forward (epropnp.py:132-182) for EProPnP6DoF
 * (initial_fit :288-302, gen_new/old_distr :304-315, estimate_params :317-342; proposals from
 * distributions.py:15-52 and pyro MultivariateStudentT), starting from a given local solution.
 *   noise_*: [opt] injected base noise, object-major, m = iteration * S + s:
 *            noise_normal (B, M, 3), noise_chi2 (B, M), noise_rot (B, M, 4) for dof 6; for dof 4
 *            (EProPnP4DoF, epropnp.py:199-260, distributions.py:55-79) noise_rot is (B, M) and holds the
 *            YAW DRAWS themselves (the reference samples yaw with numpy on the host).  All three or none;
 *            when NULL the kernel draws Philox-4x32-10 noise keyed by (seed, obj_offset + b, m),
 *            so a sharded batch reproduces the unsharded one.
 *   proposals [opt] (B, I, 19): mode[3], L_t[6] (row-major lower), L_r[10] per AMIS iteration
 *            (dof 4: mode[3], L_t[6], yaw mode, kappa, 0...).                                     */
int epnp_amis_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                  const float* lb, const float* ub, const float* delta,
                  const float* pose_opt, const float* pose_cov,
                  const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                  uint64_t seed, uint32_t obj_offset,
                  float* pose_samples /*(B,M,D)*/, float* logw /*(B,M)*/, float* proposals,
                  int B, int N, const EpnpParams* p, void* stream);

/* monte_carlo_forward with pose_init given and no init solver (epropnp.py:87-196 with force_init_solve=False):
 * LM solve + covariance + AMIS in ONE call = two launches on `stream`, no host round trip -- the warp-per-object LM
 * kernel (epnp_lm_solve_f32's), then the CTA-per-object AMIS kernel (epnp_amis_f32's); each stages the object's
 * correspondence set once into shared memory by TMA bulk copies.  (As a single kernel the LM half ran latency-bound:
 * DESIGN.md section 0.)  pose_cov [opt]: when NULL, the covariance travels between the two kernels through the first
 * dof^2 floats of each object's -- not yet written -- pose_samples rows (needs M * D >= dof^2).                      */
int epnp_lm_amis_fused_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                           const float* lb, const float* ub, const float* delta, const float* pose_init,
                           const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                           uint64_t seed, uint32_t obj_offset,
                           float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                           float* cost_init, float* pose_samples, float* logw, float* proposals,
                           int B, int N, const EpnpParams* p, void* stream);
/* epnp_lm_amis_fused_f32 with the Philox seed read from device memory (see epnp_rslm_draw_seedptr_f32). */
int epnp_lm_amis_fused_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                   const float* lb, const float* ub, const float* delta, const float* pose_init,
                                   const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                   const uint64_t* seed, uint32_t obj_offset,
                                   float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                                   float* cost_init, float* pose_samples, float* logw, float* proposals,
                                   int B, int N, const EpnpParams* p, void* stream);

/* epnp_lm_amis_fused_f32 for objects of up to epnp_max_points_split(dof, M, I) points (the dense coordinate maps of
 * out_res = 128 and beyond): the same arguments, outputs and noise conventions, plus cluster_ctas.  The LM half is
 * epnp_lm_solve_f32's kernel, which takes any N; the AMIS loop runs on one cluster of C CTAs per object.  Every rank
 * draws the same samples and, after exchanging its partial costs each iteration, holds the same costs and refits;
 * rank 0 writes pose_samples, logw and proposals.  cluster_ctas = 0 takes C = epnp_split_ctas(dof, N, M, I); a caller
 * may ask for any C from that minimum to 8 (EPNP_ERR_BAD_ARG outside it, EPNP_ERR_TOO_MANY_POINTS when no C fits).
 * Results depend on C (the order in which the ranks' partial costs are added), never on B, the shard or obj_offset;
 * they agree with epnp_lm_amis_fused_f32 to fp32 rounding, not bit for bit.  EPNP_ERR_UNSUPPORTED when the device
 * cannot run one cluster of that size (cudaOccupancyMaxActiveClusters = 0, e.g. a MIG slice); the LM kernel is not
 * launched either then.  Its push and host-buffer forms: epnp_lm_amis_fused_split_push_f32,
 * epnp_lm_amis_fused_split_host_f32.                                                                              */
int epnp_lm_amis_fused_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                 const float* lb, const float* ub, const float* delta, const float* pose_init,
                                 const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                 uint64_t seed, uint32_t obj_offset,
                                 float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                                 float* cost_init, float* pose_samples, float* logw, float* proposals,
                                 int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);
/* epnp_lm_amis_fused_split_f32 with the Philox seed read from device memory (see epnp_rslm_draw_seedptr_f32). */
int epnp_lm_amis_fused_split_seedptr_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                         const float* lb, const float* ub, const float* delta, const float* pose_init,
                                         const float* noise_normal, const float* noise_chi2, const float* noise_rot,
                                         const uint64_t* seed, uint32_t obj_offset,
                                         float* pose_opt, float* pose_cov, float* cost, float* pose_opt_plus,
                                         float* cost_init, float* pose_samples, float* logw, float* proposals,
                                         int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);

/* Multi-GPU form of epnp_lm_amis_fused_f32 (one process per GPU, one NVLink / NVSwitch node): the solve AND the gather
 * of its small results in one kernel (the AMIS kernel).  Every CTA, when its object is finished, additionally stores the object's
 * pose_opt row and its M log-weights into row (obj_offset + b) of `n_peers` (<= 8) full-batch buffers that live in
 * OTHER GPUs' memory -- peer_logw[r] (B_total, M), peer_pose[r] (B_total, D), device pointers the caller obtained with
 * cudaIpcOpenMemHandle(..., cudaIpcMemLazyEnablePeerAccess) WHILE THIS DEVICE WAS CURRENT (a mapping opened under the
 * exporting device's index is not dereferenceable by this device's kernels) -- with plain stores over NVLink, object
 * by object underneath the remaining math.  peer_logw / peer_pose themselves are DEVICE arrays of n_peers pointers (in
 * this device's memory, like a batched-BLAS pointer array; the kernel reads them when an object finishes): built once
 * per set of buffers, they must stay valid until the launch has completed.
 * There is no gather kernel and no copy afterwards (what replaces the NCCL all-gather of SURVEY.md section 8e); the
 * caller needs one rendezvous of the ranks before it reads its own full-batch buffer.  pose_opt / logw are the LOCAL
 * outputs as before -- typically the local slice [obj_offset, obj_offset + B) of this rank's own full-batch buffers.
 * obj_offset doubles as the global object index of the Philox stream, so the assembled batch is bit-identical to the
 * single-GPU run.  Injected noise, pose_opt_plus, cost_init and proposals are not offered by this entry point. */
int epnp_lm_amis_fused_push_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                const float* lb, const float* ub, const float* delta, const float* pose_init,
                                uint64_t seed, uint32_t obj_offset,
                                float* pose_opt, float* pose_cov, float* cost, float* pose_samples, float* logw,
                                float* const* peer_logw, float* const* peer_pose, int n_peers,
                                int B, int N, const EpnpParams* p, void* stream);

/* epnp_lm_amis_fused_push_f32 for objects of up to epnp_max_points_split(dof, M, I) points: the same arguments plus
 * cluster_ctas (as epnp_lm_amis_fused_split_f32).  The solve is epnp_lm_amis_fused_split_f32's into the local outputs;
 * then, on the same stream, one copy kernel stores this rank's rows -- pose_opt (B, D) and logw (B, M) -- into rows
 * [obj_offset, obj_offset + B) of every peer's buffers (nothing is launched after the solve when n_peers = 0).  The
 * peers therefore hold exactly the local results, which equal epnp_lm_amis_fused_split_f32's bit for bit.  Refusals as
 * epnp_lm_amis_fused_split_f32's, all before the first launch.                                                    */
int epnp_lm_amis_fused_split_push_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                      const float* lb, const float* ub, const float* delta, const float* pose_init,
                                      uint64_t seed, uint32_t obj_offset,
                                      float* pose_opt, float* pose_cov, float* cost, float* pose_samples, float* logw,
                                      float* const* peer_logw, float* const* peer_pose, int n_peers,
                                      int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);

/* Backward of the differentiable outputs of monte_carlo_forward (epropnp.py:108-113: cost_init and the
 * Monte-Carlo costs inside pose_sample_logweights; proposal densities and samples carry no gradient,
 * epropnp.py:139-140,172-179) and of evaluate_pnp(out_cost=True) (common.py:67-100): for every object
 *   grad_x3d/x2d/w2d/delta = sum_p grad[p] * d cost(pose p) / d (x3d, x2d, w2d, delta)
 * over two pose sets given object-major: set a (B, PA, D) with grad_a (B, PA) -- e.g. the AMIS samples and
 * -dL/dlogw -- and [opt] set b (B, PB, D), grad_b (B, PB) -- e.g. pose_init and dL/dcost_init.
 * Differentiates what the reference's autograd sees: project_b (camera.py:21-30), the z / bound clamps
 * (zero gradient where clamped, :81-93), Huber (cost_fun.py:8-12).  Outputs [opt]: (B,N,3), (B,N,2), (B,N,2), (B). */
int epnp_cost_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                           const float* lb, const float* ub, const float* delta,
                           const float* poses_a, const float* grad_a, int PA,
                           const float* poses_b, const float* grad_b, int PB,
                           float* grad_x3d, float* grad_x2d, float* grad_w2d, float* grad_delta,
                           int B, int N, int dof, float z_min, void* stream);

/* Backward of the same costs with respect to the POSE (the reference's evaluate_pnp is differentiable there too:
 * common.py:30-36, camera.py:21-30; cost_init of monte_carlo_forward with a predicted pose_init, epropnp.py:121-124):
 *   grad_pose[b, p] = grad[b, p] * d cost(poses[b, p]) / d poses[b, p]
 * for poses (B, P, D) given object-major with grad (B, P); grad_pose (B, P, D).  D = 7: [x y z w i j k], the gradient
 * with respect to the four RAW components of the un-normalised quaternion whose rotation the forward calls use
 * (R = (ww + ii - jj - kk ...), not a tangent vector; on unit quaternions it differs from the reference's
 * differentiable branch 1 - 2 (jj + kk) ... only along q itself); D = 4: [x y z yaw].  Same clamps as above: no gradient
 * through a depth clamped at z_min or a coordinate clamped at lb / ub.  One thread per pose, no atomics: a row depends
 * on its object and its pose only.  P = 0 or B = 0 writes nothing.                                              */
int epnp_cost_pose_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                const float* lb, const float* ub, const float* delta, const float* poses,
                                const float* grad, float* grad_pose, int P, int B, int N, int dof, float z_min,
                                void* stream);

/* epnp_cost_pose_backward_f32 for objects of up to epnp_max_points_split(dof, 0, 0) points, on the clusters of
 * epnp_evaluate_cost_split_f32: each rank sweeps its own range of the points, rank 0 adds the ranks' partial sums in
 * rank order and writes the rows.  cluster_ctas as there (0: epnp_split_ctas(dof, N, 0, 0); EPNP_ERR_BAD_ARG outside
 * [that minimum, 8]; EPNP_ERR_TOO_MANY_POINTS when no C fits); the gradient depends on C and never on B.
 * EPNP_ERR_UNSUPPORTED when the device cannot run one cluster of that size; nothing is launched then.           */
int epnp_cost_pose_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                      const float* lb, const float* ub, const float* delta, const float* poses,
                                      const float* grad, float* grad_pose, int P, int B, int N, int dof, float z_min,
                                      int cluster_ctas, void* stream);

/* Backward of the same costs with respect to the CAMERA (the reference differentiates cam_mats through project_a /
 * project_b and tensor lb / ub through torch.max / torch.min: camera.py:10-30,81-93):
 *   grad_cam[b] = sum_p grad[b, p] * d cost(poses[b, p]) / d cam_mats[b]                          (B, 3, 3)
 *   grad_lb[b], grad_ub[b] = the same with respect to lb[b], ub[b]                                   (B, 2)
 * over the pose sets of epnp_cost_backward_f32 (a: (B, PA, D) / (B, PA); b [opt]: (B, PB, D) / (B, PB)).  A coordinate
 * clamped at a bound passes its gradient to that bound; a depth clamped at z_min passes none.  Outputs are optional, but
 * at least one must be given, and grad_lb / grad_ub only with bounds (EPNP_ERR_BAD_ARG otherwise).  One CTA per object
 * and one fixed-order block reduction, no atomics: an object's result depends on nothing else in the batch.  N above
 * epnp_max_points(dof, 0, 0): EPNP_ERR_TOO_MANY_POINTS.  B = 0 writes nothing; PA = PB = 0 writes zeros.        */
int epnp_cost_camera_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                  const float* lb, const float* ub, const float* delta,
                                  const float* poses_a, const float* grad_a, int PA,
                                  const float* poses_b, const float* grad_b, int PB,
                                  float* grad_cam, float* grad_lb, float* grad_ub,
                                  int B, int N, int dof, float z_min, void* stream);

/* epnp_cost_camera_backward_f32 for objects of up to epnp_max_points_split(dof, 0, 0) points, on the clusters of
 * epnp_evaluate_cost_split_f32: each rank sweeps its own range of the points for every pose and reduces to 13 floats,
 * rank 0 adds the ranks' in rank order and stores.  cluster_ctas as there; the result depends on C and never on B.
 * EPNP_ERR_UNSUPPORTED when the device cannot run one cluster of that size; nothing is launched then.           */
int epnp_cost_camera_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                        const float* lb, const float* ub, const float* delta,
                                        const float* poses_a, const float* grad_a, int PA,
                                        const float* poses_b, const float* grad_b, int PB,
                                        float* grad_cam, float* grad_lb, float* grad_ub,
                                        int B, int N, int dof, float z_min, int cluster_ctas, void* stream);

/* Second order through the same costs: the Hessian-vector product of f = sum_b sum_p grad[b, p] * cost(poses[b, p]),
 * which is the backward of the three cost backwards above.  Tangent v [opt, NULL = zero]: t_x3d (B,N,3), t_x2d (B,N,2),
 * t_w2d (B,N,2), t_delta (B), t_pose (B,P,D), t_cam (B,3,3), t_lb / t_ub (B,2).  Outputs [opt]:
 *   h_x3d, h_x2d, h_w2d, h_delta, h_cam, h_lb, h_ub   (H v) with respect to the correspondences, delta and the camera
 *   h_pose (B,P,D)                                    grad[b, p] * (H_p v) with respect to pose p (raw components)
 *   h_grad (B,P)                                      d cost(poses[b, p]) . v   (the derivative with respect to grad)
 * The gates are those of the first-order backwards: nothing passes a depth clamped at z_min, a coordinate clamped at a
 * bound follows that bound, each side of the Huber threshold takes its own branch.  Two launches: point-major (one CTA
 * per object, fixed-order block reduction) when a problem output is given, pose-major (thread per pose) when h_pose or
 * h_grad is; both stream the points from global memory, so any N up to epnp_max_points_split(dof, 0, 0) runs, above it
 * EPNP_ERR_TOO_MANY_POINTS.  No atomics: results are bit-identical from run to run.  Refusals as
 * epnp_cost_backward_f32 (a single pose set, P >= 0), and t_lb / t_ub / h_lb / h_ub without bounds: EPNP_ERR_BAD_ARG.
 * B = 0 writes nothing; P = 0 writes zeros to the problem outputs.                                               */
int epnp_cost_hvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                      const float* lb, const float* ub, const float* delta, const float* poses, const float* grad, int P,
                      const float* t_x3d, const float* t_x2d, const float* t_w2d, const float* t_delta,
                      const float* t_pose, const float* t_cam, const float* t_lb, const float* t_ub,
                      float* h_x3d, float* h_x2d, float* h_w2d, float* h_delta, float* h_pose, float* h_grad,
                      float* h_cam, float* h_lb, float* h_ub, int B, int N, int dof, float z_min, void* stream);

/* The camera gradient of pose_opt_plus = pose (+) gn_step(pose) (epnp_gn_plus_backward_f32's function, differentiated
 * with respect to cam_mats and the bounds instead of the correspondences): grad_cam (B, 3, 3), grad_lb / grad_ub (B, 2),
 * optional with the rules of epnp_cost_camera_backward_f32.  K enters the projection and the Jacobian; the clip mask is
 * held constant, as in the reference's autograd.  A separate launch: epnp_gn_plus_backward_f32 is unchanged.    */
int epnp_gn_plus_camera_backward_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                     const float* lb, const float* ub, const float* delta, const float* pose,
                                     const float* grad_pose_plus, float* grad_cam, float* grad_lb, float* grad_ub,
                                     int B, int N, int dof, float z_min, float eps, float huber_eps, void* stream);

/* epnp_gn_plus_camera_backward_f32 on the clusters of epnp_gn_plus_backward_split_f32 (cluster_ctas and refusals as
 * there): every rank forms the same step and v, reduces the camera partials of its own points, and rank 0 adds the
 * ranks' in rank order.  The result depends on C and never on B.                                                 */
int epnp_gn_plus_camera_backward_split_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                                           const float* lb, const float* ub, const float* delta, const float* pose,
                                           const float* grad_pose_plus, float* grad_cam, float* grad_lb,
                                           float* grad_ub, int B, int N, int dof, float z_min, float eps,
                                           float huber_eps, int cluster_ctas, void* stream);

/* Second order through pose_opt_plus: the backward of epnp_gn_plus_backward_f32 and epnp_gn_plus_camera_backward_f32.
 * With f = grad_pose_plus . (pose (+) gn_step(pose)) as a function of theta = (x3d, x2d, w2d, delta, cam_mats, lb, ub)
 * (the pose held constant), and a tangent u of theta [opt, NULL = zero]: t_x3d (B,N,3), t_x2d (B,N,2), t_w2d (B,N,2),
 * t_delta (B), t_cam (B,3,3), t_lb / t_ub (B,2).  Outputs [opt]:
 *   h_x3d, h_x2d, h_w2d, h_delta, h_cam, h_lb, h_ub   (H u) with respect to each input, H the Hessian of f in theta
 *   h_grad (B,D)                                      d pose_opt_plus / d theta . u   (the derivative with respect to
 *                                                     grad_pose_plus)
 * The gates are those of the first-order backwards: the clip mask is constant, nothing passes a depth clamped at z_min,
 * a coordinate clamped at a bound follows that bound, each side of the Huber threshold (huber_eps included) takes its
 * own branch.  One CTA per object streams the points from global memory, so any N up to
 * epnp_max_points_split(dof, 0, 0) runs; above it EPNP_ERR_TOO_MANY_POINTS.  No atomics: results are bit-identical
 * from run to run.  Refusals as epnp_gn_plus_backward_f32, and t_lb / t_ub / h_lb / h_ub without bounds:
 * EPNP_ERR_BAD_ARG.  B = 0, or no output, writes nothing.                                                         */
int epnp_gn_plus_hvp_f32(const float* x3d, const float* x2d, const float* w2d, const float* cam_mats,
                         const float* lb, const float* ub, const float* delta, const float* pose,
                         const float* grad_pose_plus, const float* t_x3d, const float* t_x2d, const float* t_w2d,
                         const float* t_delta, const float* t_cam, const float* t_lb, const float* t_ub,
                         float* h_x3d, float* h_x2d, float* h_w2d, float* h_delta, float* h_cam, float* h_lb,
                         float* h_ub, float* h_grad, int B, int N, int dof, float z_min, float eps, float huber_eps,
                         void* stream);

/* Epilogue on the AMIS outputs -- the step AFTER the path in every caller of monte_carlo_forward (one pass over the
 * object-major log-weights instead of a dozen torch ops on (M, B) views):
 *   lse (B)        = logsumexp_m logw[b, m]      -- `loss_pred` of MonteCarloPoseLoss.forward
 *                    (EPro-PnP-6DoF/lib/models/monte_carlo_pose_loss.py:27-28, EPro-PnP-Det/epropnp_det/models/losses/
 *                    monte_carlo_pose_loss.py:21-22)
 *   loss (B)       = cost_target[b] + lse[b], NaN replaced by 0 (same files :30-31 / :24-25); cost_target [opt]
 *   weights (B, M) = softmax_m logw[b, :]        -- deform_pnp_head.py:524
 *   score_te (B)   = sum_m weights[b, m] * clamp((2.5 - log2 ||(x, z)_{b,m} - (x, z)_opt,b||) / 4, 0, 1)
 *                    -- the Monte-Carlo 'te' score, deform_pnp_head.py:533-536; needs pose_samples (B, M, D), pose_opt (B, D)
 * Every output is [opt]; at least one must be given.                                                              */
int epnp_mc_epilogue_f32(const float* logw /*(B,M)*/, const float* pose_samples, const float* pose_opt,
                         const float* cost_target, float* lse, float* loss, float* weights, float* score_te,
                         int B, int M, int dof, void* stream);
/* Backward of lse: grad_logw (B, M) = grad_lse[b] * exp(logw[b, m] - lse[b]), exactly 0 where grad_lse[b] == 0.     */
int epnp_mc_lse_backward_f32(const float* logw, const float* lse, const float* grad_lse, float* grad_logw,
                             int B, int M, void* stream);

/* Same as epnp_lm_amis_fused_f32 with HOST buffers (pinned for full speed): copies the inputs to
 * the caller-provided device workspace, runs the fused kernel and copies the results back, all on
 * `stream`, in `n_chunks` object chunks through a copy-in / solve / copy-out pipeline (helper streams owned by
 * the calling host thread, created on first use -- the only resource the library keeps).  n_chunks = 0 cuts the
 * batch at whole waves of resident CTAs (SMs x CTAs per SM objects per chunk, as few waves per chunk as the limit of
 * 64 chunks allows); n_chunks >= 1 asks for that many equal chunks (bench.py uses 8 for B = 4096, three calls in
 * flight).
 * workspace: device memory of at least epnp_fused_workspace_bytes(B, N, p) bytes.
 * Outputs [opt] as above (pose_samples_host may be NULL to skip the largest copy).              */
size_t epnp_fused_workspace_bytes(int B, int N, const EpnpParams* p);
int epnp_lm_amis_fused_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                                const float* cam_mats_host, const float* lb_host, const float* ub_host,
                                const float* delta_host, const float* pose_init_host,
                                uint64_t seed, uint32_t obj_offset,
                                float* pose_opt_host, float* pose_cov_host, float* cost_host,
                                float* pose_samples_host, float* logw_host,
                                void* workspace, size_t workspace_bytes, int n_chunks,
                                int B, int N, const EpnpParams* p, void* stream);

/* epnp_lm_amis_fused_host_f32 for objects of up to epnp_max_points_split(dof, M, I) points: the same arguments plus
 * cluster_ctas; each chunk runs epnp_lm_amis_fused_split_f32 (with obj_offset + the chunk's first object), so the
 * results equal that call's on the same inputs bit for bit, whatever the chunking.  The workspace is the same
 * epnp_fused_workspace_bytes(B, N, p).  n_chunks = 0 cuts the batch at whole waves of co-resident clusters
 * (cudaOccupancyMaxActiveClusters objects), at most 64 chunks.  Every refusal -- EPNP_ERR_TOO_MANY_POINTS above the
 * split limit, EPNP_ERR_BAD_ARG for a cluster size outside [epnp_split_ctas, 8], EPNP_ERR_UNSUPPORTED where the
 * cluster cannot be co-scheduled -- comes before any copy is enqueued.                                            */
int epnp_lm_amis_fused_split_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                                      const float* cam_mats_host, const float* lb_host, const float* ub_host,
                                      const float* delta_host, const float* pose_init_host,
                                      uint64_t seed, uint32_t obj_offset,
                                      float* pose_opt_host, float* pose_cov_host, float* cost_host,
                                      float* pose_samples_host, float* logw_host,
                                      void* workspace, size_t workspace_bytes, int n_chunks,
                                      int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);

/* The initialiser of a host-buffer solve from scratch (epnp_solve_host_f32): where LMSolver.solve gets its start
 * when no pose_init is given (levenberg_marquardt.py:113-124, init_solver.solve).
 *   EPNP_INIT_RSLM: RSLMSolver (levenberg_marquardt.py:271-353) -- epnp_rslm_draw_f32 with `seed` (the layer's
 *     rslm_seed, drawn apart from the AMIS seed) and rslm.eps, then epnp_rslm_f32 with `rslm` as its parameters
 *     (RSLMSolver(num_iter=..., **kwargs) has its own lm_iter, fast_mode, eps, z_min ...; rslm.dof must equal the
 *     solve's dof).  num_proposals = P, num_points = n.
 *   EPNP_INIT_EPNP: EPnPSolver of the 6DoF test loop (EPro-PnP-6DoF/lib/test.py:178-194) -- epnp_epnp_init_f32 with
 *     conf_quantile; dof 6 only.
 * Fields a kind does not use are ignored; the reserved ones keep the layout explicit (sizeof = 96 on every ABI).   */
enum { EPNP_INIT_RSLM = 1, EPNP_INIT_EPNP = 2 };
typedef struct EpnpInit {
    int32_t    kind;                /* EPNP_INIT_RSLM or EPNP_INIT_EPNP                          */
    int32_t    num_proposals;       /* RSLMSolver.num_proposals (P)                               */
    int32_t    num_points;          /* RSLMSolver.num_points (n)                                  */
    int32_t    reserved0;
    uint64_t   seed;                /* Philox seed of the RSLM draw                               */
    float      conf_quantile;       /* EPnP: keep the points with confidence >= this quantile     */
    int32_t    reserved1;
    EpnpParams rslm;                /* the RSLM solver's own parameters                          */
} EpnpInit;

/* Host-buffer solve from a given pose or from scratch, in the chunked copy-in / solve / copy-out pipeline of
 * epnp_lm_amis_fused_host_f32 (same helper streams, n_chunks rule, obj_offset and outputs).  It replaces the two
 * default inference paths of the reference, which have no AMIS:
 *   Det inference (EPro-PnP-Det/configs/epropnp_det_v1b_220411.py:158-160, deform_pnp_head.py:520-527): RSLM
 *     (P = 64, n = 16, 3 iterations), then LM with 5 iterations in fast mode -- init = RSLM, p->mc_samples = 0;
 *   6DoF test (EPro-PnP-6DoF/lib/test.py:91-96,178-211): EPnP on the points kept by the confidence quantile, then
 *     LMSolver(dof=6, num_iter=3) in fast mode -- init = EPNP, p->mc_samples = 0.
 * Start: exactly one of pose_init_host and init (EPNP_ERR_BAD_ARG for both or neither).
 * p->mc_samples = 0: LM only (EProPnP.forward / LMSolver.forward): epnp_lm_solve_f32 per chunk; logw_host and
 *   pose_samples_host must be NULL; pose_cov_host and cost_host stay optional under epnp_lm_solve_f32's rule (fast
 *   mode with lm_iter = 0 has none).
 * p->mc_samples > 0: LM + AMIS (monte_carlo_forward): epnp_lm_amis_fused_f32 per chunk; logw_host required.
 * Per chunk, on its compute stream after its copy-in: the RSLM draw (with obj_offset + the chunk's first object, so
 * the results never depend on the chunking) and the RSLM solve, or the EPnP initialisation; then LM or LM + AMIS.  The
 * results equal that composition of device calls on the same inputs bit for bit.
 * workspace: device memory of at least epnp_solve_workspace_bytes(B, N, p, init) bytes (init = NULL: pose_init given;
 * 0 for arguments no call takes).  Every refusal comes before the first copy, and is the refusal, with its code, that
 * the composed device calls make -- EPnP with dof 4 and an RSLM spec of another dof are EPNP_ERR_BAD_ARG.
 * n_chunks = 0 cuts the batch at whole waves of the AMIS kernel, or, with mc_samples = 0, of the initialiser's kernel
 * (one chunk for LM alone from a given pose).                                                                       */
size_t epnp_solve_workspace_bytes(int B, int N, const EpnpParams* p, const EpnpInit* init);
int epnp_solve_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                        const float* cam_mats_host, const float* lb_host, const float* ub_host,
                        const float* delta_host, const float* pose_init_host /*[opt]*/, const EpnpInit* init /*[opt]*/,
                        uint64_t seed, uint32_t obj_offset,
                        float* pose_opt_host, float* pose_cov_host, float* cost_host,
                        float* pose_samples_host, float* logw_host,
                        void* workspace, size_t workspace_bytes, int n_chunks,
                        int B, int N, const EpnpParams* p, void* stream);

/* epnp_solve_host_f32 for objects of up to epnp_max_points_split points: every stage that has a split form takes it at
 * any N -- epnp_rslm_split_f32 or epnp_epnp_init_split_f32, then epnp_lm_amis_fused_split_f32 (epnp_lm_solve_f32 takes
 * any N) -- and the results equal that composition bit for bit.  cluster_ctas = 0: each stage picks its own automatic
 * C; otherwise every split stage uses that C, which must then lie in every stage's range.  EPNP_ERR_UNSUPPORTED where
 * a stage's cluster cannot be co-scheduled; n_chunks = 0 cuts at whole waves of co-resident clusters.              */
int epnp_solve_split_host_f32(const float* x3d_host, const float* x2d_host, const float* w2d_host,
                              const float* cam_mats_host, const float* lb_host, const float* ub_host,
                              const float* delta_host, const float* pose_init_host, const EpnpInit* init,
                              uint64_t seed, uint32_t obj_offset,
                              float* pose_opt_host, float* pose_cov_host, float* cost_host,
                              float* pose_samples_host, float* logw_host,
                              void* workspace, size_t workspace_bytes, int n_chunks,
                              int B, int N, const EpnpParams* p, int cluster_ctas, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EPROPNP_B200_H */
