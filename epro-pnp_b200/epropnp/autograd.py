"""Autograd bridge for the differentiable outputs of the layer (reference epropnp.py:108-113):

    cost_init                       d/d(x3d, x2d, w2d, delta)   native kernel (epnp_cost_backward_f32)
                                    d/d pose_init               native kernel (epnp_cost_pose_backward_f32)
    pose_sample_logweights          = -cost(samples) - mixture density; only the cost term carries gradient
                                    (samples and proposals are built under no_grad, epropnp.py:139-140,172-179)
                                    -> same native kernel, upstream gradient -dL/dlogw
    evaluate_pnp(out_cost=True)     the same two kernels (correspondences / delta, poses)
    cost_init, logweights, evaluate_pnp   d/d(cam_mats, lb, ub)   native kernel (epnp_cost_camera_backward_f32)
    evaluate_pnp(out_residual / out_jacobian [, out_cost])   d/d(x3d, x2d, w2d, delta, pose, cam_mats, lb, ub)
                                    native kernel (epnp_evaluate_backward_f32), hence LMSolver.gn_step under autograd;
                                    first order only (a second backward raises)
    pose_opt_plus                   one un-damped Gauss-Newton step at the (detached) solution; differentiated
                                    by torch autograd through `PerspectiveCamera.project` + `HuberPnPCost.compute`
                                    (a single evaluation, levenberg_marquardt.py:243-253 -- not the iterated path),
                                    or, with EPNP_NATIVE_GN_STEP=1, by the native kernels epnp_gn_plus_backward_f32
                                    and, for cam_mats / lb / ub, epnp_gn_plus_camera_backward_f32

Objects with more points than one SM holds (N above epnp_max_points: about 5,400 for the AMIS loop at M = 512, 7,000
for the cost, the pose_opt_plus backward and the EPnP initialiser) take the cluster-split kernels (fused_forward,
stacked_cost, gn_plus_backward, epnp_init), up to epnp_max_points_split; at or below those limits nothing changes.  The
Monte-Carlo cost backward kernel streams the points, so it serves both; the pose_opt_plus forward (the LM kernel) streams
them too; the pose and camera backwards have split forms of their own (native.cost_pose_backward,
native.cost_camera_backward and native.gn_plus_camera_backward choose).  RSLM init takes its split
form (rslm_solve) only when the solver was built with RSLMSolver(cluster_split=True), up to min(epnp_max_points_split,
the native draw's own limit: 53,504 points at n = 16); by default it refuses objects above the resident limit.

Gradients w.r.t. poses (pose_init, stacked hypotheses) are those of the rotation the forward calls use, with respect to
the raw pose components; pose_opt, the samples and the solver's start carry none (reference epropnp.py:139-140).

The forward calls and their formulas are the epropnp custom operators of epropnp_b200.ops (register_autograd), one path
for eager calls, torch.compile and torch.export; the functions below give them the layer's camera / cost objects and
cast to the caller's dtype.  The operators' implementations take the resident or split call through the helpers here.
"""
import functools
import os

import torch

from epropnp_b200 import native, ops


@functools.lru_cache(maxsize=None)
def _resident_limit(dof, mc_samples, mc_iter):
    return native.max_points(dof, mc_samples, mc_iter)


def fused_forward(prob, pose_start, params, **kw):
    """native.lm_amis_fused, or its cluster-split form when the objects' points do not fit one SM."""
    split = prob.N > _resident_limit(params.dof, params.mc_samples, params.mc_iter)
    return (native.lm_amis_fused_split if split else native.lm_amis_fused)(prob, pose_start, params, **kw)


def stacked_cost(prob, poses, dof, z_min):
    """native.evaluate_cost, or its cluster-split form when the objects' points do not fit one SM."""
    split = prob.N > _resident_limit(dof, 0, 0)
    return (native.evaluate_cost_split if split else native.evaluate_cost)(prob, poses, dof, z_min)


def gn_plus_backward(prob, pose, grad_pose_plus, dof, z_min, eps, huber_eps, want):
    """native.gn_plus_backward, or its cluster-split form when the objects' points do not fit one SM."""
    split = prob.N > _resident_limit(dof, 0, 0)
    return (native.gn_plus_backward_split if split else native.gn_plus_backward)(
        prob, pose, grad_pose_plus, dof, z_min, eps, huber_eps, want=want)


def rslm_solve(prob, inds, start, params, allow_split):
    """native.rslm, or, when `allow_split` is set and the objects' points do not fit one SM, its cluster-split form.
    Without `allow_split` such objects are refused as before (RSLMSolver's cluster_split keyword)."""
    split = allow_split and prob.N > _resident_limit(params.dof, 0, 0)
    return (native.rslm_split if split else native.rslm)(prob, inds, start, params)


def epnp_init(x3d, x2d, w2d, cam_mats, conf_quantile):
    """native.epnp_init, or its cluster-split form when the objects' points do not fit one SM."""
    split = x3d.shape[1] > _resident_limit(6, 0, 0)
    return (native.epnp_init_split if split else native.epnp_init)(x3d, x2d, w2d, cam_mats, conf_quantile)


def _problem_args(x3d, x2d, w2d, camera, cost_fun):
    """The seven problem arguments of the epropnp operators for a camera and a cost object (ops.problem_args)."""
    return ops.problem_args(x3d, x2d, w2d, camera.cam_mats, camera.lb, camera.ub, cost_fun.delta)


def evaluate_autograd(x3d, x2d, w2d, pose, camera, cost_fun, clip_jac, want_r, want_j, want_c):
    """residual (*, B, 2N) | None, cost (*, B) | None, jacobian (*, B, 2N, dof) | None of pose hypotheses (*, B, D), with
    autograd w.r.t. x3d / x2d / w2d / cost_fun.delta / pose / cam_mats / lb / ub (first order only)."""
    dof = 4 if pose.size(-1) == 4 else 6
    lead, B, N = pose.shape[:-1], x3d.shape[0], x3d.shape[1]
    r, c, j = ops.evaluate_full(*_problem_args(x3d, x2d, w2d, camera, cost_fun), pose.reshape(-1, B, pose.size(-1)),
                                dof, float(camera.z_min), float(getattr(cost_fun, "eps", 1e-10)), bool(clip_jac),
                                want_r, want_j, want_c)
    dt = x3d.dtype
    return (r.to(dt).reshape(lead + (2 * N,)) if want_r else None, c.to(dt).reshape(lead) if want_c else None,
            j.to(dt).reshape(lead + (2 * N, dof)) if want_j else None)


def evaluate_cost_autograd(x3d, x2d, w2d, pose, camera, cost_fun):
    """cost (*, B) of pose hypotheses with autograd w.r.t. x3d / x2d / w2d / cost_fun.delta / pose / cam_mats / lb /
    ub."""
    dof = 4 if pose.size(-1) == 4 else 6
    lead = pose.shape[:-1]
    B = x3d.shape[0]
    cost = ops.evaluate_cost(*_problem_args(x3d, x2d, w2d, camera, cost_fun), pose.reshape(-1, B, pose.size(-1)), dof,
                             float(camera.z_min))
    return cost.to(x3d.dtype).reshape(lead)


def monte_carlo_autograd(x3d, x2d, w2d, camera, cost_fun, pose_start, pose_init, params, noise, seed, want_cost,
                         want_plus=False, want_cost_init=False):
    """The fused LM + AMIS operator from pose_start; `params` an (ints, floats) pair (ops.param_lists).
    -> pose_opt, cost | None, pose_opt_plus | None, pose_samples (B, M, D), logw (B, M) [differentiable],
    cost_init | None [differentiable when pose_init is given: the cost at pose_init]."""
    noise = (None,) * 3 if noise is None else noise
    pose_opt, cost, plus, cost_init, samples, logw = ops.lm_amis_fused(
        *_problem_args(x3d, x2d, w2d, camera, cost_fun), pose_start.detach(), pose_init, *noise, *ops.seed_args(seed),
        params[0], params[1], bool(want_cost), bool(want_plus), bool(want_cost_init))
    dt = x3d.dtype
    has_ci = pose_init is not None or want_cost_init
    return (pose_opt.to(dt), cost.to(dt) if want_cost else None, plus.to(dt) if want_plus else None, samples.to(dt),
            logw.to(dt), cost_init.to(dt) if has_ci else None)


class _PosePlus(torch.autograd.Function):
    """pose (+) gn_step(pose) with a native backward (epnp_gn_plus_backward_f32, or its split form above the resident
    limit; epnp_gn_plus_camera_backward_f32 for the camera): the eager form of the lm_solve operator's pose_opt_plus
    formula, over the same operator and the same backward (ops.gn_plus_grads), kept as a Function of its own so that the
    graph names it.  Under torch.compile pose_plus_autograd calls the operator itself.  `params` an EpnpParams or an
    (ints, floats) pair; delta, lb and ub tensors or Python floats (those get no gradient)."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, pose, params, huber_eps):
        ints, floats = ops.param_lists(params)
        prob = ops.problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        plus = ops.lm_solve(*prob, pose, ints, floats, False, False, True)[3]
        ctx.save_for_backward(*(t for t in prob if t is not None), pose)
        ctx.bounded = prob[4] is not None
        ctx.consts = (ints[0], floats[0], floats[6], float(huber_eps))              # dof, z_min, eps, huber_eps
        return plus.to(x3d.dtype)

    @staticmethod
    def backward(ctx, grad_plus):
        saved = list(ctx.saved_tensors)
        pose = saved.pop()
        x3d, x2d, w2d, cam_mats = saved[:4]
        lb, ub = (saved[4], saved[5]) if ctx.bounded else (None, None)
        prob = (x3d, x2d, w2d, cam_mats, lb, ub, saved[-1])
        n = ctx.needs_input_grad
        g = ops.gn_plus_grads(prob, pose, grad_plus, *ctx.consts, (n[0], n[1], n[2], n[4], n[5], n[6], n[3]))
        return g[0], g[1], g[2], g[6], g[3], g[4], g[5], None, None, None


def native_gn_step_enabled():
    """pose_opt_plus is differentiated by the native kernel (epnp_gn_plus_backward_f32; validated on the GPU against the
    float64 composite and the reference's own autograd).  EPNP_NATIVE_GN_STEP=0 selects the torch-autograd composite of
    PerspectiveCamera.project + HuberPnPCost.compute instead (exact in float64; used by the CPU tests and for A/B timing)."""
    return os.environ.get("EPNP_NATIVE_GN_STEP", "1") not in ("", "0")


def pose_plus_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun):
    """Differentiable pose (+) one un-damped Gauss-Newton step at the detached `pose` (LMSolver.forward :66-68)."""
    if not native_gn_step_enabled():
        return solver.pose_add(pose, gn_step_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun), camera)
    params = solver.param_lists(camera, cost_fun, False, lm_iter=0)     # evaluate the step at `pose` itself
    delta = cost_fun.delta
    if torch.compiler.is_compiling():
        plus = ops.lm_solve(*_problem_args(x3d, x2d, w2d, camera, cost_fun), pose.detach(), *params, False, False,
                            True)[3]
        return plus.to(x3d.dtype)
    return _PosePlus.apply(x3d, x2d, w2d, delta if torch.is_tensor(delta) else float(delta), camera.cam_mats,
                           camera.lb, camera.ub, pose.detach(), params, float(getattr(cost_fun, "eps", 1e-10)))


def gn_step_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun):
    """Differentiable un-damped Gauss-Newton increment at a detached pose (levenberg_marquardt.py:243-253)."""
    pose = pose.detach()
    x2d_proj, jac_cam = camera.project(x3d, pose, out_jac=True, clip_jac=True)
    residual, _, jac = cost_fun.compute(x2d_proj, x2d, w2d, jac_cam=jac_cam, out_residual=True, out_jacobian=True)
    jac_t = jac.transpose(-1, -2)
    jtj = jac_t @ jac + torch.eye(solver.dof, device=jac.device, dtype=jac.dtype) * solver.eps
    return -torch.linalg.solve(jtj, jac_t @ residual.unsqueeze(-1)).squeeze(-1)
