"""Autograd bridge for the differentiable outputs of the layer (reference epropnp.py:108-113):

    cost_init                       d/d(x3d, x2d, w2d, delta)   native kernel (epnp_cost_backward_f32)
    pose_sample_logweights          = -cost(samples) - mixture density; only the cost term carries gradient
                                    (samples and proposals are built under no_grad, epropnp.py:139-140,172-179)
                                    -> same native kernel, upstream gradient -dL/dlogw
    evaluate_pnp(out_cost=True)     same kernel
    pose_opt_plus                   one un-damped Gauss-Newton step at the (detached) solution; differentiated
                                    by torch autograd through `PerspectiveCamera.project` + `HuberPnPCost.compute`
                                    (a single evaluation, levenberg_marquardt.py:243-253 -- not the iterated path),
                                    or, with EPNP_NATIVE_GN_STEP=1, by the native kernel epnp_gn_plus_backward_f32

Objects with more points than one SM holds (N above epnp_max_points: about 5,400 for the AMIS loop at M = 512, 7,000
for the cost) take the cluster-split kernels (fused_forward, stacked_cost); at or below those limits nothing changes.
The backward kernel streams the points, so it serves both.

Gradients w.r.t. poses (pose_init / stacked hypotheses) are not provided: the reference's losses never use
them (pose_init is the ground truth, lib/train.py:178-180), and asking for them raises.
"""
import functools

import torch

from epropnp_b200 import native


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


def _delta_tensor(delta, ref):
    if torch.is_tensor(delta):
        return delta
    return ref.new_tensor(float(delta))


def _grads_to(like_list, grads):
    """Native gradients (B,N,3) / (B,N,2) / (B,N,2) / (B) -> dtype and shape of the inputs they belong to
    (a scalar / 1-element delta tensor receives the sum over objects)."""
    out = []
    for like, g in zip(like_list, grads):
        if like is None or g is None:
            out.append(None)
            continue
        g = g.to(like.dtype)
        out.append(g.sum().reshape(like.shape) if like.numel() == 1 and g.numel() != 1 else g.reshape(like.shape))
    return out


class _MonteCarloForward(torch.autograd.Function):
    """Fused LM + AMIS forward; backward = native Monte-Carlo cost gradient."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, pose_start, cost_init_pose, params, noise, seed,
                want_cost, z_min):
        prob = native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        out = fused_forward(prob, pose_start, params, noise=noise, seed=seed, want_cost=want_cost,
                            want_cost_init=False, want_cov=False)
        dof = params.dof
        cost_init = None
        if cost_init_pose is not None:
            cost_init = stacked_cost(prob, cost_init_pose.detach().unsqueeze(0), dof, z_min)[0]
        ctx.prob, ctx.dof, ctx.z_min = prob, dof, z_min
        ctx.samples = out["pose_samples"]
        ctx.cost_init_pose = None if cost_init_pose is None else cost_init_pose.detach()
        ctx.in_like = (x3d, x2d, w2d, delta if torch.is_tensor(delta) else None)
        ctx.needs = (x3d.requires_grad, x2d.requires_grad, w2d.requires_grad,
                     torch.is_tensor(delta) and delta.requires_grad)
        cost = out["cost"] if want_cost else x3d.new_zeros(0)
        ci = cost_init if cost_init is not None else x3d.new_zeros(0)
        dt = x3d.dtype
        # cast FIRST, then mark the tensors that are actually returned (for non-fp32 inputs .to() makes new tensors)
        pose_opt, cost, samples = out["pose_opt"].to(dt), cost.to(dt), out["pose_samples"].to(dt)
        ctx.mark_non_differentiable(pose_opt, cost, samples)
        return pose_opt, cost, samples, out["logw"].to(dt), ci.to(dt)

    @staticmethod
    def backward(ctx, g_pose, g_cost, g_samples, g_logw, g_cost_init):
        prob = ctx.prob
        B = prob.B
        if g_logw is None:
            g_logw = torch.zeros(B, ctx.samples.shape[1], device=prob.device)
        poses_b = grad_b = None
        if ctx.cost_init_pose is not None and g_cost_init is not None and g_cost_init.numel() == B:
            poses_b = ctx.cost_init_pose.reshape(B, 1, -1)
            grad_b = g_cost_init.reshape(B, 1)
        grads = native.cost_backward(prob, ctx.dof, ctx.z_min, ctx.samples, -g_logw.contiguous(), poses_b, grad_b,
                                     want=ctx.needs)
        gx3d, gx2d, gw2d, gdel = _grads_to(ctx.in_like, grads)
        return gx3d, gx2d, gw2d, gdel, None, None, None, None, None, None, None, None, None, None


class _CostOnly(torch.autograd.Function):
    """evaluate_pnp(out_cost=True) with gradients w.r.t. the correspondences / delta."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, poses, dof, z_min):
        prob = native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        S = poses.shape[0]
        cost = stacked_cost(prob, poses, dof, z_min)                            # (S, B)
        ctx.prob, ctx.dof, ctx.z_min = prob, dof, z_min
        ctx.poses = poses.detach().transpose(0, 1).contiguous()                 # object-major (B, S, D)
        ctx.in_like = (x3d, x2d, w2d, delta if torch.is_tensor(delta) else None)
        ctx.needs = (x3d.requires_grad, x2d.requires_grad, w2d.requires_grad,
                     torch.is_tensor(delta) and delta.requires_grad)
        return cost.to(x3d.dtype)

    @staticmethod
    def backward(ctx, g_cost):
        grads = native.cost_backward(ctx.prob, ctx.dof, ctx.z_min, ctx.poses, g_cost.transpose(0, 1).contiguous(),
                                     want=ctx.needs)
        gx3d, gx2d, gw2d, gdel = _grads_to(ctx.in_like, grads)
        return gx3d, gx2d, gw2d, gdel, None, None, None, None, None, None


def _no_pose_grad(pose):
    if torch.is_tensor(pose) and pose.requires_grad:
        raise NotImplementedError("gradients with respect to poses are not provided by the native EPro-PnP path "
                                  "(detach the pose; the reference's losses never differentiate through it)")


def evaluate_cost_autograd(x3d, x2d, w2d, pose, camera, cost_fun):
    """cost (*, B) of pose hypotheses with autograd w.r.t. x3d / x2d / w2d / cost_fun.delta."""
    _no_pose_grad(pose)
    dof = 4 if pose.size(-1) == 4 else 6
    lead = pose.shape[:-1]
    B = x3d.shape[0]
    cost = _CostOnly.apply(x3d, x2d, w2d, _delta_tensor(cost_fun.delta, x2d), camera.cam_mats, camera.lb, camera.ub,
                           pose.detach().reshape(-1, B, pose.size(-1)), dof, float(camera.z_min))
    return cost.reshape(lead)


def monte_carlo_autograd(x3d, x2d, w2d, camera, cost_fun, pose_start, pose_init, params, noise, seed, want_cost):
    """-> pose_opt, cost | None, pose_samples (B,M,D), logw (B,M) [differentiable], cost_init | None [differentiable]."""
    _no_pose_grad(pose_init)
    pose_opt, cost, samples, logw, cost_init = _MonteCarloForward.apply(
        x3d, x2d, w2d, _delta_tensor(cost_fun.delta, x2d), camera.cam_mats, camera.lb, camera.ub, pose_start.detach(),
        None if pose_init is None else pose_init.detach(), params, noise, seed, bool(want_cost), float(camera.z_min))
    return pose_opt, (cost if want_cost else None), samples, logw, (cost_init if pose_init is not None else None)


class _PosePlus(torch.autograd.Function):
    """pose (+) gn_step(pose) with a native backward (epnp_gn_plus_backward_f32)."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, pose, params, huber_eps):
        prob = native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        plus = native.lm_solve(prob, pose, params, want_plus=True)["pose_opt_plus"]
        ctx.prob, ctx.pose, ctx.dof = prob, pose.detach(), params.dof
        ctx.consts = (float(params.z_min), float(params.eps), float(huber_eps))
        ctx.in_like = (x3d, x2d, w2d, delta if torch.is_tensor(delta) else None)
        ctx.needs = (x3d.requires_grad, x2d.requires_grad, w2d.requires_grad,
                     torch.is_tensor(delta) and delta.requires_grad)
        return plus.to(x3d.dtype)

    @staticmethod
    def backward(ctx, grad_plus):
        z_min, eps, huber_eps = ctx.consts
        grads = native.gn_plus_backward(ctx.prob, ctx.pose, grad_plus, ctx.dof, z_min, eps, huber_eps, want=ctx.needs)
        g3, g2, gw, gd = _grads_to(ctx.in_like, grads)
        return g3, g2, gw, gd, None, None, None, None, None, None


def native_gn_step_enabled():
    """pose_opt_plus is differentiated by the native kernel (epnp_gn_plus_backward_f32; validated on the GPU against the
    float64 composite and the reference's own autograd).  EPNP_NATIVE_GN_STEP=0 selects the torch-autograd composite of
    PerspectiveCamera.project + HuberPnPCost.compute instead (exact in float64; used by the CPU tests and for A/B timing)."""
    import os
    return os.environ.get("EPNP_NATIVE_GN_STEP", "1") not in ("", "0")


def pose_plus_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun):
    """Differentiable pose (+) one un-damped Gauss-Newton step at the detached `pose` (LMSolver.forward :66-68)."""
    if not native_gn_step_enabled():
        return solver.pose_add(pose, gn_step_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun), camera)
    params = solver.native_params(camera, cost_fun, False)
    params.lm_iter = 0                                       # evaluate the step at `pose` itself
    delta = cost_fun.delta
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
