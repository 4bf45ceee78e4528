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
                                    first order only (once_differentiable)
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
        if like.numel() == 1 and g.numel() != 1:
            out.append(g.sum().reshape(like.shape))
        else:       # a broadcast input, such as a (B, N, 1) weight, receives the sum over the axes it was expanded along
            out.append(g.reshape(like.shape) if g.numel() == like.numel() else g.sum_to_size(like.shape))
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
        ctx.pose_like = cost_init_pose if cost_init_pose is not None and cost_init_pose.requires_grad else None
        ctx.cam_like = _camera_like(prob, cam_mats, lb, ub)
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
        grads = (None,) * 4
        if any(ctx.needs):
            grads = native.cost_backward(prob, ctx.dof, ctx.z_min, ctx.samples, -g_logw.contiguous(), poses_b, grad_b,
                                         want=ctx.needs)
        gx3d, gx2d, gw2d, gdel = _grads_to(ctx.in_like, grads)
        gpose = None
        if ctx.pose_like is not None and poses_b is not None:
            gpose = _pose_grad_to(ctx.pose_like, native.cost_pose_backward(prob, ctx.dof, ctx.z_min, poses_b, grad_b)[:, 0])
        gcam, glb, gub = _camera_grads(ctx.cam_like, lambda want: native.cost_camera_backward(
            prob, ctx.dof, ctx.z_min, ctx.samples, -g_logw.contiguous(), poses_b, grad_b, want=want))
        return gx3d, gx2d, gw2d, gdel, gcam, glb, gub, None, gpose, None, None, None, None, None


class _CostOnly(torch.autograd.Function):
    """evaluate_pnp(out_cost=True) with gradients w.r.t. the correspondences / delta and the poses (S, B, D)."""

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
        ctx.pose_like = poses if poses.requires_grad else None
        ctx.cam_like = _camera_like(prob, cam_mats, lb, ub)
        return cost.to(x3d.dtype)

    @staticmethod
    def backward(ctx, g_cost):
        g_cost = g_cost.transpose(0, 1).contiguous()                            # object-major (B, S)
        grads = (None,) * 4
        if any(ctx.needs):
            grads = native.cost_backward(ctx.prob, ctx.dof, ctx.z_min, ctx.poses, g_cost, want=ctx.needs)
        gx3d, gx2d, gw2d, gdel = _grads_to(ctx.in_like, grads)
        gpose = None
        if ctx.pose_like is not None:
            gpose = _pose_grad_to(ctx.pose_like,
                                  native.cost_pose_backward(ctx.prob, ctx.dof, ctx.z_min, ctx.poses, g_cost).transpose(0, 1))
        gcam, glb, gub = _camera_grads(ctx.cam_like, lambda want: native.cost_camera_backward(
            ctx.prob, ctx.dof, ctx.z_min, ctx.poses, g_cost, want=want))
        return gx3d, gx2d, gw2d, gdel, gcam, glb, gub, gpose, None, None


class _Evaluate(torch.autograd.Function):
    """evaluate_pnp's residual / cost / Jacobian at poses (S, B, D) with a native backward (epnp_evaluate_backward_f32)
    with respect to the correspondences, delta, the poses and the camera.  The forward is the no-grad path's
    native.evaluate_full call, stacked poses replicating the problem as there, so its values are the same bits."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, poses, dof, z_min, huber_eps, clip_jac, want_r, want_j,
                want_c):
        ctx.set_materialize_grads(False)                 # an output the loss does not use costs the backward nothing
        prob = native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        S, B, N = poses.shape[0], prob.B, prob.N
        run = prob
        if S != 1:
            rep = lambda t: t.unsqueeze(0).expand((S,) + t.shape).reshape((S * B,) + t.shape[1:])
            run = native.Problem(rep(prob.x3d), rep(prob.x2d), rep(prob.w2d), rep(prob.cam),
                                 None if prob.lb is None else rep(prob.lb), None if prob.ub is None else rep(prob.ub),
                                 rep(prob.delta))
        r, c, j = native.evaluate_full(run, poses.reshape(-1, poses.size(-1)), dof, z_min, huber_eps, clip_jac, want_r,
                                       want_j, want_c)
        ctx.prob, ctx.poses, ctx.consts = prob, poses.detach(), (dof, z_min, huber_eps, clip_jac)
        ctx.in_like = (x3d, x2d, w2d, delta if torch.is_tensor(delta) else None)
        ctx.needs = (x3d.requires_grad, x2d.requires_grad, w2d.requires_grad,
                     torch.is_tensor(delta) and delta.requires_grad)
        ctx.pose_like = poses if poses.requires_grad else None
        ctx.cam_like = _camera_like(prob, cam_mats, lb, ub)
        dt, empty = x3d.dtype, x3d.new_zeros(0)
        out = (r.reshape(S, B, 2 * N).to(dt) if want_r else empty, c.reshape(S, B).to(dt) if want_c else empty,
               j.reshape(S, B, 2 * N, dof).to(dt) if want_j else empty)
        ctx.mark_non_differentiable(*(t for t, w in zip(out, (want_r, want_c, want_j)) if not w))
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_res, g_cost, g_jac):
        dof, z_min, huber_eps, clip_jac = ctx.consts
        ups = [g if g is not None and g.numel() else None for g in (g_res, g_jac, g_cost)]
        cam_want = tuple(t is not None for t in ctx.cam_like)
        want = ctx.needs + (ctx.pose_like is not None,) + cam_want
        if all(g is None for g in ups) or not any(want):
            return (None,) * 15
        grads = native.evaluate_backward(ctx.prob, ctx.poses, dof, z_min, huber_eps, clip_jac, *ups, want=want)
        gx3d, gx2d, gw2d, gdel = _grads_to(ctx.in_like, grads[:4])
        gpose = None if ctx.pose_like is None else _pose_grad_to(ctx.pose_like, grads[4])
        gcam, glb, gub = _camera_grads(ctx.cam_like, lambda _: grads[5:])
        return gx3d, gx2d, gw2d, gdel, gcam, glb, gub, gpose, None, None, None, None, None, None, None


def evaluate_autograd(x3d, x2d, w2d, pose, camera, cost_fun, clip_jac, want_r, want_j, want_c):
    """residual (*, B, 2N) | None, cost (*, B) | None, jacobian (*, B, 2N, dof) | None of pose hypotheses (*, B, D), with
    autograd w.r.t. x3d / x2d / w2d / cost_fun.delta / pose / cam_mats / lb / ub."""
    dof = 4 if pose.size(-1) == 4 else 6
    lead, B, N = pose.shape[:-1], x3d.shape[0], x3d.shape[1]
    r, c, j = _Evaluate.apply(x3d, x2d, w2d, _delta_tensor(cost_fun.delta, x2d), camera.cam_mats, camera.lb, camera.ub,
                              pose.reshape(-1, B, pose.size(-1)), dof, float(camera.z_min),
                              float(getattr(cost_fun, "eps", 1e-10)), bool(clip_jac), want_r, want_j, want_c)
    return (r.reshape(lead + (2 * N,)) if want_r else None, c.reshape(lead) if want_c else None,
            j.reshape(lead + (2 * N, dof)) if want_j else None)


def _pose_grad_to(like, g):
    """Native pose gradient -> dtype and shape of the pose tensor it belongs to."""
    return g.to(like.dtype).reshape(like.shape)


def _camera_like(prob, cam_mats, lb, ub):
    """The camera inputs that require grad (cam_mats, lb, ub; None elsewhere).  Python-float bounds get no gradient, and
    neither does a bound while the other is missing: the projection is then not clamped."""
    grad = lambda t: torch.is_tensor(t) and t.requires_grad
    bounded = prob.lb is not None
    return (cam_mats if grad(cam_mats) else None, lb if bounded and grad(lb) else None,
            ub if bounded and grad(ub) else None)


def _camera_grads(like, run):
    """run(want) -> native (B, 3, 3) / (B, 2) / (B, 2) camera gradients, each reduced to the dtype and shape of the
    tensor the caller passed: a (3, 3) camera or a (2,) bound shared by every object receives the sum over objects (an
    expanded one receives them per object; autograd sums them through the expand)."""
    want = tuple(t is not None for t in like)
    if not any(want):
        return None, None, None
    out = []
    for t, g in zip(like, run(want)):
        if t is None:
            out.append(None)
            continue
        g = g.to(t.dtype)
        out.append(g.sum_to_size(t.shape) if t.dim() else g.sum())
    return tuple(out)


def evaluate_cost_autograd(x3d, x2d, w2d, pose, camera, cost_fun):
    """cost (*, B) of pose hypotheses with autograd w.r.t. x3d / x2d / w2d / cost_fun.delta / pose."""
    dof = 4 if pose.size(-1) == 4 else 6
    lead = pose.shape[:-1]
    B = x3d.shape[0]
    cost = _CostOnly.apply(x3d, x2d, w2d, _delta_tensor(cost_fun.delta, x2d), camera.cam_mats, camera.lb, camera.ub,
                           pose.reshape(-1, B, pose.size(-1)), dof, float(camera.z_min))
    return cost.reshape(lead)


def monte_carlo_autograd(x3d, x2d, w2d, camera, cost_fun, pose_start, pose_init, params, noise, seed, want_cost):
    """-> pose_opt, cost | None, pose_samples (B,M,D), logw (B,M) [differentiable], cost_init | None [differentiable]."""
    pose_opt, cost, samples, logw, cost_init = _MonteCarloForward.apply(
        x3d, x2d, w2d, _delta_tensor(cost_fun.delta, x2d), camera.cam_mats, camera.lb, camera.ub, pose_start.detach(),
        pose_init, params, noise, seed, bool(want_cost), float(camera.z_min))
    return pose_opt, (cost if want_cost else None), samples, logw, (cost_init if pose_init is not None else None)


class _PosePlus(torch.autograd.Function):
    """pose (+) gn_step(pose) with a native backward (epnp_gn_plus_backward_f32, or its split form above the resident
    limit)."""

    @staticmethod
    def forward(ctx, x3d, x2d, w2d, delta, cam_mats, lb, ub, pose, params, huber_eps):
        prob = native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
        plus = native.lm_solve(prob, pose, params, want_plus=True)["pose_opt_plus"]
        ctx.prob, ctx.pose, ctx.dof = prob, pose.detach(), params.dof
        ctx.consts = (float(params.z_min), float(params.eps), float(huber_eps))
        ctx.in_like = (x3d, x2d, w2d, delta if torch.is_tensor(delta) else None)
        ctx.needs = (x3d.requires_grad, x2d.requires_grad, w2d.requires_grad,
                     torch.is_tensor(delta) and delta.requires_grad)
        ctx.cam_like = _camera_like(prob, cam_mats, lb, ub)
        return plus.to(x3d.dtype)

    @staticmethod
    def backward(ctx, grad_plus):
        z_min, eps, huber_eps = ctx.consts
        grads = (None,) * 4
        if any(ctx.needs):
            grads = gn_plus_backward(ctx.prob, ctx.pose, grad_plus, ctx.dof, z_min, eps, huber_eps, ctx.needs)
        g3, g2, gw, gd = _grads_to(ctx.in_like, grads)
        gcam, glb, gub = _camera_grads(ctx.cam_like, lambda want: native.gn_plus_camera_backward(
            ctx.prob, ctx.pose, grad_plus, ctx.dof, z_min, eps, huber_eps, want=want))
        return g3, g2, gw, gd, gcam, glb, gub, None, None, None


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
