"""LMSolver / RSLMSolver with the reference's constructor and call signatures
(reference epropnp/levenberg_marquardt.py), executing on the native sm_90a kernels.

What runs where:
  * the K-iteration Levenberg-Marquardt (or Gauss-Newton `fast_mode`) loop, the pose covariance and
    the optional extra GN step are ONE kernel launch (epnp_lm_solve_f32): no per-iteration launches,
    no host round trips, no materialised (B, 2N, 6) Jacobian;
  * RSLMSolver: two launches -- the random subsets / start orientations (epnp_rslm_draw_f32), then refining and
    scoring all P hypotheses of every object (epnp_rslm_f32); with cluster_split=True, objects too large for one SM
    take epnp_rslm_split_f32 instead (refine, score on a thread-block cluster, select: three launches).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from epropnp_b200 import ops
from .autograd import _problem_args
from .builder import PNP, build_pnp
from .common import _needs_grad, evaluate_pnp, philox_seed, pnp_normalize, pnp_denormalize


def solve_wrapper(b, A):
    """A^-1 b with the reference's empty-batch convention (levenberg_marquardt.py:15-19)."""
    if A.numel() > 0:
        return torch.linalg.solve(A, b)
    return b + A.reshape_as(b)


@PNP.register_module()
class LMSolver(nn.Module):
    """Levenberg-Marquardt solver with a fixed number of iterations.

    4DoF pose = [x, y, z, yaw] (yaw about the Y axis); 6DoF pose = [x, y, z, w, i, j, k]."""

    def __init__(self, dof=4, num_iter=10, min_lm_diagonal=1e-6, max_lm_diagonal=1e32,
                 min_relative_decrease=1e-3, initial_trust_region_radius=30.0,
                 max_trust_region_radius=1e16, eps=1e-5, normalize=False, init_solver=None):
        super(LMSolver, self).__init__()
        self.dof = dof
        self.num_iter = num_iter
        self.min_lm_diagonal = min_lm_diagonal
        self.max_lm_diagonal = max_lm_diagonal
        self.min_relative_decrease = min_relative_decrease
        self.initial_trust_region_radius = initial_trust_region_radius
        self.max_trust_region_radius = max_trust_region_radius
        self.eps = eps
        self.normalize = normalize
        self.init_solver = build_pnp(init_solver)        # instance, None, or a config dict (detection-style configs)

    # ------------------------------------------------------------------ native parameter block
    def native_params(self, camera, cost_fun, fast_mode=False, **extra):
        """The solver's EpnpParams block (ctypes), as the C ABI takes it."""
        return ops.make_params(*self.param_lists(camera, cost_fun, fast_mode, **extra))

    def param_lists(self, camera, cost_fun, fast_mode=False, **extra):
        """The same block as the (ints, floats) lists the epropnp operators take (ops.param_lists; traceable)."""
        fields = dict(lm_iter=int(self.num_iter), fast_mode=int(bool(fast_mode)), z_min=float(camera.z_min),
                      min_lm_diagonal=float(self.min_lm_diagonal), max_lm_diagonal=float(self.max_lm_diagonal),
                      min_relative_decrease=float(self.min_relative_decrease),
                      initial_radius=float(self.initial_trust_region_radius),
                      max_radius=float(self.max_trust_region_radius), eps=float(self.eps),
                      huber_eps=float(getattr(cost_fun, "eps", 1e-10)))
        fields.update(extra)
        return ops.param_lists(None, self.dof, **fields)

    def _pose_dim(self):
        return 4 if self.dof == 4 else 7

    # ------------------------------------------------------------------ reference API
    def forward(self, x3d, x2d, w2d, camera, cost_fun, with_pose_opt_plus=False, pose_init=None,
                normalize_override=None, **kwargs):
        normalize = normalize_override if isinstance(normalize_override, bool) else self.normalize
        if normalize:
            transform, x3d, pose_init = pnp_normalize(x3d, pose_init, detach_transformation=True)
        delta = getattr(cost_fun, "delta", None)
        differentiable = with_pose_opt_plus and _needs_grad(x3d, x2d, w2d, delta, camera.cam_mats, camera.lb,
                                                            camera.ub)
        pose_opt, pose_cov, cost, pose_opt_plus = self._solve_impl(
            x3d, x2d, w2d, camera, cost_fun, pose_init=pose_init,
            with_pose_opt_plus=with_pose_opt_plus and not differentiable, **kwargs)
        if differentiable:       # y* (+) GN step, differentiable w.r.t. the correspondences (:66-68)
            from .autograd import pose_plus_autograd
            pose_opt_plus = pose_plus_autograd(self, x3d, x2d, w2d, pose_opt, camera, cost_fun)
        if normalize:
            pose_opt = pnp_denormalize(transform, pose_opt)
            if pose_cov is not None:
                raise NotImplementedError('Normalized covariance unsupported')
            if pose_opt_plus is not None:
                pose_opt_plus = pnp_denormalize(transform, pose_opt_plus)
        return pose_opt, pose_cov, cost, pose_opt_plus

    def solve(self, x3d, x2d, w2d, camera, cost_fun, pose_init=None, cost_init=None,
              with_pose_cov=False, with_cost=False, force_init_solve=False, fast_mode=False):
        """-> pose_opt (B, 4|7), pose_cov (B, dof, dof) | None, cost (B) | None."""
        return self._solve_impl(x3d, x2d, w2d, camera, cost_fun, pose_init=pose_init, cost_init=cost_init,
                                with_pose_cov=with_pose_cov, with_cost=with_cost,
                                force_init_solve=force_init_solve, fast_mode=fast_mode)[:3]

    def _starting_pose(self, x3d, x2d, w2d, camera, cost_fun, pose_init, cost_init, force_init_solve, fast_mode):
        """pose the LM iterations start from (levenberg_marquardt.py:115-130)."""
        if pose_init is not None and not force_init_solve:
            return pose_init.detach()
        assert self.init_solver is not None
        if pose_init is None:
            return self.init_solver.solve(x3d, x2d, w2d, camera, cost_fun, fast_mode=fast_mode)[0]
        if cost_init is None:
            cost_init = evaluate_pnp(x3d.detach(), x2d.detach(), w2d.detach(), pose_init.detach(), camera, cost_fun,
                                     out_cost=True)[1]
        pose_rs, _, cost_rs = self.init_solver.solve(x3d, x2d, w2d, camera, cost_fun, with_cost=True,
                                                     fast_mode=fast_mode)
        keep = (cost_init.detach() < cost_rs)[:, None]
        return torch.where(keep, pose_init.detach().to(pose_rs.dtype), pose_rs)

    @torch.no_grad()
    def _solve_impl(self, x3d, x2d, w2d, camera, cost_fun, pose_init=None, cost_init=None, with_pose_cov=False,
                    with_cost=False, force_init_solve=False, fast_mode=False, with_pose_opt_plus=False):
        num_obj = x2d.size(0)
        kw = dict(dtype=x2d.dtype, device=x2d.device)
        if num_obj == 0:
            return (torch.empty((0, self._pose_dim()), **kw),
                    torch.empty((0, self.dof, self.dof), **kw) if with_pose_cov else None,
                    torch.empty((0,), **kw) if with_cost else None,
                    torch.empty((0, self._pose_dim()), **kw) if with_pose_opt_plus else None)
        start = self._starting_pose(x3d, x2d, w2d, camera, cost_fun, pose_init, cost_init, force_init_solve, fast_mode)
        out = ops.lm_solve(*_problem_args(x3d, x2d, w2d, camera, cost_fun), start,
                           *self.param_lists(camera, cost_fun, fast_mode), with_pose_cov, with_cost, with_pose_opt_plus)
        cast = lambda t, want: t.to(x2d.dtype) if want else None
        return (cast(out[0], True), cast(out[1], with_pose_cov), cast(out[2], with_cost),
                cast(out[3], with_pose_opt_plus))

    def gn_step(self, x3d, x2d, w2d, pose, camera, cost_fun):
        """Undamped Gauss-Newton increment -(J^T J + eps I)^-1 J^T r at `pose` (levenberg_marquardt.py:243-253)."""
        residual, _, jac = evaluate_pnp(x3d, x2d, w2d, pose, camera, cost_fun, out_jacobian=True, out_residual=True)
        jac_t = jac.transpose(-1, -2)
        jtj = jac_t @ jac + torch.eye(self.dof, device=jac.device, dtype=jac.dtype) * self.eps
        return -solve_wrapper(jac_t @ residual.unsqueeze(-1), jtj).squeeze(-1)

    def _lm_iter(self, pose_opt, jac, residual, cost, jac_new, residual_new, cost_new, step_is_successful, radius,
                 decrease_factor, evaluate_fun, camera):
        """One trust-region iteration on caller-owned state, all tensors updated IN PLACE (reference :192-241; same
        argument list).  `solve` does not call this -- its iterations run inside lm_warp_kernel (pnp_math.cuh lm_adopt /
        lm_propose / lm_update) -- it is kept as a stand-alone torch restatement for code that drives the solver step by
        step.  evaluate_fun(pose=, out_jacobian=, out_residual=, out_cost=) fills the given buffers, as
        functools.partial(evaluate_pnp, ...) does.  Steps: adopt the last accepted evaluation; damped normal equations
        (J^T J + clamp(diag) / radius + eps) step = -J^T r; evaluate the candidate; accept when the cost falls by at
        least min_relative_decrease of what the quadratic model promised; grow / shrink the radius (Ceres' rule)."""
        took = step_is_successful
        jac.copy_(torch.where(took[:, None, None], jac_new, jac))
        residual.copy_(torch.where(took[:, None], residual_new, residual))
        cost.copy_(torch.where(took, cost_new, cost))
        jac_t = jac.transpose(-1, -2)
        jtj = jac_t @ jac
        gradient = jac_t @ residual.unsqueeze(-1)
        diag = torch.diagonal(jtj, dim1=-2, dim2=-1)
        damping = diag.clamp(min=self.min_lm_diagonal, max=self.max_lm_diagonal) / radius[:, None] + self.eps
        step = -solve_wrapper(gradient, jtj + torch.diag_embed(damping))
        pose_new = self.pose_add(pose_opt, step.squeeze(-1), camera)
        evaluate_fun(pose=pose_new, out_jacobian=jac_new, out_residual=residual_new, out_cost=cost_new)
        predicted = -(step.transpose(-1, -2) @ (0.5 * (jtj @ step) + gradient)).flatten()
        gain = (cost - cost_new) / predicted
        took.copy_((gain >= self.min_relative_decrease) & (predicted > 0.0))
        pose_opt.copy_(torch.where(took[:, None], pose_new, pose_opt))
        grown = radius / (1.0 - (2.0 * gain - 1.0) ** 3).clamp(min=1.0 / 3.0)
        radius.copy_(torch.where(took, grown, radius).clamp(max=self.max_trust_region_radius, min=self.eps))
        radius.copy_(torch.where(took, radius, radius / decrease_factor))
        decrease_factor.copy_(torch.where(took, torch.full_like(decrease_factor, 2.0), decrease_factor * 2.0))

    def pose_add(self, pose_opt, step, camera):
        """pose (+) step; rotations are updated on the unit-quaternion manifold (levenberg_marquardt.py:255-265)."""
        if self.dof == 4:
            return pose_opt + step
        q = pose_opt[..., 3:]
        dq = (camera.get_quaternion_transfrom_mat(q) @ step[..., 3:, None]).squeeze(-1)
        return torch.cat((pose_opt[..., :3] + step[..., :3], F.normalize(q + dq, dim=-1)), dim=-1)


@PNP.register_module()
class RSLMSolver(LMSolver):
    """Random-sample LM: a RANSAC-like initialiser for ambiguous problems (levenberg_marquardt.py:268-353)."""

    def __init__(self, num_points=16, num_proposals=64, num_iter=3, draws='native', cluster_split=False, **kwargs):
        """draws='native' (default): the weighted subsets and start orientations come from one kernel launch
        (epnp_rslm_draw_f32, Philox keyed by a seed taken from torch's default generator, so torch.manual_seed governs
        it); draws='torch': torch.multinomial / randn / rand exactly as the reference calls them (:306-324) -- the same
        distribution from torch's own streams, for code that replays or compares them (the parity tests do).

        cluster_split=True lets objects with more points than one SM holds (above epnp_max_points(dof, 0, 0): 7,000 in
        6DoF) be solved by the cluster-split initialiser (epnp_rslm_split_f32) instead of being refused.  Objects at or
        below that limit take the resident kernel either way.  The largest N is then epnp_max_points_split(dof, 0, 0)
        (55,232 in 6DoF) with draws='torch', and with draws='native' the smaller of that and the draw kernel's own
        shared-memory limit, 4 N + 8 n 128 + 2 KB <= 227 KB (53,504 points at n = 16)."""
        super(RSLMSolver, self).__init__(num_iter=num_iter, **kwargs)
        self.num_points = num_points
        self.num_proposals = num_proposals
        if draws not in ('native', 'torch'):
            raise ValueError(f"draws must be 'native' or 'torch', got {draws!r}")
        self.draws = draws
        self.cluster_split = bool(cluster_split)

    def center_based_init(self, x2d, x3d, camera, eps=1e-6):
        """Translation guess from the spread of the 2D points vs the 3D points (:283-298)."""
        homo = F.pad(x2d, [0, 1], mode='constant', value=1.)
        rays = torch.linalg.solve(camera.cam_mats, homo.transpose(-1, -2)).transpose(-1, -2)
        rays = rays[..., :2] / rays[..., 2:].clamp(min=eps)
        ray_std, ray_mean = torch.std_mean(rays, dim=-2)
        obj_std = torch.std(x3d, dim=-2)
        direction = F.pad(ray_mean, [0, 1], mode='constant', value=1.)
        if self.dof == 4:
            depth = obj_std[..., 1] / ray_std[..., 1].clamp(min=eps)
        else:
            depth = math.sqrt(2 / 3) * obj_std.norm(dim=-1) / ray_std.norm(dim=-1).clamp(min=eps)
        return direction * depth.unsqueeze(-1)

    def _starting_hypotheses(self, x3d, x2d, camera):
        """(P, B, D): centre-based translation, uniformly random orientation (:314-324)."""
        P, bs = self.num_proposals, x2d.size(0)
        start = x2d.new_empty((P, bs, self._pose_dim()))
        start[..., :3] = self.center_based_init(x2d, x3d, camera)
        if self.dof == 4:
            start[..., 3] = torch.rand((P, bs), dtype=x2d.dtype, device=x2d.device) * (2 * math.pi)
        else:
            q = torch.randn((P, bs, 4), dtype=x2d.dtype, device=x2d.device)
            qn = q.norm(dim=-1, keepdim=True)
            unit = q.new_tensor([1., 0., 0., 0.])
            start[..., 3:] = torch.where(qn < self.eps, unit, q / qn)
        return start

    @torch.no_grad()
    def solve(self, x3d, x2d, w2d, camera, cost_fun, **kwargs):
        """-> pose (B, 4|7), None, min_cost (B).

        Two launches: the set-up (epnp_rslm_draw_f32: the centre-based translation guess and, per (proposal, object), a
        weighted subset without replacement and a random start orientation, in place of torch.multinomial on the (P*B, N)
        weight rows) and the solve (epnp_rslm_f32: one
        CTA per object, thread <-> hypothesis, LM / GN on the n sampled correspondences read from the object's resident
        pair records, scored on all N points, cheapest kept).  The reference's gather of (P*B, n, .) mini-problems, its
        P-fold repeated camera / cost objects and its P*B tiny solves do not exist; run on the same kernels that
        formulation measured slower and was removed.
        `rslm_seed=` fixes the Philox stream of the native draws: an int, or a one-element int64 CUDA tensor the kernel
        reads at run time (common.philox_seed; a graph being captured draws its own on the device)."""
        bs, pn, _ = x2d.size()
        pd = self._pose_dim()
        if bs == 0:
            return x2d.new_empty((0, pd)), None, x2d.new_empty((0,))
        P, n = self.num_proposals, self.num_points
        x3d, x2d, w2d = x3d.detach(), x2d.detach(), w2d.detach()
        if self.draws == 'torch':
            if torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing():
                raise RuntimeError(
                    "RSLMSolver(draws='torch') cannot be captured into a CUDA graph: center_based_init's "
                    "torch.linalg.solve checks its result on the host, a synchronisation that capture forbids.  "
                    "draws='native' (the default) is capturable: its kernel reads a seed drawn on the device")
            # weighted subsets without replacement, one row per (proposal, object)
            prob_rows = w2d.mean(dim=-1).unsqueeze(0).expand(P, bs, pn).reshape(P * bs, pn)
            inds = torch.multinomial(prob_rows, n).reshape(P, bs, n)
            start = self._starting_hypotheses(x3d, x2d, camera)
        else:
            seed = philox_seed(kwargs.get("rslm_seed"), x2d.device)
            # a subclass that overrides center_based_init keeps its say; otherwise the kernel computes the guess itself
            own_guess = type(self).center_based_init is not RSLMSolver.center_based_init
            t_init = self.center_based_init(x2d, x3d, camera) if own_guess else None
            inds, start = ops.rslm_draw(x3d, x2d, w2d, camera.cam_mats, t_init, P, n, self.dof, float(self.eps),
                                        *ops.seed_args(seed))
        pose, cost = ops.rslm(*_problem_args(x3d, x2d, w2d, camera, cost_fun), inds, start,
                              *self.param_lists(camera, cost_fun, kwargs.get("fast_mode", False)), self.cluster_split)
        return pose.to(x2d.dtype), None, cost.to(x2d.dtype)
