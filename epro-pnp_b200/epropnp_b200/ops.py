"""The native entry points as PyTorch custom operators (namespace `epropnp`), so that torch.compile, torch.export and
AOTInductor see each C-ABI call as one opaque node with a known output shape and an autograd formula.

Every operator takes only tensors (Optional where the C ABI takes NULL), ints, floats, bools and lists of them; the
EpnpParams block travels as two lists of scalars (param_lists) and is rebuilt inside the implementation, so no ctypes
object reaches traced code.  The implementations call through `native`'s functions (which normalise the inputs:
float32, broadcast, contiguous) and choose the resident or cluster-split call by N through epropnp.autograd's helpers,
so the library's refusals and the resident limits are the same as for a direct call.  Outputs are fresh float32 tensors
(the RSLM subsets int32); an output that was not asked for is an empty tensor.  Casting to the caller's dtype is left to
the caller.

Seeds of the Philox draws: `seed` (an int) or `seed_t` (a one-element int64 tensor the kernel reads when it runs,
native's *_seedptr_f32 entry points); seed_t wins when given.

Autograd (register_autograd) is registered on evaluate_cost, evaluate_full, lm_solve (pose_opt_plus), lm_amis_fused and
mc_epilogue, and for second order on the cost backwards (cost_backward, cost_pose_backward, cost_camera_backward: the
Hessian-vector product cost_hvp), on the pose_opt_plus backwards (gn_plus_backward, gn_plus_camera_backward: the
Hessian-vector product gn_plus_hvp) and on mc_lse_backward.  cost_hvp and gn_plus_hvp have none, so a third derivative
raises.  evaluate_full's residual / Jacobian are first-order only: a second backward through evaluate_backward raises.
lm_solve_stacked (the solve from stacked starts) has no differentiable output.

Forward mode (torch.autograd.forward_ad, torch.func.jvp and linearize) runs eagerly through the jvp formulas of the eager Functions of
evaluate_cost, evaluate_full (the kernel evaluate_jvp), lm_amis_fused (logw and cost_init), lm_solve (pose_opt_plus,
through gn_plus_hvp) and mc_epilogue (lse); each is the transpose of the reverse-mode formula beside it, with its detach
rules.  needs_derivative is the one predicate every routing point of the layer uses.  Under torch.func.jvp / linearize
the formulas run as autograd.Functions and their kernel calls go through the dispatcher (which unwraps functorch's
tensors).  Under torch.compile / torch.export a forward tangent raises; vmap-based transforms, forward over reverse (the
backward and Hessian operators) and reverse through evaluate_jvp are not supported.

The module's names (adaptive_delta, ..., mc_lse_backward) are the entry points the layer calls (_entry): the operator
while anything traces, its implementation directly in eager code.  The operators themselves are FORWARD / BACKWARD /
SECOND_ORDER / FORWARD_MODE / STACKED and torch.ops.epropnp.*; each entry point's `.op` is its operator.
"""
from typing import List, Optional

import torch
import torch.autograd.forward_ad as _fwAD
from torch import Tensor

from . import capi, native

_INT_FIELDS = ("dof", "lm_iter", "fast_mode", "mc_samples", "mc_iter", "acg_mle_iter")
_FLOAT_FIELDS = ("z_min", "min_lm_diagonal", "max_lm_diagonal", "min_relative_decrease", "initial_radius", "max_radius",
                 "eps", "huber_eps", "amis_eps", "acg_dispersion")


_DEFAULTS = {}


@torch.compiler.assume_constant_result
def _default_lists(dof):
    if dof not in _DEFAULTS:
        p = capi.default_params(dof)
        _DEFAULTS[dof] = (tuple(getattr(p, k) for k in _INT_FIELDS), tuple(getattr(p, k) for k in _FLOAT_FIELDS))
    return _DEFAULTS[dof]


def param_lists(params=None, dof=6, **overrides):
    """(ints, floats): the EpnpParams block as two lists of Python scalars.  `params` an EpnpParams, an (ints, floats)
    pair, or None for the library's defaults for `dof`; `overrides` by field name.  Traceable: the defaults are read from
    the library once, as a constant."""
    if isinstance(params, capi.EpnpParams):
        ints, floats = [getattr(params, k) for k in _INT_FIELDS], [getattr(params, k) for k in _FLOAT_FIELDS]
    elif params is not None:
        ints, floats = list(params[0]), list(params[1])
    else:
        ints, floats = _default_lists(int(dof))
        ints, floats = list(ints), list(floats)
    for k, v in overrides.items():
        if k in _INT_FIELDS:
            ints[_INT_FIELDS.index(k)] = int(v)
        elif k in _FLOAT_FIELDS:
            floats[_FLOAT_FIELDS.index(k)] = float(v)
        else:
            raise AttributeError(k)
    return ints, floats


def make_params(ints, floats):
    """(ints, floats) -> the ctypes EpnpParams the C ABI takes."""
    return capi.EpnpParams(**dict(zip(_INT_FIELDS, ints)), **dict(zip(_FLOAT_FIELDS, floats)))


def bound(b, ref):
    """A camera bound as an operator argument: None stays None, a Python float becomes a (2,) float32 tensor (it gets
    no gradient), a tensor is passed as it is."""
    if b is None or torch.is_tensor(b):
        return b
    return torch.full((2,), float(b), dtype=torch.float32, device=ref.device)


def delta_tensor(delta, ref):
    """The Huber threshold as an operator argument: a Python float becomes a 0-dim tensor of `ref`'s dtype."""
    return delta if torch.is_tensor(delta) else ref.new_tensor(float(delta))


def problem_args(x3d, x2d, w2d, cam_mats, lb, ub, delta):
    """The seven problem arguments of the operators: bounds are passed only as a pair (one alone does not clamp), a
    Python-float delta or bound becomes a tensor that gets no gradient."""
    bounded = lb is not None and ub is not None
    return (x3d, x2d, w2d, cam_mats, bound(lb, x3d) if bounded else None, bound(ub, x3d) if bounded else None,
            delta_tensor(delta, x2d))


def seed_args(seed):
    """A Philox seed (an int, or a one-element int64 tensor) -> the (seed, seed_t) operator arguments.  An int at or
    above 2^63 goes as its two's-complement int64: the C ABI's uint64 sees the same value."""
    if torch.is_tensor(seed):
        return 0, seed
    seed = int(seed)
    return (seed - 2 ** 64 if seed >= 2 ** 63 else seed), None


def _route():
    # the resident / cluster-split choice by N lives in epropnp.autograd (fused_forward, stacked_cost, ...)
    from epropnp import autograd
    return autograd


def _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta):
    return native.Problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)


def _empty(ref):
    return ref.new_empty((0,), dtype=torch.float32)


def _or_empty(t, ref):
    return _empty(ref) if t is None else t


def _pose_dim(dof):
    return 7 if dof == 6 else 4


def _bounded(lb, ub):
    return lb is not None and ub is not None


_IMPLS = {}


def _op(name):
    def register(fn):
        op = torch.library.custom_op(f"epropnp::{name}", mutates_args=())(fn)
        _IMPLS[op] = fn
        return op
    return register


# ---------------------------------------------------------------------------------------------------- forward operators
@_op("adaptive_delta")
def adaptive_delta(x2d: Tensor, w2d: Tensor, relative_delta: float) -> Tensor:
    return native.adaptive_delta(x2d, w2d, relative_delta)


@adaptive_delta.register_fake
def _(x2d, w2d, relative_delta):
    return x2d.new_empty((x2d.shape[0],), dtype=torch.float32)


@_op("evaluate_cost")
def evaluate_cost(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                  delta: Tensor, poses: Tensor, dof: int, z_min: float) -> Tensor:
    """poses (S, B, D) -> cost (S, B)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    return _route().stacked_cost(prob, poses, dof, z_min)


@evaluate_cost.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, dof, z_min):
    return x3d.new_empty((poses.shape[0], x3d.shape[0]), dtype=torch.float32)


@_op("evaluate_full")
def evaluate_full(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                  delta: Tensor, poses: Tensor, dof: int, z_min: float, huber_eps: float, clip_jac: bool, want_r: bool,
                  want_j: bool, want_c: bool) -> tuple[Tensor, Tensor, Tensor]:
    """poses (S, B, D) -> residual (S, B, 2N), cost (S, B), Jacobian (S, B, 2N, dof); stacked poses replicate the
    problem, every (pose, object) its own object."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    S, B, N = poses.shape[0], prob.B, prob.N
    run = prob
    if S != 1:
        rep = lambda t: t.unsqueeze(0).expand((S,) + t.shape).reshape((S * B,) + t.shape[1:])
        run = native.Problem(rep(prob.x3d), rep(prob.x2d), rep(prob.w2d), rep(prob.cam),
                             None if prob.lb is None else rep(prob.lb), None if prob.ub is None else rep(prob.ub),
                             rep(prob.delta))
    r, c, j = native.evaluate_full(run, poses.reshape(-1, poses.size(-1)), dof, z_min, huber_eps, clip_jac, want_r,
                                   want_j, want_c)
    return (r.reshape(S, B, 2 * N) if want_r else _empty(x3d), c.reshape(S, B) if want_c else _empty(x3d),
            j.reshape(S, B, 2 * N, dof) if want_j else _empty(x3d))


@evaluate_full.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, dof, z_min, huber_eps, clip_jac, want_r, want_j, want_c):
    S, B, N = poses.shape[0], x3d.shape[0], x3d.shape[1]
    new = lambda *s: x3d.new_empty(s, dtype=torch.float32)
    return (new(S, B, 2 * N) if want_r else new(0), new(S, B) if want_c else new(0),
            new(S, B, 2 * N, dof) if want_j else new(0))


@_op("lm_solve")
def lm_solve(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
             delta: Tensor, pose_init: Tensor, ints: List[int], floats: List[float], want_cov: bool, want_cost: bool,
             want_plus: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> pose_opt (B, D), pose_cov (B, dof, dof), cost (B), pose_opt_plus (B, D)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    out = native.lm_solve(prob, pose_init, make_params(ints, floats), want_cov=want_cov, want_cost=want_cost,
                          want_plus=want_plus)
    return tuple(_or_empty(out[k], x3d) for k in ("pose_opt", "pose_cov", "cost", "pose_opt_plus"))


@lm_solve.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, ints, floats, want_cov, want_cost, want_plus):
    B, dof = x3d.shape[0], ints[0]
    new = lambda *s: x3d.new_empty(s, dtype=torch.float32)
    D = _pose_dim(dof)
    return (new(B, D), new(B, dof, dof) if want_cov else new(0), new(B) if want_cost else new(0),
            new(B, D) if want_plus else new(0))


@_op("lm_solve_stacked")
def lm_solve_stacked(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                     ub: Optional[Tensor], delta: Tensor, pose_init: Tensor, ints: List[int], floats: List[float],
                     want_cov: bool, want_cost: bool, want_plus: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """lm_solve from stacked starts pose_init (S, B, D) -> pose_opt (S, B, D), pose_cov (S, B, dof, dof), cost (S, B),
    pose_opt_plus (S, B, D); start s of object b as lm_solve solves it with pose_init[s].  No output is
    differentiable."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    out = native.lm_solve_stacked(prob, pose_init, make_params(ints, floats), want_cov=want_cov, want_cost=want_cost,
                                  want_plus=want_plus)
    return tuple(_or_empty(out[k], x3d) for k in ("pose_opt", "pose_cov", "cost", "pose_opt_plus"))


@lm_solve_stacked.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, ints, floats, want_cov, want_cost, want_plus):
    S, B, dof = pose_init.shape[0], x3d.shape[0], ints[0]
    new = lambda *s: x3d.new_empty(s, dtype=torch.float32)
    D = _pose_dim(dof)
    return (new(S, B, D), new(S, B, dof, dof) if want_cov else new(0), new(S, B) if want_cost else new(0),
            new(S, B, D) if want_plus else new(0))


@_op("lm_amis_fused")
def lm_amis_fused(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                  delta: Tensor, pose_init: Tensor, cost_init_pose: Optional[Tensor], noise3: Optional[Tensor],
                  chi2: Optional[Tensor], noise4: Optional[Tensor], seed: int, seed_t: Optional[Tensor],
                  ints: List[int], floats: List[float], want_cost: bool, want_plus: bool,
                  want_cost_init: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """LM solve + AMIS from pose_init (B, D) -> pose_opt (B, D), cost (B), pose_opt_plus (B, D), cost_init (B),
    pose_samples (B, M, D), logw (B, M) [object-major].  cost_init is the cost at cost_init_pose (B, D) when that is
    given (differentiable, with the log-weights, in one backward launch), else the fused kernel's own with
    want_cost_init."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    params = make_params(ints, floats)
    noise = None if noise3 is None else (noise3, chi2, noise4)
    route = _route()
    out = route.fused_forward(prob, pose_init, params, noise=noise, seed=seed if seed_t is None else seed_t,
                              want_cost=want_cost, want_plus=want_plus,
                              want_cost_init=want_cost_init and cost_init_pose is None, want_cov=False)
    cost_init = out["cost_init"]
    if cost_init_pose is not None:
        cost_init = route.stacked_cost(prob, cost_init_pose.unsqueeze(0), params.dof, params.z_min)[0]
    return (out["pose_opt"], _or_empty(out["cost"], x3d), _or_empty(out["pose_opt_plus"], x3d),
            _or_empty(cost_init, x3d), out["pose_samples"], out["logw"])


@lm_amis_fused.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose_init, cost_init_pose, noise3, chi2, noise4, seed, seed_t, ints,
      floats, want_cost, want_plus, want_cost_init):
    B, dof, M = x3d.shape[0], ints[0], ints[3]
    D = _pose_dim(dof)
    new = lambda *s: x3d.new_empty(s, dtype=torch.float32)
    return (new(B, D), new(B) if want_cost else new(0), new(B, D) if want_plus else new(0),
            new(B) if (cost_init_pose is not None or want_cost_init) else new(0), new(B, M, D), new(B, M))


@_op("rslm_draw")
def rslm_draw(x3d: Optional[Tensor], x2d: Optional[Tensor], w2d: Tensor, cam_mats: Optional[Tensor],
              t_init: Optional[Tensor], P: int, n: int, dof: int, eps: float, seed: int,
              seed_t: Optional[Tensor]) -> tuple[Tensor, Tensor]:
    """-> inds (P, B, n) int32, start (P, B, D) (native.rslm_draw)."""
    return native.rslm_draw(x3d, x2d, w2d, cam_mats, P, n, dof, eps=eps, seed=seed if seed_t is None else seed_t,
                            t_init=t_init)


@rslm_draw.register_fake
def _(x3d, x2d, w2d, cam_mats, t_init, P, n, dof, eps, seed, seed_t):
    B = w2d.shape[0]
    return (w2d.new_empty((P, B, n), dtype=torch.int32), w2d.new_empty((P, B, _pose_dim(dof)), dtype=torch.float32))


@_op("rslm")
def rslm(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
         delta: Tensor, inds: Tensor, start: Tensor, ints: List[int], floats: List[float],
         cluster_split: bool) -> tuple[Tensor, Tensor]:
    """Random-sample LM over inds (P, B, n) / start (P, B, D) -> pose (B, D), cost (B).  Above the resident limit the
    cluster-split form runs only with cluster_split; without it such objects are refused."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    out = _route().rslm_solve(prob, inds, start, make_params(ints, floats), allow_split=cluster_split)
    return out["pose"], out["cost"]


@rslm.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, inds, start, ints, floats, cluster_split):
    B = x3d.shape[0]
    return x3d.new_empty((B, _pose_dim(ints[0])), dtype=torch.float32), x3d.new_empty((B,), dtype=torch.float32)


@_op("epnp_init")
def epnp_init(x3d: Tensor, x2d: Tensor, w2d: Optional[Tensor], cam_mats: Tensor, conf_quantile: float) -> Tensor:
    """-> pose (B, 7) (native.epnp_init, or its split form above the resident limit)."""
    return _route().epnp_init(x3d, x2d, w2d, cam_mats, conf_quantile)


@epnp_init.register_fake
def _(x3d, x2d, w2d, cam_mats, conf_quantile):
    return x3d.new_empty((x3d.shape[0], 7), dtype=torch.float32)


@_op("mc_epilogue")
def mc_epilogue(logw_bm: Tensor, pose_samples_bmd: Optional[Tensor], pose_opt: Optional[Tensor],
                cost_target: Optional[Tensor], want_lse: bool, want_loss: bool, want_weights: bool,
                want_score: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """logw (B, M) [, pose_samples (B, M, D), pose_opt (B, D), cost_target (B)] -> lse (B), loss (B), weights (B, M),
    score_te (B) (native.mc_epilogue)."""
    out = native.mc_epilogue(logw_bm, pose_samples_bmd, pose_opt, cost_target, want_lse=want_lse, want_loss=want_loss,
                             want_weights=want_weights, want_score=want_score)
    return tuple(_or_empty(out[k], logw_bm) for k in ("lse", "loss", "weights", "score_te"))


@mc_epilogue.register_fake
def _(logw_bm, pose_samples_bmd, pose_opt, cost_target, want_lse, want_loss, want_weights, want_score):
    B, M = logw_bm.shape
    new = lambda *s: logw_bm.new_empty(s, dtype=torch.float32)
    return (new(B) if want_lse else new(0), new(B) if want_loss else new(0), new(B, M) if want_weights else new(0),
            new(B) if want_score else new(0))


# --------------------------------------------------------------------------------------------------- backward operators
@_op("cost_backward")
def cost_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                  delta: Tensor, poses_a: Tensor, grad_a: Tensor, poses_b: Optional[Tensor], grad_b: Optional[Tensor],
                  dof: int, z_min: float, want: List[bool]) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """native.cost_backward -> (B, N, 3), (B, N, 2), (B, N, 2), (B) gradients of x3d, x2d, w2d, delta."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    grads = native.cost_backward(prob, dof, z_min, poses_a, grad_a, poses_b, grad_b, want=tuple(want))
    return tuple(_or_empty(g, x3d) for g in grads)


@cost_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses_a, grad_a, poses_b, grad_b, dof, z_min, want):
    B, N = x3d.shape[0], x3d.shape[1]
    return _grad_fakes(x3d, want, ((B, N, 3), (B, N, 2), (B, N, 2), (B,)))


def _grad_fakes(ref, want, shapes):
    return tuple(ref.new_empty(s if w else (0,), dtype=torch.float32) for w, s in zip(want, shapes))


@_op("cost_pose_backward")
def cost_pose_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                       ub: Optional[Tensor], delta: Tensor, poses: Tensor, grad: Tensor, dof: int,
                       z_min: float) -> Tensor:
    """native.cost_pose_backward: poses (B, P, D), grad (B, P) -> (B, P, D)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    return native.cost_pose_backward(prob, dof, z_min, poses, grad)


@cost_pose_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, grad, dof, z_min):
    return poses.new_empty(poses.shape, dtype=torch.float32)


@_op("cost_camera_backward")
def cost_camera_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                         ub: Optional[Tensor], delta: Tensor, poses_a: Tensor, grad_a: Tensor, poses_b: Optional[Tensor],
                         grad_b: Optional[Tensor], dof: int, z_min: float,
                         want: List[bool]) -> tuple[Tensor, Tensor, Tensor]:
    """native.cost_camera_backward -> (B, 3, 3), (B, 2), (B, 2) gradients of cam_mats, lb, ub."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    grads = native.cost_camera_backward(prob, dof, z_min, poses_a, grad_a, poses_b, grad_b, want=tuple(want))
    return tuple(_or_empty(g, x3d) for g in grads)


@cost_camera_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses_a, grad_a, poses_b, grad_b, dof, z_min, want):
    B = x3d.shape[0]
    return _grad_fakes(x3d, want, ((B, 3, 3), (B, 2), (B, 2)))


@_op("gn_plus_backward")
def gn_plus_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                     ub: Optional[Tensor], delta: Tensor, pose: Tensor, grad_pose_plus: Tensor, dof: int, z_min: float,
                     eps: float, huber_eps: float, want: List[bool]) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """Gradients of x3d, x2d, w2d, delta through pose_opt_plus = pose (+) gn_step(pose) (native.gn_plus_backward, or
    its split form above the resident limit)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    grads = _route().gn_plus_backward(prob, pose, grad_pose_plus, dof, z_min, eps, huber_eps, tuple(want))
    return tuple(_or_empty(g, x3d) for g in grads)


@gn_plus_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, dof, z_min, eps, huber_eps, want):
    B, N = x3d.shape[0], x3d.shape[1]
    return _grad_fakes(x3d, want, ((B, N, 3), (B, N, 2), (B, N, 2), (B,)))


@_op("gn_plus_camera_backward")
def gn_plus_camera_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                            ub: Optional[Tensor], delta: Tensor, pose: Tensor, grad_pose_plus: Tensor, dof: int,
                            z_min: float, eps: float, huber_eps: float,
                            want: List[bool]) -> tuple[Tensor, Tensor, Tensor]:
    """Gradients of cam_mats, lb, ub through pose_opt_plus (native.gn_plus_camera_backward)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    grads = native.gn_plus_camera_backward(prob, pose, grad_pose_plus, dof, z_min, eps, huber_eps, want=tuple(want))
    return tuple(_or_empty(g, x3d) for g in grads)


@gn_plus_camera_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, dof, z_min, eps, huber_eps, want):
    B = x3d.shape[0]
    return _grad_fakes(x3d, want, ((B, 3, 3), (B, 2), (B, 2)))


@_op("evaluate_backward")
def evaluate_backward(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor],
                      ub: Optional[Tensor], delta: Tensor, poses: Tensor, dof: int, z_min: float, huber_eps: float,
                      clip_jac: bool, g_res: Optional[Tensor], g_jac: Optional[Tensor], g_cost: Optional[Tensor],
                      want: List[bool]) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """native.evaluate_backward -> gradients of x3d, x2d, w2d, delta, poses (S, B, D), cam_mats, lb, ub."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    grads = native.evaluate_backward(prob, poses, dof, z_min, huber_eps, clip_jac, g_res, g_jac, g_cost,
                                     want=tuple(want))
    return tuple(_or_empty(g, x3d) for g in grads)


@evaluate_backward.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, dof, z_min, huber_eps, clip_jac, g_res, g_jac, g_cost, want):
    B, N, S = x3d.shape[0], x3d.shape[1], poses.shape[0]
    return _grad_fakes(x3d, want, ((B, N, 3), (B, N, 2), (B, N, 2), (B,), (S, B, _pose_dim(dof)), (B, 3, 3), (B, 2),
                                   (B, 2)))


@_op("cost_hvp")
def cost_hvp(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
             delta: Tensor, poses: Tensor, grad: Tensor, t_x3d: Optional[Tensor], t_x2d: Optional[Tensor],
             t_w2d: Optional[Tensor], t_delta: Optional[Tensor], t_pose: Optional[Tensor], t_cam: Optional[Tensor],
             t_lb: Optional[Tensor], t_ub: Optional[Tensor], dof: int, z_min: float,
             want: List[bool]) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """native.cost_hvp: poses (B, P, D), grad (B, P) and the tangent's parts (None: zero) -> H v with respect to x3d,
    x2d, w2d, delta, the poses (times grad), d cost_p . v (B, P), H v with respect to cam_mats, lb, ub."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    tangents = dict(zip(native.HVP_TANGENTS, (t_x3d, t_x2d, t_w2d, t_delta, t_pose, t_cam, t_lb, t_ub)))
    out = native.cost_hvp(prob, dof, z_min, poses, grad, tangents, tuple(want))
    return tuple(_or_empty(t, x3d) for t in out)


@cost_hvp.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, grad, t_x3d, t_x2d, t_w2d, t_delta, t_pose, t_cam, t_lb, t_ub,
      dof, z_min, want):
    B, N, P = x3d.shape[0], x3d.shape[1], poses.shape[1]
    return _grad_fakes(x3d, want, ((B, N, 3), (B, N, 2), (B, N, 2), (B,), (B, P, _pose_dim(dof)), (B, P), (B, 3, 3),
                                   (B, 2), (B, 2)))


@_op("gn_plus_hvp")
def gn_plus_hvp(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                delta: Tensor, pose: Tensor, grad_pose_plus: Tensor, t_x3d: Optional[Tensor], t_x2d: Optional[Tensor],
                t_w2d: Optional[Tensor], t_delta: Optional[Tensor], t_cam: Optional[Tensor], t_lb: Optional[Tensor],
                t_ub: Optional[Tensor], dof: int, z_min: float, eps: float, huber_eps: float,
                want: List[bool]) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """native.gn_plus_hvp: the tangent's parts (None: zero) -> H u with respect to x3d, x2d, w2d, delta, cam_mats, lb,
    ub of f = grad_pose_plus . pose_opt_plus, and d pose_opt_plus . u (B, D)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    tangents = dict(zip(native.GN_HVP_TANGENTS, (t_x3d, t_x2d, t_w2d, t_delta, t_cam, t_lb, t_ub)))
    out = native.gn_plus_hvp(prob, pose, grad_pose_plus, dof, z_min, eps, huber_eps, tangents, tuple(want))
    return tuple(_or_empty(t, x3d) for t in out)


@gn_plus_hvp.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, grad_pose_plus, t_x3d, t_x2d, t_w2d, t_delta, t_cam, t_lb, t_ub,
      dof, z_min, eps, huber_eps, want):
    B, N = x3d.shape[0], x3d.shape[1]
    return _grad_fakes(x3d, want, ((B, N, 3), (B, N, 2), (B, N, 2), (B,), (B, 3, 3), (B, 2), (B, 2),
                                   (B, _pose_dim(dof))))


@_op("evaluate_jvp")
def evaluate_jvp(x3d: Tensor, x2d: Tensor, w2d: Tensor, cam_mats: Tensor, lb: Optional[Tensor], ub: Optional[Tensor],
                 delta: Tensor, poses: Tensor, t_x3d: Optional[Tensor], t_x2d: Optional[Tensor],
                 t_w2d: Optional[Tensor], t_delta: Optional[Tensor], t_pose: Optional[Tensor], t_cam: Optional[Tensor],
                 t_lb: Optional[Tensor], t_ub: Optional[Tensor], dof: int, z_min: float, huber_eps: float,
                 clip_jac: bool, want: List[bool]) -> tuple[Tensor, Tensor, Tensor]:
    """native.evaluate_jvp: poses (S, B, D) and the tangent's parts (None: zero) -> the tangents of the residual
    (S, B, 2N), the Jacobian (S, B, 2N, dof) and the cost (S, B)."""
    prob = _problem(x3d, x2d, w2d, cam_mats, lb, ub, delta)
    tangents = dict(zip(native.JVP_TANGENTS, (t_x3d, t_x2d, t_w2d, t_delta, t_pose, t_cam, t_lb, t_ub)))
    out = native.evaluate_jvp(prob, poses, dof, z_min, huber_eps, clip_jac, tangents, tuple(want))
    return tuple(_or_empty(t, x3d) for t in out)


@evaluate_jvp.register_fake
def _(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, t_x3d, t_x2d, t_w2d, t_delta, t_pose, t_cam, t_lb, t_ub, dof,
      z_min, huber_eps, clip_jac, want):
    S, B, N = poses.shape[0], x3d.shape[0], x3d.shape[1]
    return _grad_fakes(x3d, want, ((S, B, 2 * N), (S, B, 2 * N, dof), (S, B)))


@_op("mc_lse_backward")
def mc_lse_backward(logw_bm: Tensor, lse: Tensor, grad_lse: Tensor) -> Tensor:
    """grad_logw (B, M) = grad_lse[b] * exp(logw[b, m] - lse[b]) (native.mc_lse_backward)."""
    return native.mc_lse_backward(logw_bm, lse, grad_lse)


@mc_lse_backward.register_fake
def _(logw_bm, lse, grad_lse):
    return logw_bm.new_empty(logw_bm.shape, dtype=torch.float32)


# ----------------------------------------------------------------------------------------------------- autograd formulas
def _sum_to(like, g):
    """A native gradient -> the dtype and shape of the input it belongs to: a one-element input (a scalar delta, a
    Python-float bound made a tensor) receives the sum over objects, a broadcast one (a (B, N, 1) weight, a (3, 3)
    camera, a (2,) bound) the sum over the axes it was expanded along."""
    g = g.to(like.dtype)
    if like.numel() == 1 and g.numel() != 1:
        return g.sum().reshape(like.shape)
    return g.reshape(like.shape) if g.numel() == like.numel() else g.sum_to_size(like.shape)


_EAGER = {}
_EAGER_FUNC = {}


def _register_autograd(op, backward, setup_context, jvp=None):
    """op.register_autograd, and the same functions as autograd.Functions that run the implementation directly: the
    eager drivers of the formula (see _entry).  `jvp(ctx, inputs, output, tangents)` [opt]: the forward-mode formula,
    the tangents of the outputs (None: none) from those of the inputs; it runs eagerly only (the operator's
    register_autograd has no forward rule).  Two classes: one with forward(ctx, ...) for reverse mode and
    torch.autograd.forward_ad, and, for torch.func's transforms, one in setup_context style (which torch.func requires,
    but whose apply binds the arguments through inspect.signature on every call: host time the training step does not
    need to pay)."""
    op.register_autograd(backward, setup_context=setup_context)
    impl_direct = _IMPLS[op]

    def impl(*args):
        # under a torch-dispatch mode (make_fx, which torch.func.linearize traces with) the operator itself, which the
        # mode records: the implementation's ctypes call is invisible to it, and its outputs would be traced as empty
        # tensors that a replay of the graph leaves unwritten
        return op(*args) if torch._C._len_torch_dispatch_stack() else impl_direct(*args)

    def setup(ctx, inputs, output):
        setup_context(ctx, inputs, output)
        if jvp is not None and _fwAD._current_level >= 0:         # a forward-AD level (torch.func.jvp opens one too)
            ctx.fw_consts = tuple(None if torch.is_tensor(a) else a for a in inputs)
            ctx.fw_tensor = tuple(torch.is_tensor(a) for a in inputs)
            ctx.save_for_forward(*(a for a in inputs if torch.is_tensor(a)), *output)

    def forward(ctx, *args):
        out = impl(*args)
        setup(ctx, args, out)
        return out

    name = f"epropnp_{op._name.split('::')[-1]}"
    body = dict(backward=staticmethod(backward))
    if jvp is not None:
        def fw(ctx, *tangents):
            saved = iter(ctx.saved_tensors)
            inputs = tuple(next(saved) if t else c for t, c in zip(ctx.fw_tensor, ctx.fw_consts))
            return jvp(ctx, inputs, tuple(saved), tangents)
        body["jvp"] = staticmethod(fw)
    _EAGER[op] = type(name, (torch.autograd.Function,), dict(body, forward=staticmethod(forward)))
    _EAGER_FUNC[op] = type(name, (torch.autograd.Function,),
                           dict(body, forward=staticmethod(impl), setup_context=staticmethod(setup)))


def _save_problem(ctx, inputs, extra=()):
    x3d, x2d, w2d, cam_mats, lb, ub, delta = inputs[:7]
    ctx.bounded = _bounded(lb, ub)
    ctx.has_lb, ctx.has_ub = lb is not None, ub is not None
    saved = [x3d, x2d, w2d, cam_mats, delta] + [t for t in (lb, ub) if t is not None]
    ctx.save_for_backward(*saved, *extra)


def _load_problem(ctx, n_extra=0):
    """-> the seven problem inputs and the extra saved tensors, as saved: under create_graph a formula's backward
    operators see the graph (the cost and pose_opt_plus backwards have second-order formulas; the others raise)."""
    saved = ctx.saved_tensors
    n = len(saved) - n_extra
    x3d, x2d, w2d, cam_mats, delta = saved[:5]
    rest = list(saved[5:n])
    lb = rest.pop(0) if ctx.has_lb else None
    ub = rest.pop(0) if ctx.has_ub else None
    return (x3d, x2d, w2d, cam_mats, lb, ub, delta), saved[n:]


def _problem_wants(ctx):
    """needs_input_grad of the seven problem inputs -> (x3d, x2d, w2d, delta), (cam_mats, lb, ub).  A bound gets a
    gradient only while both bounds are given: the projection is otherwise not clamped."""
    n = ctx.needs_input_grad
    return (n[0], n[1], n[2], n[6]), (n[3], ctx.bounded and n[4], ctx.bounded and n[5])


def _problem_grads(prob, corr, cam):
    """Gradients of the seven problem inputs, in argument order, from the native (x3d, x2d, w2d, delta) and
    (cam_mats, lb, ub) ones (None where not wanted)."""
    x3d, x2d, w2d, cam_mats, lb, ub, delta = prob
    g = lambda like, t: None if t is None else _sum_to(like, t)
    return (g(x3d, corr[0]), g(x2d, corr[1]), g(w2d, corr[2]), g(cam_mats, cam[0]), g(lb, cam[1]), g(ub, cam[2]),
            g(delta, corr[3]))


def _cost_grads(ctx, prob, poses_a, grad_a, poses_b=None, grad_b=None):
    """Correspondence / delta and camera gradients of sum_p grad[p] * cost(pose p) (two native launches at most).  The
    inputs are passed as they are: under create_graph the backward operators' own formulas (_cost_hvp_backward) make
    these gradients differentiable."""
    want_corr, want_cam = _problem_wants(ctx)
    p = prob
    corr = (None,) * 4
    if any(want_corr):
        out = cost_backward(*p, poses_a, grad_a, poses_b, grad_b, ctx.dof, ctx.z_min, list(want_corr))
        corr = tuple(t if w else None for t, w in zip(out, want_corr))
    cam = (None,) * 3
    if any(want_cam):
        out = cost_camera_backward(*p, poses_a, grad_a, poses_b, grad_b, ctx.dof, ctx.z_min, list(want_cam))
        cam = tuple(t if w else None for t, w in zip(out, want_cam))
    return _problem_grads(prob, corr, cam)


def _evaluate_cost_setup(ctx, inputs, output):
    poses = inputs[7]
    ctx.dof, ctx.z_min = inputs[8], inputs[9]
    _save_problem(ctx, inputs, (poses,))


def _evaluate_cost_backward(ctx, g_cost):
    prob, (poses,) = _load_problem(ctx, 1)
    poses_bm = poses.transpose(0, 1).contiguous()                                # object-major (B, S, D)
    g = g_cost.transpose(0, 1).contiguous()                                        # object-major (B, S)
    grads = _cost_grads(ctx, prob, poses_bm, g)
    gpose = None
    if ctx.needs_input_grad[7]:
        gpose = cost_pose_backward(*prob, poses_bm, g, ctx.dof, ctx.z_min).transpose(0, 1).to(poses.dtype) \
            .reshape(poses.shape)
    return grads + (gpose, None, None)


# ------------------------------------------------------------------------------------------------ forward-mode formulas
def _expand_to(t, shape):
    """The reverse of _sum_to: a tangent of a broadcast input (a scalar delta, a (3, 3) camera, a (2,) bound, a
    (B, N, 1) weight) expanded to the native shape (None stays None)."""
    if t is None:
        return None
    if t.numel() == 1:
        return t.reshape(()).expand(shape)
    return t.reshape(shape) if t.numel() == _numel(shape) else t.expand(shape)


def _numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


def _problem_tangents(prob, tangents):
    """The tangents of the seven problem inputs (argument order) by native.JVP_TANGENTS name, in the native shapes: none
    for a bound without the other one (it does not clamp)."""
    x3d = prob[0]
    B, N = x3d.shape[0], x3d.shape[1]
    bounded = _bounded(prob[4], prob[5])
    t_x3d, t_x2d, t_w2d, t_cam, t_lb, t_ub, t_delta = tangents[:7]
    return dict(x3d=_expand_to(t_x3d, (B, N, 3)), x2d=_expand_to(t_x2d, (B, N, 2)), w2d=_expand_to(t_w2d, (B, N, 2)),
                delta=_expand_to(t_delta, (B,)), cam=_expand_to(t_cam, (B, 3, 3)),
                lb=_expand_to(t_lb, (B, 2)) if bounded else None, ub=_expand_to(t_ub, (B, 2)) if bounded else None)


def cost_jvp(prob, poses, t_prob, t_pose, dof, z_min):
    """d cost(poses) . v (S, B) at poses (S, B, D): v = the problem tangents (a dict, _problem_tangents) and t_pose
    (S, B, D) or None."""
    t = dict(t_prob, pose=t_pose)
    return evaluate_jvp(*prob, poses, *(t.get(k) for k in native.JVP_TANGENTS), dof, z_min, 1e-10, False,
                        [False, False, True])[2]


def _evaluate_cost_jvp(ctx, inputs, output, tangents):
    return cost_jvp(inputs[:7], inputs[7], _problem_tangents(inputs[:7], tangents), tangents[7], ctx.dof, ctx.z_min)


_register_autograd(evaluate_cost, _evaluate_cost_backward, _evaluate_cost_setup, _evaluate_cost_jvp)


def _evaluate_full_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)             # an output the loss does not use costs the backward nothing
    ctx.consts = inputs[8:12]
    want_r, want_j, want_c = inputs[12:15]
    ctx.mark_non_differentiable(*(t for t, w in zip(output, (want_r, want_c, want_j)) if not w))   # (r, c, j)
    _save_problem(ctx, inputs, (inputs[7],))


def _evaluate_full_backward(ctx, g_res, g_cost, g_jac):
    prob, (poses,) = _load_problem(ctx, 1)
    ups = [g if g is not None and g.numel() else None for g in (g_res, g_jac, g_cost)]
    want_corr, want_cam = _problem_wants(ctx)
    want = want_corr + (ctx.needs_input_grad[7],) + want_cam
    if all(g is None for g in ups) or not any(want):
        return (None,) * 15
    dof, z_min, huber_eps, clip_jac = ctx.consts
    # the saved inputs are passed as they are: under create_graph a second backward reaches evaluate_backward, which
    # has no formula, and raises (first order only)
    grads = evaluate_backward(*prob, poses.detach(), dof, z_min, huber_eps, clip_jac, *ups, list(want))
    grads = [t if w else None for t, w in zip(grads, want)]
    out = _problem_grads(prob, grads[:4], grads[5:])
    gpose = None if grads[4] is None else grads[4].to(poses.dtype).reshape(poses.shape)
    return out + (gpose,) + (None,) * 7


def _evaluate_full_jvp(ctx, inputs, output, tangents):
    dof, z_min, huber_eps, clip_jac = ctx.consts
    want = list(inputs[12:15])                                                   # (r, j, c)
    t = dict(_problem_tangents(inputs[:7], tangents), pose=tangents[7])
    d_r, d_j, d_c = evaluate_jvp(*inputs[:8], *(t.get(k) for k in native.JVP_TANGENTS), dof, z_min, huber_eps,
                                 clip_jac, want)
    return d_r if want[0] else None, d_c if want[2] else None, d_j if want[1] else None


_register_autograd(evaluate_full, _evaluate_full_backward, _evaluate_full_setup, _evaluate_full_jvp)


def _fused_setup(ctx, inputs, output):
    ints, floats = inputs[14], inputs[15]
    ctx.dof, ctx.z_min = ints[0], floats[0]
    cost_init_pose = inputs[8]
    ctx.has_ci = cost_init_pose is not None
    pose_opt, cost, plus, cost_init, samples, logw = output
    ctx.mark_non_differentiable(pose_opt, cost, plus, samples)
    if not ctx.has_ci:
        ctx.mark_non_differentiable(cost_init)
    _save_problem(ctx, inputs, (samples,) + ((cost_init_pose,) if ctx.has_ci else ()))


def _fused_backward(ctx, g_pose, g_cost, g_plus, g_cost_init, g_samples, g_logw):
    prob, extra = _load_problem(ctx, 2 if ctx.has_ci else 1)
    samples = extra[0]
    B = samples.shape[0]
    poses_b = grad_b = None
    if ctx.has_ci and g_cost_init is not None and g_cost_init.numel() == B:
        cost_init_pose = extra[1]
        poses_b = cost_init_pose.reshape(B, 1, -1)
        grad_b = g_cost_init.reshape(B, 1)
    if g_logw is None:
        g_logw = torch.zeros(B, samples.shape[1], device=samples.device)
    grads = _cost_grads(ctx, prob, samples, -g_logw.contiguous(), poses_b, grad_b)
    gpose = None
    if ctx.has_ci and ctx.needs_input_grad[8] and poses_b is not None:
        gpose = cost_pose_backward(*prob, poses_b, grad_b, ctx.dof, ctx.z_min)[:, 0].to(extra[1].dtype) \
            .reshape(extra[1].shape)
    return grads + (None, gpose) + (None,) * 10


def _fused_jvp(ctx, inputs, output, tangents):
    """logw = -cost(samples) - log q: -d cost(samples) . v with the samples constant; cost_init (at cost_init_pose):
    d cost(cost_init_pose) . (v, its tangent), in the same launch.  pose_opt, cost, pose_opt_plus and the samples carry
    none, as in reverse mode."""
    prob, samples = inputs[:7], output[4]
    B = samples.shape[0]
    poses = samples.transpose(0, 1)                                              # (M, B, D)
    t_pose = None
    if ctx.has_ci:
        poses = torch.cat((inputs[8].to(poses.dtype).reshape(1, B, -1), poses))
        tci = tangents[8]
        t_pose = torch.zeros(poses.shape, dtype=torch.float32, device=poses.device)
        if tci is not None:
            t_pose[0] = tci.reshape(B, -1)
    dc = cost_jvp(prob, poses.contiguous(), _problem_tangents(prob, tangents), t_pose, ctx.dof, ctx.z_min)
    t_ci = dc[0].clone() if ctx.has_ci else None
    t_logw = -dc[1 if ctx.has_ci else 0:].transpose(0, 1).contiguous()         # the layout of logw (B, M)
    return None, None, None, t_ci, None, t_logw


_register_autograd(lm_amis_fused, _fused_backward, _fused_setup, _fused_jvp)


def gn_plus_grads(prob, pose, grad_plus, dof, z_min, eps, huber_eps, needs):
    """Gradients of the seven problem inputs (argument order; None where `needs` is False) through pose_opt_plus =
    pose (+) gn_step(pose): the gn_plus backward operators, then the reduction to each input's shape.  The problem
    inputs and grad_plus are passed as they are (the pose detached): under create_graph the backward operators' own
    formulas (_gn_plus_hvp_backward) make these gradients differentiable."""
    lb_ub = prob[4] is not None and prob[5] is not None
    corr_w = (needs[0], needs[1], needs[2], needs[6])
    cam_w = (needs[3], lb_ub and needs[4], lb_ub and needs[5])
    pose = pose.detach()
    corr = (None,) * 4
    if any(corr_w):
        out = gn_plus_backward(*prob, pose, grad_plus, dof, z_min, eps, huber_eps, list(corr_w))
        corr = tuple(t if w else None for t, w in zip(out, corr_w))
    cam = (None,) * 3
    if any(cam_w):
        out = gn_plus_camera_backward(*prob, pose, grad_plus, dof, z_min, eps, huber_eps, list(cam_w))
        cam = tuple(t if w else None for t, w in zip(out, cam_w))
    return _problem_grads(prob, corr, cam)


def gn_plus_jvp(prob, pose, tangents, dof, z_min, eps, huber_eps):
    """d pose_opt_plus . u (B, D) of pose_opt_plus = pose (+) gn_step(pose), the pose held constant: gn_plus_hvp's grad
    output with no problem output wanted.  `tangents`: those of the seven problem inputs in argument order."""
    t = _problem_tangents(prob, tangents)
    if all(v is None for v in t.values()):
        return None
    pose = pose.detach()
    zero = torch.zeros(pose.shape, dtype=torch.float32, device=pose.device)
    return gn_plus_hvp(*prob, pose, zero, *(t[k] for k in native.GN_HVP_TANGENTS), dof, z_min, eps, huber_eps,
                       [False] * 7 + [True])[7]


def _lm_solve_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[:3])
    ints, floats = inputs[8], inputs[9]
    ctx.consts = (ints[0], floats[0], floats[6], floats[7])                  # dof, z_min, eps, huber_eps
    _save_problem(ctx, inputs, (inputs[7],))


def _lm_solve_backward(ctx, g_opt, g_cov, g_cost, g_plus):
    if g_plus is None:
        return (None,) * 13
    prob, (pose,) = _load_problem(ctx, 1)
    return gn_plus_grads(prob, pose, g_plus, *ctx.consts, ctx.needs_input_grad[:7]) + (None,) * 6


def _lm_solve_jvp(ctx, inputs, output, tangents):
    if not inputs[12]:                                                           # want_plus
        return None, None, None, None
    return None, None, None, gn_plus_jvp(inputs[:7], inputs[7], tangents[:7], *ctx.consts)


_register_autograd(lm_solve, _lm_solve_backward, _lm_solve_setup, _lm_solve_jvp)


def _lm_solve_stacked_setup(ctx, inputs, output):
    ctx.mark_non_differentiable(*output)


def _lm_solve_stacked_backward(ctx, *grads):
    return (None,) * 13


_register_autograd(lm_solve_stacked, _lm_solve_stacked_backward, _lm_solve_stacked_setup)


def _mc_epilogue_setup(ctx, inputs, output):
    ctx.mark_non_differentiable(*output[1:])
    ctx.save_for_backward(inputs[0], output[0])


def _mc_epilogue_backward(ctx, g_lse, g_loss, g_weights, g_score):
    logw_bm, lse = ctx.saved_tensors
    g = None
    if g_lse is not None and ctx.needs_input_grad[0]:
        g = mc_lse_backward(logw_bm, lse, g_lse).to(logw_bm.dtype)
    return (g,) + (None,) * 7


def _mc_epilogue_jvp(ctx, inputs, output, tangents):
    """lse: sum_m softmax(logw)_m t_logw_m (torch on (B, M)).  The loss and the weights are non-differentiable outputs
    in reverse mode; with a tangent they raise rather than come back with none (the layer asks for them only without
    one: mc_sample_weights takes torch's softmax then).  The score carries none (its inputs are detached)."""
    if inputs[5] or inputs[6]:
        raise RuntimeError("epropnp::mc_epilogue: the loss and the sample weights have no forward-mode formula; take "
                           "them from logw with torch ops (logsumexp, softmax) under forward AD")
    t = tangents[0]
    if t is None or not inputs[4]:
        return None, None, None, None
    w = torch.exp(inputs[0].to(torch.float32) - output[0].unsqueeze(1))
    return (w * t.to(torch.float32)).sum(1), None, None, None


_register_autograd(mc_epilogue, _mc_epilogue_backward, _mc_epilogue_setup, _mc_epilogue_jvp)


# ---------------------------------------------------------------------------------------------- second-order formulas
def _cost_hvp_setup(ctx, inputs, output):
    """cost_backward / cost_camera_backward (two pose sets) and cost_pose_backward (one): the problem and the sets."""
    ctx.set_materialize_grads(False)
    two_sets = len(inputs) == 14
    ctx.dof, ctx.z_min = (inputs[11], inputs[12]) if two_sets else (inputs[9], inputs[10])
    sets = [inputs[7:9]] + ([inputs[9:11]] if two_sets and inputs[9] is not None else [])
    ctx.n_sets, ctx.n_inputs = len(sets), len(inputs)
    _save_problem(ctx, inputs, tuple(t for s in sets for t in s))


def _cost_hvp_backward(ctx, tangents):
    """The gradients of a cost backward's inputs from the tangents of its outputs (a dict by native.HVP_TANGENTS name):
    one cost_hvp over the pose sets laid side by side, then each output back to its input's shape."""
    prob, extra = _load_problem(ctx, 2 * ctx.n_sets)
    sets = [extra[2 * i:2 * i + 2] for i in range(ctx.n_sets)]
    n = ctx.needs_input_grad
    want_corr, want_cam = _problem_wants(ctx)
    want_pose = any(n[7 + 2 * i] for i in range(ctx.n_sets))
    want_grad = any(n[8 + 2 * i] for i in range(ctx.n_sets))
    want = list(want_corr) + [want_pose, want_grad] + list(want_cam)
    tangents = {k: t for k, t in tangents.items() if t is not None and t.numel()}
    if not any(want) or not tangents:
        return (None,) * ctx.n_inputs
    poses = torch.cat([s[0] for s in sets], 1) if ctx.n_sets > 1 else sets[0][0]
    grad = torch.cat([s[1] for s in sets], 1) if ctx.n_sets > 1 else sets[0][1]
    h = cost_hvp(*prob, poses, grad, *(tangents.get(k) for k in native.HVP_TANGENTS), ctx.dof, ctx.z_min, want)
    h = [t if w else None for t, w in zip(h, want)]
    out = list(_problem_grads(prob, h[:4], h[6:]))
    sizes = [s[1].shape[1] for s in sets]
    for i, (p, g) in enumerate(sets):
        lo = sum(sizes[:i])
        out.append(None if h[4] is None or not n[7 + 2 * i] else h[4][:, lo:lo + sizes[i]].to(p.dtype))
        out.append(None if h[5] is None or not n[8 + 2 * i] else h[5][:, lo:lo + sizes[i]].to(g.dtype))
    return tuple(out) + (None,) * (ctx.n_inputs - len(out))


def _cost_backward_backward(ctx, v_x3d, v_x2d, v_w2d, v_delta):
    return _cost_hvp_backward(ctx, dict(x3d=v_x3d, x2d=v_x2d, w2d=v_w2d, delta=v_delta))


def _cost_pose_backward_backward(ctx, v_pose):
    return _cost_hvp_backward(ctx, dict(pose=v_pose))


def _cost_camera_backward_backward(ctx, v_cam, v_lb, v_ub):
    return _cost_hvp_backward(ctx, dict(cam=v_cam, lb=v_lb, ub=v_ub))


_register_autograd(cost_backward, _cost_backward_backward, _cost_hvp_setup)
_register_autograd(cost_pose_backward, _cost_pose_backward_backward, _cost_hvp_setup)
_register_autograd(cost_camera_backward, _cost_camera_backward_backward, _cost_hvp_setup)


def _gn_plus_hvp_setup(ctx, inputs, output):
    """gn_plus_backward / gn_plus_camera_backward: the problem, the (detached) pose and grad_pose_plus."""
    ctx.set_materialize_grads(False)
    ctx.consts = inputs[9:13]                                                  # dof, z_min, eps, huber_eps
    _save_problem(ctx, inputs, inputs[7:9])


def _gn_plus_hvp_backward(ctx, tangents):
    """The gradients of a pose_opt_plus backward's inputs from the tangents of its outputs (a dict by
    native.GN_HVP_TANGENTS name): one gn_plus_hvp, then each output back to its input's shape.  The pose gets none."""
    prob, (pose, grad_plus) = _load_problem(ctx, 2)
    want_corr, want_cam = _problem_wants(ctx)
    want = list(want_corr) + list(want_cam) + [ctx.needs_input_grad[8]]
    tangents = {k: t for k, t in tangents.items() if t is not None and t.numel()}
    if not any(want) or not tangents:
        return (None,) * 14
    h = gn_plus_hvp(*prob, pose, grad_plus, *(tangents.get(k) for k in native.GN_HVP_TANGENTS), *ctx.consts, want)
    h = [t if w else None for t, w in zip(h, want)]
    g_plus = None if h[7] is None else h[7].to(grad_plus.dtype)
    return _problem_grads(prob, h[:4], h[4:7]) + (None, g_plus) + (None,) * 5


def _gn_plus_backward_backward(ctx, v_x3d, v_x2d, v_w2d, v_delta):
    return _gn_plus_hvp_backward(ctx, dict(x3d=v_x3d, x2d=v_x2d, w2d=v_w2d, delta=v_delta))


def _gn_plus_camera_backward_backward(ctx, v_cam, v_lb, v_ub):
    return _gn_plus_hvp_backward(ctx, dict(cam=v_cam, lb=v_lb, ub=v_ub))


_register_autograd(gn_plus_backward, _gn_plus_backward_backward, _gn_plus_hvp_setup)
_register_autograd(gn_plus_camera_backward, _gn_plus_camera_backward_backward, _gn_plus_hvp_setup)


def _mc_lse_backward_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs)


def _mc_lse_backward_backward(ctx, v):
    """out = grad_lse[b] exp(logw[b, m] - lse[b]) with lse an input of its own (its graph carries the softmax part):
    torch ops on (B, M), differentiable again."""
    logw_bm, lse, grad_lse = ctx.saved_tensors
    w = torch.exp(logw_bm - lse.unsqueeze(1))
    vo = v * w * grad_lse.unsqueeze(1)
    return vo, -vo.sum(1), (v * w).sum(1)


_register_autograd(mc_lse_backward, _mc_lse_backward_backward, _mc_lse_backward_setup)


FORWARD = (adaptive_delta, evaluate_cost, evaluate_full, lm_solve, lm_amis_fused, rslm_draw, rslm, epnp_init, mc_epilogue)
BACKWARD = (cost_backward, cost_pose_backward, cost_camera_backward, gn_plus_backward, gn_plus_camera_backward,
            evaluate_backward, mc_lse_backward)
SECOND_ORDER = (cost_hvp, gn_plus_hvp)
FORWARD_MODE = (evaluate_jvp,)
STACKED = (lm_solve_stacked,)                       # the solve from stacked starts, pose_init (S, B, D)
# operators whose outputs the layer never differentiates (the solver's start, the stacked solve): under forward AD their
# inputs' tangents are dropped, as reverse mode's no_grad drops the graph
_NO_DERIVATIVE = (rslm_draw, rslm, epnp_init, lm_solve_stacked)


@torch.compiler.disable
def _eager_call(fn, *args):
    """fn(*args) with torch.compile's frame evaluation off: when a compiled region falls back to running an entry point
    eagerly (its refusal of a forward tangent), the ctypes calls below must not be traced frame by frame."""
    return fn(*args)


def forward_tangent(*args):
    """An argument carries a forward-mode tangent (torch.autograd.forward_ad, torch.func.jvp) or is wrapped by a
    torch.func transform.  One module-attribute read when neither is active."""
    if _fwAD._current_level < 0 and not torch._C._are_functorch_transforms_active():
        return False
    for a in args:
        if torch.is_tensor(a) and (torch._C._functorch.is_functorch_wrapped_tensor(a)
                                   or (_fwAD._current_level >= 0 and _fwAD.unpack_dual(a).tangent is not None)):
            return True
    return False


def needs_derivative(*args):
    """The layer's one routing predicate: an argument needs the differentiable path -- reverse mode (grad enabled and
    requires_grad), a forward-mode tangent or a torch.func transform (forward_tangent).  Non-tensors are ignored."""
    if torch.is_grad_enabled() and any(torch.is_tensor(a) and a.requires_grad for a in args):
        return True
    return forward_tangent(*args)


def _entry(op):
    """The callable the layer uses for `op`.  While anything traces (torch.compile, torch.export, a torch-dispatch mode)
    it is the operator itself.  Eagerly it runs the operator's implementation directly and, when an input needs the
    gradient, under the operator's own autograd formula (_register_autograd); an operator without a formula is called
    as such, so that differentiating through it raises.  The direct call skips the dispatcher and custom_op's argument
    handling, whose eager host time per call is several small kernel launches' worth."""
    impl, eager, eager_func = _IMPLS[op], _EAGER.get(op), _EAGER_FUNC.get(op)
    name = op._name

    def dual_tangent(args):
        return _fwAD._current_level >= 0 and any(torch.is_tensor(a) and _fwAD.unpack_dual(a).tangent is not None
                                                 for a in args)

    def under_functorch(args):
        # torch.func.jvp / linearize: the tensors are functorch wrappers.  A call with a tangent at this level runs its
        # formula as an autograd.Function (functorch unwraps the forward's arguments); a call without one -- a formula's
        # own kernel call on the primals and tangents -- goes through the dispatcher, which unwraps its arguments before
        # the implementation.  So ctypes never sees a wrapper.
        if not dual_tangent(args):
            return op(*args)
        if eager is not None and "jvp" in vars(eager):
            return eager_func.apply(*args)
        if op in _NO_DERIVATIVE:
            return op(*(a.detach() if torch.is_tensor(a) else a for a in args))
        raise RuntimeError(f"{name} has no forward-mode formula: a tangent cannot pass through it (forward over "
                           "reverse is not supported)")

    def entry(*args):
        if torch.compiler.is_compiling():
            # the traced operator has no forward rule and would drop a tangent; the module attribute is traceable
            if _fwAD._current_level >= 0:
                raise RuntimeError(f"{name}: forward-mode tangents are not supported under torch.compile / "
                                   "torch.export; compute the JVP eagerly")
            return op(*args)
        if torch._C._len_torch_dispatch_stack():
            if forward_tangent(*args):
                # torch.func.linearize traces a forward-AD pass under make_fx's dispatch mode: the formulas run, and
                # their kernel calls are traced as operators
                if torch._C._are_functorch_transforms_active():
                    return under_functorch(args)
                if eager is not None and "jvp" in vars(eager):
                    return eager.apply(*args)
                raise RuntimeError(f"{name} has no forward-mode formula: a tangent cannot pass through it")
            return op(*args)
        if torch.is_grad_enabled() and any(torch.is_tensor(a) and a.requires_grad for a in args):
            if eager is None:
                return op(*args)
            return (eager_func if torch._C._are_functorch_transforms_active() else eager).apply(*args)
        if forward_tangent(*args):
            if torch._C._are_functorch_transforms_active():
                return under_functorch(args)
            if eager is not None and "jvp" in vars(eager):
                return _eager_call(eager.apply, *args)
            if op in _NO_DERIVATIVE:
                return _eager_call(impl, *(a.detach() if torch.is_tensor(a) else a for a in args))
            raise RuntimeError(f"{name} has no forward-mode formula: a tangent cannot pass through it (forward over "
                               "reverse is not supported)")
        return impl(*args)
    entry.op = op
    return entry


# the names the layer (and the formulas above) call; the operators stay in FORWARD / BACKWARD and torch.ops.epropnp
(adaptive_delta, evaluate_cost, evaluate_full, lm_solve, lm_amis_fused, rslm_draw, rslm, epnp_init,
 mc_epilogue) = (_entry(op) for op in FORWARD)
(cost_backward, cost_pose_backward, cost_camera_backward, gn_plus_backward, gn_plus_camera_backward, evaluate_backward,
 mc_lse_backward) = (_entry(op) for op in BACKWARD)
cost_hvp, gn_plus_hvp = (_entry(op) for op in SECOND_ORDER)
evaluate_jvp = _entry(evaluate_jvp)
lm_solve_stacked = _entry(lm_solve_stacked)
