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
mc_epilogue; the backward operators themselves have none.  evaluate_full's residual / Jacobian are first-order only: a
second backward through them raises.

The module's names (adaptive_delta, ..., mc_lse_backward) are the entry points the layer calls (_entry): the operator
while anything traces, its implementation directly in eager code.  The operators themselves are FORWARD / BACKWARD and
torch.ops.epropnp.*; each entry point's `.op` is its operator.
"""
from typing import List, Optional

import torch
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


def _register_autograd(op, backward, setup_context):
    """op.register_autograd, and the same two functions as an autograd.Function that runs the implementation directly:
    the eager driver of the formula (see _entry)."""
    op.register_autograd(backward, setup_context=setup_context)
    impl = _IMPLS[op]

    def forward(ctx, *args):
        out = impl(*args)
        setup_context(ctx, args, out)
        return out
    _EAGER[op] = type(f"epropnp_{op._name.split('::')[-1]}", (torch.autograd.Function,),
                      dict(forward=staticmethod(forward), backward=staticmethod(backward)))


def _save_problem(ctx, inputs, extra=()):
    x3d, x2d, w2d, cam_mats, lb, ub, delta = inputs[:7]
    ctx.bounded = _bounded(lb, ub)
    ctx.has_lb, ctx.has_ub = lb is not None, ub is not None
    saved = [x3d, x2d, w2d, cam_mats, delta] + [t for t in (lb, ub) if t is not None]
    ctx.save_for_backward(*saved, *extra)


def _load_problem(ctx, n_extra=0):
    """-> the seven problem inputs (detached: the backward operators are first-order) and the extra saved tensors."""
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
    """Correspondence / delta and camera gradients of sum_p grad[p] * cost(pose p) (two native launches at most)."""
    want_corr, want_cam = _problem_wants(ctx)
    d = lambda t: None if t is None else t.detach()
    p = tuple(d(t) for t in prob)
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
    poses_bm = poses.detach().transpose(0, 1).contiguous()                       # object-major (B, S, D)
    g = g_cost.transpose(0, 1).contiguous()                                        # object-major (B, S)
    grads = _cost_grads(ctx, prob, poses_bm, g)
    gpose = None
    if ctx.needs_input_grad[7]:
        d = tuple(None if t is None else t.detach() for t in prob)
        gpose = cost_pose_backward(*d, poses_bm, g, ctx.dof, ctx.z_min).transpose(0, 1).to(poses.dtype) \
            .reshape(poses.shape)
    return grads + (gpose, None, None)


_register_autograd(evaluate_cost, _evaluate_cost_backward, _evaluate_cost_setup)


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


_register_autograd(evaluate_full, _evaluate_full_backward, _evaluate_full_setup)


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
        poses_b = cost_init_pose.detach().reshape(B, 1, -1)
        grad_b = g_cost_init.reshape(B, 1)
    if g_logw is None:
        g_logw = torch.zeros(B, samples.shape[1], device=samples.device)
    grads = _cost_grads(ctx, prob, samples, -g_logw.contiguous(), poses_b, grad_b)
    gpose = None
    if ctx.has_ci and ctx.needs_input_grad[8] and poses_b is not None:
        d = tuple(None if t is None else t.detach() for t in prob)
        gpose = cost_pose_backward(*d, poses_b, grad_b, ctx.dof, ctx.z_min)[:, 0].to(extra[1].dtype) \
            .reshape(extra[1].shape)
    return grads + (None, gpose) + (None,) * 10


_register_autograd(lm_amis_fused, _fused_backward, _fused_setup)


def gn_plus_grads(prob, pose, grad_plus, dof, z_min, eps, huber_eps, needs):
    """Gradients of the seven problem inputs (argument order; None where `needs` is False) through pose_opt_plus =
    pose (+) gn_step(pose): the gn_plus backward operators, then the reduction to each input's shape."""
    lb_ub = prob[4] is not None and prob[5] is not None
    corr_w = (needs[0], needs[1], needs[2], needs[6])
    cam_w = (needs[3], lb_ub and needs[4], lb_ub and needs[5])
    d = tuple(None if t is None else t.detach() for t in prob)
    pose = pose.detach()
    corr = (None,) * 4
    if any(corr_w):
        out = gn_plus_backward(*d, pose, grad_plus, dof, z_min, eps, huber_eps, list(corr_w))
        corr = tuple(t if w else None for t, w in zip(out, corr_w))
    cam = (None,) * 3
    if any(cam_w):
        out = gn_plus_camera_backward(*d, pose, grad_plus, dof, z_min, eps, huber_eps, list(cam_w))
        cam = tuple(t if w else None for t, w in zip(out, cam_w))
    return _problem_grads(prob, corr, cam)


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


_register_autograd(lm_solve, _lm_solve_backward, _lm_solve_setup)


def _mc_epilogue_setup(ctx, inputs, output):
    ctx.mark_non_differentiable(*output[1:])
    ctx.save_for_backward(inputs[0], output[0])


def _mc_epilogue_backward(ctx, g_lse, g_loss, g_weights, g_score):
    logw_bm, lse = ctx.saved_tensors
    g = None
    if g_lse is not None and ctx.needs_input_grad[0]:
        g = mc_lse_backward(logw_bm.detach(), lse, g_lse).to(logw_bm.dtype)
    return (g,) + (None,) * 7


_register_autograd(mc_epilogue, _mc_epilogue_backward, _mc_epilogue_setup)


FORWARD = (adaptive_delta, evaluate_cost, evaluate_full, lm_solve, lm_amis_fused, rslm_draw, rslm, epnp_init, mc_epilogue)
BACKWARD = (cost_backward, cost_pose_backward, cost_camera_backward, gn_plus_backward, gn_plus_camera_backward,
            evaluate_backward, mc_lse_backward)


def _entry(op):
    """The callable the layer uses for `op`.  While anything traces (torch.compile, torch.export, a torch-dispatch mode)
    it is the operator itself.  Eagerly it runs the operator's implementation directly and, when an input needs the
    gradient, under the operator's own autograd formula (_register_autograd); an operator without a formula is called
    as such, so that differentiating through it raises.  The direct call skips the dispatcher and custom_op's argument
    handling, whose eager host time per call is several small kernel launches' worth."""
    impl, eager = _IMPLS[op], _EAGER.get(op)

    def entry(*args):
        if torch.compiler.is_compiling() or torch._C._len_torch_dispatch_stack():
            return op(*args)
        if torch.is_grad_enabled() and any(torch.is_tensor(a) and a.requires_grad for a in args):
            return op(*args) if eager is None else eager.apply(*args)
        return impl(*args)
    entry.op = op
    return entry


# the names the layer (and the formulas above) call; the operators stay in FORWARD / BACKWARD and torch.ops.epropnp
(adaptive_delta, evaluate_cost, evaluate_full, lm_solve, lm_amis_fused, rslm_draw, rslm, epnp_init,
 mc_epilogue) = (_entry(op) for op in FORWARD)
(cost_backward, cost_pose_backward, cost_camera_backward, gn_plus_backward, gn_plus_camera_backward, evaluate_backward,
 mc_lse_backward) = (_entry(op) for op in BACKWARD)
