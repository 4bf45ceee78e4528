"""Robust (Huber) reprojection cost objects with the reference's public surface (epropnp/cost_fun.py).

The solver kernels consume only two things from these objects: `.delta` (a float or a (B,) tensor, the
Huber threshold per object) and `.eps`.  `compute` is the stand-alone utility of the reference API for
callers that already hold projected points; it is a few elementwise torch ops and not what the solvers run.
"""
import torch

from epropnp_b200 import ops
from .builder import COSTFUN


def huber_kernel(s_sqrt, delta):
    """Half of the Huber loss, rho(s)/2, at residual norm `s_sqrt`: quadratic inside `delta`, linear outside."""
    quadratic = 0.5 * s_sqrt * s_sqrt
    linear = delta * s_sqrt - 0.5 * delta * delta
    return torch.where(s_sqrt <= delta, quadratic, linear)


def huber_d_kernel(s_sqrt, delta, eps: float = 1e-10):
    """sqrt(rho'(s)) = sqrt(min(delta / s, 1)): the factor that rescales residual and Jacobian (Triggs)."""
    ratio = delta / s_sqrt.clamp(min=eps)
    return ratio.clamp(max=1.0).sqrt()


def _deliver(slot, value, shape=None):
    """out_* convention of the reference: a tensor argument is filled in place (and returned)."""
    if shape is not None:
        value = value.reshape(shape)
    if torch.is_tensor(slot):
        slot.view(value.shape).copy_(value)
        return slot
    return value


class _DeltaHolder(object):
    """Batch-shape helpers shared by both cost classes; they only ever touch a tensor-valued delta."""

    def _apply(self, fn):
        if torch.is_tensor(self.delta):
            self.delta = fn(self.delta)
        return self

    def reshape_(self, *batch_shape):
        return self._apply(lambda d: d.reshape(*batch_shape))

    def expand_(self, *batch_shape):
        return self._apply(lambda d: d.expand(*batch_shape))

    def repeat_(self, *batch_repeat):
        return self._apply(lambda d: d.repeat(*batch_repeat))


@COSTFUN.register_module()
class HuberPnPCost(_DeltaHolder):

    def __init__(self, delta=1.0, eps=1e-10):
        self.delta = delta
        self.eps = eps

    def set_param(self, *args, **kwargs):
        """A fixed threshold has nothing to adapt."""
        return None

    def compute(self, x2d_proj, x2d, w2d, jac_cam=None, out_residual=False, out_cost=False, out_jacobian=False):
        """Weighted residual r = (proj - x2d) * w2d, cost sum_n rho(|r_n|)/2, and the robustly rescaled
        residual (*, 2n) / Jacobian (*, 2n, dof).  Each out_* may be False (skip), True or a tensor to fill."""
        batch, n_pts = x2d_proj.shape[:-2], x2d_proj.size(-2)
        thr = self.delta if torch.is_tensor(self.delta) else x2d.new_tensor(self.delta)
        thr = thr.unsqueeze(-1)
        weighted = (x2d_proj - x2d) * w2d
        norms = weighted.norm(dim=-1)

        cost = None
        if out_cost is not False:
            cost = _deliver(out_cost, huber_kernel(norms, thr).sum(dim=-1))

        residual = jacobian = None
        if out_residual is not False or out_jacobian is not False:
            gain = huber_d_kernel(norms, thr, eps=self.eps).unsqueeze(-1)
            if out_residual is not False:
                residual = _deliver(out_residual, weighted * gain, batch + (n_pts * 2,))
            if out_jacobian is not False:
                if jac_cam is None:
                    raise AssertionError("jac_cam is required for out_jacobian")
                dof = jac_cam.size(-1)
                jacobian = _deliver(out_jacobian, jac_cam * (w2d * gain).unsqueeze(-1), batch + (n_pts * 2, dof))
        return residual, cost, jacobian

    def shallow_copy(self):
        return HuberPnPCost(delta=self.delta, eps=self.eps)


@COSTFUN.register_module()
class AdaptiveHuberPnPCost(HuberPnPCost):
    """Huber threshold tied to the data: delta_b = relative_delta * mean(w2d_b) * std(x2d_b)."""

    def __init__(self, delta=None, relative_delta=0.5, eps=1e-10):
        HuberPnPCost.__init__(self, delta=delta, eps=eps)
        self.relative_delta = relative_delta

    def set_param(self, x2d, w2d):
        needs_graph = ops.needs_derivative(x2d, w2d)
        if x2d.is_cuda and x2d.dim() == 3 and not needs_graph:
            self.delta = ops.adaptive_delta(x2d, w2d, float(self.relative_delta)).to(x2d.dtype)   # one native kernel
            return
        # differentiable / generic-shape path: the same formula in torch so autograd reaches w2d (and x2d)
        spread = torch.var(x2d, dim=-2).sum(dim=-1).sqrt()
        self.delta = self.relative_delta * w2d.mean(dim=(-2, -1)) * spread

    def shallow_copy(self):
        return AdaptiveHuberPnPCost(delta=self.delta, relative_delta=self.relative_delta, eps=self.eps)
