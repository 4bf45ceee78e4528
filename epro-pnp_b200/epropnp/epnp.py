"""EPnPSolver: the EPnP initialisation of the reference's 6DoF test loop (EPro-PnP-6DoF/lib/test.py:178-194) as an
`init_solver` of LMSolver, executing on the native sm_90a kernel (epnp_epnp_init_f32, one launch, no host round trip;
objects larger than one SM holds, such as the 16,384 points of a 128 x 128 coordinate map, take its cluster-split form
epnp_epnp_init_split_f32, up to epnp_max_points_split(6, 0, 0)).

    solver = LMSolver(dof=6, num_iter=3, init_solver=EPnPSolver(conf_quantile=0.8))
    pose_opt = EProPnP6DoF(solver=solver)(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]   # pose_init=None

The reference keeps, per object, the points whose confidence w2d.mean(-1) reaches np.quantile(conf, 0.8), runs
cv2.solvePnP(..., flags=cv2.SOLVEPNP_EPNP) on them on the host and converts the result to a [w, i, j, k] quaternion; the
kernel does the same on the device.  EPnP is 6-DoF only: as the init solver of a 4-DoF LMSolver its 7-wide pose is
refused with ValueError at the first solve.
"""
import torch
import torch.nn as nn

from epropnp_b200 import ops
from . import autograd
from .builder import PNP


@PNP.register_module()
class EPnPSolver(nn.Module):
    """EPnP (Lepetit et al., IJCV 2009) on the most confident correspondences of every object.

    conf_quantile: a point is used when mean(w2d[i]) >= np.quantile(mean(w2d, -1), conf_quantile); 0 uses every
    point.  The camera's bounds and z_min play no part, as in cv2's EPnP."""

    def __init__(self, conf_quantile=0.8):
        super(EPnPSolver, self).__init__()
        if not 0.0 <= float(conf_quantile) <= 1.0:
            raise ValueError(f"conf_quantile must lie in [0, 1], got {conf_quantile}")
        self.conf_quantile = float(conf_quantile)

    @torch.no_grad()
    def solve(self, x3d, x2d, w2d, camera, cost_fun, with_cost=False, **kwargs):
        """-> pose (B, 7), None, cost (B) | None.  With with_cost, the cost is evaluate_pnp's at the EPnP pose (what
        LMSolver compares against pose_init under force_init_solve)."""
        pose = ops.epnp_init(x3d.detach(), x2d.detach(), w2d.detach(), camera.cam_mats, self.conf_quantile)
        cost = None
        if with_cost:
            cost = ops.evaluate_cost(*autograd._problem_args(x3d, x2d, w2d, camera, cost_fun), pose[None], 6,
                                     float(camera.z_min))[0].to(x2d.dtype)
        return pose.to(x2d.dtype), None, cost
