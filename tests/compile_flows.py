"""The four call sequences the torch.compile / torch.export tests run (tests/test_compile_simt_cpu.py,
tests/test_compile_gpu.py), each built fresh so an eager and a compiled copy hold no shared state:

    det_infer   the Det test path (deform_pnp_head.py test_post): camera / cost set_param, pnp(fast_mode=True) with RSLM
                init, evaluate_pnp(out_cost=True) over an orientation grid
    det_train   the Det training step: set_param on scaled weights, monte_carlo_forward(pose_init=gt,
                force_init_solve=True), MonteCarloPoseLoss, pnp(with_pose_opt_plus=True); 4DoF, normalize=True
    train6      the 6DoF training step: RSLM init, force_init_solve, with_pose_opt_plus, MonteCarloPoseLoss
    test6       the 6DoF test path: EPnPSolver + Gauss-Newton (3 iterations, fast_mode)

build(kind, dev, B, N, ...) -> Flow(fn, args, leaves): fn(*args) returns a tuple of tensors, the first of them the loss
for the training flows; `leaves` are the args whose gradients the tests compare.  seeds="int": fixed ints;
"tensor": the last two args are one-element int64 seed tensors (AMIS, RSLM) on `dev`; "none": fresh seeds per call
(common.philox_seed)."""
import collections
import math

import torch

from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.epnp import EPnPSolver
from epropnp.epropnp import EProPnP4DoF, EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
from epropnp_b200.synth import make_problem

Flow = collections.namedtuple("Flow", "fn args leaves")
KINDS = ("det_infer", "det_train", "train6", "test6")


class SeededRSLM(RSLMSolver):
    """RSLMSolver whose native draws take the seed set on it (an int or a seed tensor)."""
    seed = 0

    def solve(self, *args, **kwargs):
        return super().solve(*args, rslm_seed=self.seed, **kwargs)


def build(kind, dev, B, N, M=64, P=8, data_seed=1, seeds="int", cluster_split=False):
    dof = 6 if kind in ("train6", "test6") else 4
    pc = make_problem(B, N, seed=data_seed, dof=dof)
    t = lambda k: pc[k].to(dev)
    x3d, x2d, w2d, cam, gt = t("x3d"), t("x2d"), t("w2d"), t("cam_mats"), t("pose_gt")
    rslm = SeededRSLM(dof=dof, num_points=8, num_proposals=P, num_iter=3, cluster_split=cluster_split)
    rslm.seed, amis_seed = (7, 11) if seeds == "int" else (None, None)
    seeds = ((torch.tensor([11], dtype=torch.int64, device=dev), torch.tensor([7], dtype=torch.int64, device=dev))
             if seeds == "tensor" else ())
    camera = PerspectiveCamera(z_min=0.5 if dof == 4 else 0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)

    def use_seeds(s):
        if s:
            rslm.seed = s[1]
            return s[0]
        return amis_seed

    if kind == "det_infer":
        layer = EProPnP4DoF(mc_samples=M, num_iter=4, normalize=True,
                            solver=LMSolver(dof=4, num_iter=10, normalize=True, init_solver=rslm))
        img_shape = torch.tensor([[480.0, 640.0]], device=dev).expand(B, 2)
        yaw = torch.linspace(0, 2 * math.pi * 7 / 8, 8, device=dev)

        def fn(x3d, x2d, w2d, cam, img_shape, yaw, *s):
            use_seeds(s)
            camera.set_param(cam, img_shape=img_shape)
            cost_fun.set_param(x2d, w2d)
            pose_opt = layer(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]
            grid = torch.cat((pose_opt[None, :, :3].expand(yaw.shape[0], -1, -1),
                              yaw[:, None, None].expand(-1, pose_opt.shape[0], 1)), dim=-1)
            cost = evaluate_pnp(x3d, x2d, w2d, grid, camera, cost_fun, out_cost=True)[1]
            return pose_opt, cost
        return Flow(fn, (x3d, x2d, w2d, cam, img_shape, yaw) + seeds, ())

    if kind == "det_train":
        layer = EProPnP4DoF(mc_samples=M, num_iter=4, normalize=True,
                            solver=LMSolver(dof=4, num_iter=10, normalize=True, init_solver=rslm))
        loss_fn = MonteCarloPoseLoss(loss_weight=0.5, sync_norm_factor=False).to(dev)
        img_shape = torch.tensor([[480.0, 640.0]], device=dev).expand(B, 2)
        x3d, w2d = x3d.clone().requires_grad_(True), w2d.clone().requires_grad_(True)
        scale = torch.full((B, 1, 2), 1.5, device=dev, requires_grad=True)

        def fn(x3d, x2d, w2d, scale, cam, img_shape, gt, *s):
            seed = use_seeds(s)
            camera.set_param(cam, img_shape=img_shape)
            w2d_s = w2d * scale
            cost_fun.set_param(x2d.detach(), w2d_s)
            _, _, _, _, logw, cost_tgt = layer.monte_carlo_forward(x3d, x2d, w2d_s, camera, cost_fun, pose_init=gt,
                                                                   force_init_solve=True, amis_seed=seed)
            loss = loss_fn(logw, cost_tgt, torch.ones((), device=x3d.device))
            cost_fun.delta = cost_fun.delta.detach()
            plus = layer(x3d, x2d, w2d * scale.detach(), camera, cost_fun, with_pose_opt_plus=True)[3]
            loss = loss + (plus[:, :3] - gt[:, :3]).norm(dim=-1).mean()
            return loss, logw, cost_tgt, plus
        return Flow(fn, (x3d, x2d, w2d, scale, cam, img_shape, gt) + seeds, (0, 2, 3))

    if kind == "train6":
        layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=10, init_solver=rslm))
        loss_fn = MonteCarloPoseLoss().to(dev)
        x3d, x2d, w2d = (v.clone().requires_grad_(True) for v in (x3d, x2d, w2d))

        def fn(x3d, x2d, w2d, cam, gt, *s):
            seed = use_seeds(s)
            camera.set_param(cam)
            cost_fun.set_param(x2d.detach(), w2d)
            _, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(
                x3d, x2d, w2d, camera, cost_fun, pose_init=gt, force_init_solve=True, with_pose_opt_plus=True,
                amis_seed=seed)
            loss = loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - gt).abs().sum()
            return loss, logw, cost_tgt, plus
        return Flow(fn, (x3d, x2d, w2d, cam, gt) + seeds, (0, 1, 2))

    layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=3, init_solver=EPnPSolver()))

    def fn(x3d, x2d, w2d, cam, *s):
        camera.set_param(cam)
        cost_fun.set_param(x2d, w2d)
        return (layer(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0],)
    return Flow(fn, (x3d, x2d, w2d, cam), ())


def run(flow, fn=None, backward=True):
    """-> outputs (detached) and the leaves' gradients (training flows), leaves' grads cleared first."""
    for i in flow.leaves:
        flow.args[i].grad = None
    out = (fn or flow.fn)(*flow.args)
    grads = []
    if backward and flow.leaves:
        out[0].backward()
        grads = [flow.args[i].grad.clone() for i in flow.leaves]
    return [o.detach().clone() for o in out], grads
