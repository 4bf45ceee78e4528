"""Cluster-split backward of pose_opt_plus (epnp_gn_plus_backward_split_f32): the derivative-regularisation term of
training on objects with more points than one SM holds, each spread over a thread-block cluster of 2..8 CTAs.  Against
the float64 composite (torch autograd through PerspectiveCamera.project + HuberPnPCost.compute + linalg.solve +
pose_add), against the resident kernel where both run, for determinism and batch independence, end to end through
EProPnP6DoF.monte_carlo_forward with the reference's training loss, and for the refusals."""
import numpy as np
import pytest
import torch

from conftest import err_stats, err_vs, record_parity
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

K_FLOOR = 5         # the bound against the float64 composite: max(1e-4, K_FLOOR * floor)
EPS, HUBER_EPS = 1e-5, 1e-10


def composite_grads(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, gplus, dof, z_min, dtype):
    """dL/d(x3d, x2d, w2d, delta) of L = <gplus, pose (+) gn_step(pose)> by torch autograd through the composite, in
    `dtype`, on the inputs' device."""
    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
    x3d, x2d, w2d, d = leaf(x3d), leaf(x2d), leaf(w2d), leaf(delta)
    cast = lambda t: None if t is None else t.to(dtype)
    camera = PerspectiveCamera(cam_mats=cast(cam_mats), z_min=z_min, lb=cast(lb), ub=cast(ub))
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1, eps=HUBER_EPS)
    cost_fun.delta = d
    solver = LMSolver(dof=dof, eps=EPS)
    pose = pose.detach().to(dtype)
    plus = solver.pose_add(pose, ag.gn_step_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun), camera)
    (plus * gplus.to(dtype)).sum().backward()
    return [t.grad for t in (x3d, x2d, w2d, d)]


def train_bounds(x2d):
    """Camera lb / ub as EPro-PnP-6DoF/lib/train.py:169-174 sets them: the coordinate map's pixel window widened by 30
    pixel steps on every side."""
    side = round(x2d.shape[1] ** 0.5)
    lo, hi = x2d.amin(1), x2d.amax(1)
    border = 30 * (hi - lo) / (side - 1)
    return lo - border, hi + border


def setup(dev, dof, B, N, seed, bounds=True, outlier_frac=0.0):
    dense = dof == 6 and round(N ** 0.5) ** 2 == N
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, dof=dof, grid2d=dense,
                                                outlier_frac=outlier_frac).items()}
    lb, ub = train_bounds(pc["x2d"]) if bounds else (None, None)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.1)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta)
    gp = torch.randn(B, 7 if dof == 6 else 4, generator=torch.Generator().manual_seed(seed)).to(dev)
    return pc, prob, gp


def split_call(prob, pose, gp, dof, ctas=0, z_min=0.01):
    return native.gn_plus_backward_split(prob, pose, gp, dof, z_min, EPS, HUBER_EPS, cluster_ctas=ctas)


def check_against_composite(dev, dof, B, N, seed, ctas=0, record=None, against_resident=False, outlier_frac=0.0):
    """Split backward within max(1e-4, K_FLOOR * floor) of the float64 composite, floor = the fp32 composite against
    the fp64 one; against_resident: within max(1e-5, 3 * floor) of the resident kernel."""
    pc, prob, gp = setup(dev, dof, B, N, seed, outlier_frac=outlier_frac)
    pose = pc["pose_init"]
    out = split_call(prob, pose, gp, dof, ctas)
    args = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], prob.lb, prob.ub, prob.delta, pose, gp, dof, 0.01)
    c64 = composite_grads(*args, torch.float64)
    c32 = composite_grads(*args, torch.float32)
    res = native.gn_plus_backward(prob, pose, gp, dof, 0.01, EPS, HUBER_EPS) if against_resident else None
    stats = {}
    for i, what in enumerate(("x3d", "x2d", "w2d", "delta")):
        g, g64 = out[i].cpu().numpy(), c64[i].cpu().numpy()
        floor = err_vs(c32[i].cpu().numpy(), g64)
        assert np.isfinite(g).all(), what
        assert err_vs(g, g64) < max(1e-4, K_FLOOR * floor), (what, err_vs(g, g64), floor)
        if res is not None:
            assert err_vs(g, res[i].cpu().numpy()) < max(1e-5, 3 * floor), (what, floor)
        stats[f"grad_{what}_vs_f64"] = err_stats(g, g64)
        stats[f"f32_composite_vs_f64_{what}"] = err_stats(c32[i].cpu().numpy(), g64)
    if record:
        record_parity(record, cluster_ctas=ctas or native.split_ctas(dof, N), bound_k=K_FLOOR, **stats)
    return out


# ------------------------------------------------------------------------------------------------
def test_split_against_composite_dense_128(cuda_device):
    """out_res = 128: N = 16,384 points per object, beyond what one SM holds; the automatic cluster size."""
    assert 16384 > native.max_points(6) and native.split_ctas(6, 16384) >= 2
    check_against_composite(cuda_device, 6, 4, 16384, seed=3, record="gn_plus_split/6dof_B4_N16384")


def test_split_against_composite_4dof(cuda_device):
    check_against_composite(cuda_device, 4, 4, 10004, seed=5, record="gn_plus_split/4dof_B4_N10004", outlier_frac=0.1)


def test_split_c2_against_resident(cuda_device):
    """At N = 4,096 both forms run: the split one on two CTAs against the resident kernel, both near the composite."""
    check_against_composite(cuda_device, 6, 8, 4096, seed=7, ctas=2, against_resident=True,
                            record="gn_plus_split/6dof_B8_N4096_C2")


def test_split_deterministic_and_batch_independent(cuda_device):
    """Same inputs, same bits; an object's gradient rows and grad_delta do not depend on the batch around it."""
    dev, B, N = cuda_device, 257, 16384
    pc, prob, gp = setup(dev, 6, B, N, seed=9)
    a = split_call(prob, pc["pose_init"], gp, 6)
    b = split_call(prob, pc["pose_init"], gp, 6)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert all(torch.isfinite(x).all() for x in a)
    for i in (0, 128, 256):
        s = slice(i, i + 1)
        one = native.Problem(pc["x3d"][s], pc["x2d"][s], pc["w2d"][s], pc["cam_mats"][s], prob.lb[s], prob.ub[s],
                             prob.delta[s])
        o = split_call(one, pc["pose_init"][s], gp[s], 6)
        for x, y in zip(o, a):
            assert torch.equal(x[0], y[i]), i


def test_training_objective_end_to_end_at_16384(cuda_device, monkeypatch):
    """EProPnP6DoF.monte_carlo_forward on 16,384-point objects with the reference's training loss (lib/train.py:182-193:
    Monte-Carlo pose loss + loss_t + loss_r on pose_opt_plus): backward() succeeds with finite gradients, which equal
    cost_backward + gn_plus_backward_split called directly, and agree with the EPNP_NATIVE_GN_STEP=0 composite."""
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    dev, B, N, M, I = cuda_device, 2, 16384, 512, 4
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=17, grid2d=True).items()}
    lb, ub = train_bounds(pc["x2d"])
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.01, lb=lb, ub=ub)
    layer = EProPnP6DoF(mc_samples=M, num_iter=I, solver=LMSolver(dof=6, num_iter=3))
    mc_loss = MonteCarloPoseLoss().to(dev)
    pose_gt = pc["pose_gt"]

    def run(native_step):
        monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1" if native_step else "0")
        x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
        cost_fun.set_param(pc["x2d"], pc["w2d"])
        cost_fun.delta = cost_fun.delta.detach().clone().requires_grad_(True)
        pose_opt, _, plus, samples, logw, cost_tgt = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=pc["pose_init"], force_init_solve=False,
            with_pose_opt_plus=True, fast_mode=True, amis_seed=5)
        loss_mc = mc_loss(logw, cost_tgt, torch.tensor(1.0, device=dev))
        loss_t = (plus[:, :3] - pose_gt[:, :3]).norm(dim=-1)
        beta = 0.05
        loss_t = torch.where(loss_t < beta, 0.5 * loss_t.square() / beta, loss_t - 0.5 * beta).mean()
        dot_quat = (plus[:, None, 3:] @ pose_gt[:, 3:, None]).squeeze(-1).squeeze(-1)
        loss_r = ((1 - dot_quat.square()) * 2).mean()
        loss = loss_mc + loss_t + loss_r
        ups = torch.autograd.grad(loss, [logw, cost_tgt, plus], retain_graph=True)
        loss.backward()
        grads = [t.grad for t in (x3d, x2d, w2d, cost_fun.delta)]
        return grads, ups, pose_opt.detach(), samples.detach(), cost_fun.delta.detach()

    grads, (g_logw, g_cost, g_plus), pose_opt, samples, delta = run(True)
    for g in grads:
        assert torch.isfinite(g).all() and g.abs().sum() > 0
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta)
    mc = native.cost_backward(prob, 6, 0.01, samples.transpose(0, 1).contiguous(), -g_logw.transpose(0, 1).contiguous(),
                              pc["pose_init"].reshape(B, 1, 7), g_cost.reshape(B, 1))
    gn = split_call(prob, pose_opt, g_plus, 6)
    for a, b, c in zip(grads, mc, gn):
        assert err_vs(a.cpu(), (b + c).cpu()) < 1e-6
    comp, *_ = run(False)
    args = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta, pose_opt, g_plus, 6, 0.01)
    c64, c32 = composite_grads(*args, torch.float64), composite_grads(*args, torch.float32)
    for a, b, g64, g32 in zip(grads, comp, c64, c32):
        floor = err_vs(g32.cpu().numpy(), g64.cpu().numpy())
        assert err_vs(a.cpu().numpy(), b.cpu().numpy()) < max(1e-4, K_FLOOR * floor), floor


def test_refusals(cuda_device):
    """Above epnp_max_points_split(dof, 0, 0) the split call refuses; the resident call keeps refusing 16,384 points;
    a cluster size outside [minimum, 8] is a bad argument."""
    dev = cuda_device

    def prob_of(N, B=1):
        z = lambda *s: torch.zeros(*s, device=dev)
        return native.Problem(z(B, N, 3), z(B, N, 2), z(B, N, 2), torch.eye(3, device=dev)[None].repeat(B, 1, 1), None,
                              None, 1.0), z(B, 7)
    big, pose = prob_of(native.max_points_split(6) + 64)
    with pytest.raises(native.NativeError, match="shared memory"):
        split_call(big, pose, pose, 6)
    mid, pose = prob_of(16384)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.gn_plus_backward(mid, pose, pose, 6, 0.01, EPS, HUBER_EPS)
    for bad in (1, 9, -1):
        with pytest.raises(native.NativeError, match="bad argument"):
            split_call(mid, pose, pose, 6, bad)
