"""The cluster-split RSLM initialiser (epnp_rslm_split_f32) on an H100.

  * Against the resident kernel at N = 512, 4 096 and max_points(dof): pose_all bit-identical to rslm_kernel's, cost_all
    bit-identical to evaluate_cost_split's on those poses and within fp32 summation order of the resident costs, the
    same winner or a cost-equivalent one; every cluster size from the minimum to 8, both DOF, LM and fast mode.
  * At N = 16 384 (automatic C = 3) with subsets drawn from the first 7 000 points: pose_all bit-identical to the
    resident kernel on the truncated object; every cost held to the float64 oracle's cost of the same pose.
  * Parity with the unmodified reference's goldens through the split path (native call and RSLMSolver).
  * The reference's 6DoF training step at N = 16 384 with cluster_split=True, eager and under CUDA-graph capture; the
    default RSLMSolver still refuses that size.
"""
import math

import numpy as np
import pytest
import torch

from conftest import err_stats, record_parity
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.epropnp import EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
from epropnp_b200 import native
from epropnp_b200.synth import make_problem
from oracle import pnp_oracle as orc
from test_graph_capture_gpu import _SeededRSLM, _check_replays_match_eager
from test_oracle_rslm_cpu import RSLM_CASES, load_rslm
from test_rslm_parity_gpu import _Playback, _check_object_level, _hypothesis_agreement, _problem

pytestmark = pytest.mark.gpu

COST_MIN, COST_K = 1e-4, 5.0        # bound on |cost - float64 cost| / |float64 cost|: max(MIN, K x the float32 floor)


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return torch.equal(bits(a), bits(b))


def _setup(dev, dof, B, N, P, n, seed, bounds=False, z_min=0.1, draw_from=None):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.2)
    d = {k: v.to(dev) for k, v in pc.items()}
    lb = ub = None
    if bounds:
        lb = torch.tensor([[260.0, 190.0]], device=dev).repeat(B, 1)
        ub = torch.tensor([[380.0, 290.0]], device=dev).repeat(B, 1)
    delta = native.adaptive_delta(d["x2d"], d["w2d"], 0.1)
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], lb, ub, delta)
    m = draw_from or N
    inds, start = native.rslm_draw(d["x3d"][:, :m], d["x2d"][:, :m], d["w2d"][:, :m], d["cam_mats"], P, n, dof,
                                   seed=seed + 1)
    return d, prob, inds, start, (lb, ub)


def _depths(d, dof):
    pose = d["pose_gt"]
    R = orc.pose_rotmat(pose)
    return (d["x3d"] @ R.transpose(-1, -2) + pose[:, None, :3])[..., 2]


@pytest.mark.parametrize("dof", [6, 4])
@pytest.mark.parametrize("fast", [0, 1])
@pytest.mark.parametrize("N", [512, 4096, "max"])
def test_against_the_resident_kernel(cuda_device, dof, fast, N):
    N = native.max_points(dof) if N == "max" else N
    B, P, n = 4, 64, 16
    d, prob, inds, start, _ = _setup(cuda_device, dof, B, N, P, n, seed=N + dof)
    params = native.default_params(dof, lm_iter=3, fast_mode=fast, z_min=0.1)
    res = native.rslm(prob, inds, start, params, want_all=True)
    c_min = native.split_ctas(dof, N)
    assert 2 <= c_min <= 8
    for C in range(c_min, 9):
        out = native.rslm_split(prob, inds, start, params, want_all=True, cluster_ctas=C)
        assert same(out["pose_all"], res["pose_all"]), C
        assert same(out["cost_all"], native.evaluate_cost_split(prob, out["pose_all"], dof, 0.1, C)), C
        finite = torch.isfinite(res["cost_all"])
        assert finite.float().mean() > 0.9 and torch.equal(finite, torch.isfinite(out["cost_all"]))
        rel = ((out["cost_all"] - res["cost_all"]).abs() / res["cost_all"].abs())[finite]
        assert rel.max() < 2e-5, (C, float(rel.max()))
        same_winner = (out["cost"] == out["cost_all"].gather(0, res["cost_all"].argmin(0, keepdim=True))[0])
        crel = (out["cost"] - res["cost"]).abs() / res["cost"].abs()
        both_nan = out["cost"].isnan() & res["cost"].isnan()
        assert (same_winner | (crel < 2e-5) | both_nan).all(), (C, crel)
        rows = torch.arange(B, device=cuda_device)
        win = out["cost_all"].argmin(0)
        assert same(out["cost"], out["cost_all"][win, rows]) and same(out["pose"], out["pose_all"][win, rows])


@pytest.mark.parametrize("case", ["plain", "bounded_below_zmin"])
def test_16384_points_against_truncated_resident_and_float64(cuda_device, case):
    dof, B, N, P, n, M = 6, 4, 16384, 64, 16, 7000
    assert native.max_points(dof) == M and native.split_ctas(dof, N) == 3
    bounded = case != "plain"
    d, prob, inds, start, (lb, ub) = _setup(cuda_device, dof, B, N, P, n, seed=31, bounds=bounded, draw_from=M)
    z_min = 0.1
    if bounded:                     # at the true pose, some points lie in front of z_min and some behind
        z_min = float(_depths(d, dof).median())
    params = native.default_params(dof, lm_iter=3, z_min=z_min)
    out = native.rslm_split(prob, inds, start, params, want_all=True)
    assert same(out["cost_all"], native.evaluate_cost_split(prob, out["pose_all"], dof, z_min, 3))
    trunc = native.Problem(d["x3d"][:, :M], d["x2d"][:, :M], d["w2d"][:, :M], d["cam_mats"], lb, ub, prob.delta)
    res = native.rslm(trunc, inds, start, params, want_all=True)
    assert same(out["pose_all"], res["pose_all"])
    # every cost against the float64 oracle's cost of the same pose
    f64 = torch.float64
    cam64 = orc.Camera(d["cam_mats"].to(f64), z_min, None if lb is None else lb.to(f64), None if ub is None else ub.to(f64))
    pose = out["pose_all"]
    c64 = orc.evaluate(d["x3d"].to(f64), d["x2d"].to(f64), d["w2d"].to(f64), pose.to(f64), cam64, prob.delta.to(f64))["cost"]
    cam32 = orc.Camera(d["cam_mats"], z_min, lb, ub)
    c32 = orc.evaluate(d["x3d"], d["x2d"], d["w2d"], pose, cam32, prob.delta)["cost"]
    finite = torch.isfinite(c64)
    assert finite.all()
    floor = ((c32.to(f64) - c64).abs() / c64.abs()).max(0).values             # per object
    err = (out["cost_all"].to(f64) - c64).abs() / c64.abs()
    bound = torch.clamp(COST_K * floor, min=COST_MIN)
    assert (err <= bound[None]).all(), (err.max(0).values, bound)
    if bounded:
        # the bounds clamp and the depth clamp both act at the poses scored
        assert (_depths(d, dof) < z_min).float().mean() > 0.05
    record_parity(f"rslm_split/16384/{case}", cost_rel_vs_float64=err_stats(out["cost_all"].cpu().numpy(), c64.cpu().numpy()),
                  float32_floor_max=float(floor.max()))


@pytest.mark.parametrize("name", RSLM_CASES)
def test_split_path_against_reference_goldens(cuda_device, name, monkeypatch):
    g = load_rslm(name)
    dev = cuda_device
    prob, lb, ub = _problem(g, dev)
    dof, P, n = int(g["dof"]), int(g["P"]), int(g["n"])
    params = native.default_params(dof, lm_iter=int(g["rs_iter"]), fast_mode=int(g["fast_mode"]), z_min=float(g["z_min"]))
    inds = torch.from_numpy(g["inds"]).to(dev)
    start = torch.from_numpy(g["ref32_start"]).to(dev)
    r = native.rslm_split(prob, inds, start, params, want_all=True)
    resident = native.rslm(prob, inds, start, params, want_all=True)
    assert same(r["pose_all"], resident["pose_all"])
    pose_all, cost_all = r["pose_all"].cpu().numpy(), r["cost_all"].cpu().numpy()
    frac64, cerr64 = _hypothesis_agreement(pose_all, cost_all, g, "ref64")
    frac32, cerr32 = _hypothesis_agreement(pose_all, cost_all, g, "ref32")
    floor_frac, _ = _hypothesis_agreement(g["ref32_hyp_pose"], g["ref32_hyp_cost"], g, "ref64")
    assert frac64 >= min(0.9, floor_frac - 0.05), (frac64, floor_frac)
    ref_c32, ref_c64 = g["ref32_hyp_cost"], g["ref64_hyp_cost"]
    floor_cost = float((np.abs(ref_c32 - ref_c64) / np.maximum(np.abs(ref_c64), 1e-30)).max())
    assert cerr64 < max(1e-4, 3 * floor_cost) and cerr32 < max(1e-4, 3 * floor_cost), (cerr64, cerr32, floor_cost)
    perr, crel = _check_object_level(r["pose"].cpu().numpy(), r["cost"].cpu().numpy(), g, f"{name}/split")
    # the drop-in class, the reference's draws played back, every N above the (lowered) resident limit
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    camera = PerspectiveCamera(cam_mats=t("cam_mats"), z_min=float(g["z_min"]), lb=lb, ub=ub)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=float(g["relative_delta"]))
    cost_fun.set_param(t("x2d"), t("w2d"))
    calls = []
    fn = native.rslm_split
    monkeypatch.setattr(native, "rslm_split", lambda *a, **k: calls.append(1) or fn(*a, **k))
    monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i: 0)
    rs = RSLMSolver(dof=dof, num_points=n, num_proposals=P, num_iter=int(g["rs_iter"]), draws="torch", cluster_split=True)
    _Playback(monkeypatch, dev, [g["inds"]], [g["rot_draw"]], dof)
    pose, _, cost = rs.solve(t("x3d"), t("x2d"), t("w2d"), camera, cost_fun, fast_mode=bool(g["fast_mode"]))
    assert calls == [1]
    cperr, ccrel = _check_object_level(pose.cpu().numpy(), cost.cpu().numpy(), g, name + "/split/RSLMSolver.solve")
    record_parity(f"rslm/{name}/split", hyp_frac_within_1em4_vs_ref64=frac64, hyp_frac_within_1em4_vs_ref32=frac32,
                  ref32_frac_within_1em4_vs_ref64=floor_frac, hyp_cost_rel_max=max(cerr64, cerr32),
                  best_pose_rel_max=float(perr.max()), min_cost_rel_max=float(crel.max()),
                  solver_pose_rel_max=float(cperr.max()), solver_cost_rel_max=float(ccrel.max()),
                  hyp_cost=err_stats(cost_all, g["ref64_hyp_cost"]))


def _train_layer(cluster_split, P=4):
    """The reference's 6DoF training configuration (EPro-PnP-6DoF/lib/train.py)."""
    rslm = _SeededRSLM(dof=6, num_points=16, num_proposals=P, num_iter=3, cluster_split=cluster_split)
    return EProPnP6DoF(mc_samples=512, num_iter=4, solver=LMSolver(dof=6, num_iter=5, init_solver=rslm)), rslm


def _inputs(dev, B, N, seed):
    pc = make_problem(B, N, seed=seed, dof=6)
    return {k: pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats", "pose_gt")}


def test_reference_training_step_at_16384_points(cuda_device, monkeypatch):
    B, N, seed = 4, 16384, 0x5EED
    inp = _inputs(cuda_device, B, N, 7)
    layer, rslm = _train_layer(True)
    rslm.seed = seed
    starts = []
    fused = ag.fused_forward
    monkeypatch.setattr(ag, "fused_forward", lambda prob, pose_start, params, **k: starts.append(pose_start.clone())
                        or fused(prob, pose_start, params, **k))
    x3d, x2d, w2d = (inp[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
    camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(x2d.detach(), w2d)
    loss_fn = MonteCarloPoseLoss().to(cuda_device)
    pose_opt, _, plus, samples, logw, cost_tgt = layer.monte_carlo_forward(
        x3d, x2d, w2d, camera, cost_fun, pose_init=inp["pose_gt"], force_init_solve=True, with_pose_opt_plus=True,
        amis_seed=3)
    loss = loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - inp["pose_gt"]).abs().sum()
    loss.backward()
    for t in (loss, pose_opt, plus, samples, logw, cost_tgt, x3d.grad, x2d.grad, w2d.grad):
        assert torch.isfinite(t).all()
    assert x2d.grad.abs().sum() > 0 and w2d.grad.abs().sum() > 0
    # the LM start: the cheaper of pose_init and the RSLM winner, rebuilt from evaluate_pnp and RSLMSolver.solve
    with torch.no_grad():
        cost_init = evaluate_pnp(x3d.detach(), x2d.detach(), w2d.detach(), inp["pose_gt"], camera, cost_fun,
                                 out_cost=True)[1]
        pose_rs, _, cost_rs = rslm.solve(x3d.detach(), x2d.detach(), w2d.detach(), camera, cost_fun, with_cost=True)
    want = torch.where((cost_init < cost_rs)[:, None], inp["pose_gt"], pose_rs)
    assert len(starts) == 1 and same(starts[0], want)
    # inference without pose_init: the RSLM winner, refined by the LM solve, recovers the synthetic pose
    solver = LMSolver(dof=6, num_iter=10, init_solver=RSLMSolver(dof=6, num_points=16, num_proposals=64, num_iter=3,
                                                                 cluster_split=True))
    with torch.no_grad():
        pose = solver(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun)[0]
    gt = inp["pose_gt"]
    t_err = (pose[:, :3] - gt[:, :3]).norm(dim=-1) / gt[:, :3].norm(dim=-1)
    q = pose[:, 3:] / pose[:, 3:].norm(dim=-1, keepdim=True)
    r_err = 2 * torch.acos((q * gt[:, 3:]).sum(-1).abs().clamp(max=1.0)) * 180 / math.pi
    assert (t_err < 0.01).all() and (r_err < 1.0).all(), (t_err, r_err)
    record_parity("rslm_split/train_step_16384", inference_t_rel_max=float(t_err.max()),
                  inference_rot_deg_max=float(r_err.max()), loss=float(loss))


def test_default_solver_still_refuses_16384_points(cuda_device):
    inp = _inputs(cuda_device, 2, 16384, 9)
    camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(inp["x2d"], inp["w2d"])
    with pytest.raises(native.NativeError, match="shared memory"):
        RSLMSolver(dof=6).solve(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun)


def test_training_step_at_16384_points_replays_match_eager(cuda_device):
    """The training step above (B = 2) under CUDA-graph capture: seed-pointer RSLM draw, then refine, score and select,
    with new inputs and seeds at every replay, equal to eager calls bit for bit."""
    layer, rslm = _train_layer(True)
    loss_fn = MonteCarloPoseLoss().to("cuda")

    def run(inp, seeds):
        rslm.seed = seeds.get("rslm")
        if inp.get("_leaves") is None:
            inp["_leaves"] = tuple(inp[k].detach().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
        x3d, x2d, w2d = inp["_leaves"]
        for t in (x3d, x2d, w2d):
            t.grad = None
        loss_fn.norm_factor.fill_(1.0)
        camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d.detach(), w2d)
        pose_opt, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=inp["pose_gt"], force_init_solve=True,
            with_pose_opt_plus=True, amis_seed=seeds.get("amis"))
        loss = loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - inp["pose_gt"]).abs().sum()
        loss.backward()
        return dict(loss=loss.detach(), pose_opt=pose_opt, gx3d=x3d.grad, gx2d=x2d.grad, gw2d=w2d.grad)

    calls = []
    fn = native.rslm_split
    native.rslm_split = lambda *a, **k: calls.append(1) or fn(*a, **k)
    try:
        _check_replays_match_eager(cuda_device, run, 2, 16384, 6, ("amis", "rslm"))
    finally:
        native.rslm_split = fn
    assert calls
