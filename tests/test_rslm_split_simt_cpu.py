"""The cluster-split RSLM initialiser (epnp_rslm_split_f32) on the CPU: pnp_kernels.cu under the cluster SIMT emulator
(tests/simt_cluster), at toy sizes.  The refined hypotheses are bit-identical to the resident rslm_kernel's, the costs
to evaluate_cost_split's on those poses, the winner is torch.min's over the hypotheses (NaN first, then the smaller cost,
then the earlier hypothesis); an object alone equals its row of the batch; a build or device without clusters refuses
and writes nothing; RSLMSolver takes the split call only when built with cluster_split=True and only above the resident
limit."""
import ctypes
import math

import pytest
import torch

import simt_cluster_native
import simt_native
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.levenberg_marquardt import RSLMSolver
from epropnp_b200 import capi, native
from epropnp_b200.synth import _yaw_to_mat, make_problem, quat_to_mat_ref


def _case(dof, N, P, n, B=3, bounds=False, z_min=0.1, seed=5):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.2)
    gen = torch.Generator().manual_seed(seed + 1)
    D = 7 if dof == 6 else 4
    inds = torch.stack([torch.stack([torch.randperm(N, generator=gen)[:n] for _ in range(B)]) for _ in range(P)])
    start = pc["pose_gt"][None].repeat(P, 1, 1)
    start[..., :3] += 0.2 * torch.randn(P, B, 3, generator=gen)
    if dof == 6:
        q = torch.randn(P, B, 4, generator=gen)
        start[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        start[..., 3] = torch.rand(P, B, generator=gen) * (2 * math.pi)
    lb = ub = None
    if bounds:
        lb = torch.tensor([[260.0, 190.0]]).repeat(B, 1)
        ub = torch.tensor([[380.0, 290.0]]).repeat(B, 1)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.1)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta)
    assert start.shape == (P, B, D)
    return pc, prob, inds.to(torch.int32), start


def _depths(pc, dof):
    pose = pc["pose_gt"]
    R = quat_to_mat_ref(pose[:, 3:]) if dof == 6 else _yaw_to_mat(pose[:, 3])
    return (pc["x3d"] @ R.transpose(-1, -2) + pose[:, None, :3])[..., 2]


def bits(t):
    """The float32 bit patterns of `t`: equal bits, including those of a NaN."""
    return t.contiguous().view(torch.int32)


def same(a, b):
    return torch.equal(bits(a), bits(b))


def _winner(cost_all):
    """torch.min's choice over the hypotheses (dim 0), written out: a NaN cost wins, then the smaller, then the earlier."""
    P, B = cost_all.shape
    win = []
    for b in range(B):
        w = 0
        for h in range(1, P):
            c, wc = float(cost_all[h, b]), float(cost_all[w, b])
            if math.isnan(c) != math.isnan(wc):
                better = math.isnan(c)
            else:
                better = not math.isnan(c) and c < wc
            if better:
                w = h
        win.append(w)
    return torch.tensor(win)


def _check_select(out):
    win = _winner(out["cost_all"])
    rows = torch.arange(out["cost_all"].shape[1])
    assert same(out["pose"], out["pose_all"][win, rows]) and same(out["cost"], out["cost_all"][win, rows])
    return win


# (dof, fast_mode, lm_iter, bounds, z_min, C): both DOF, LM and fast mode, bounds, depths below z_min, lm_iter = 0,
# C = 2 .. 4
CASES = [
    (6, 0, 3, False, 0.1, 2),
    (6, 1, 2, True, 0.1, 3),
    (6, 0, 2, False, 6.5, 4),
    (4, 0, 0, True, 0.1, 2),
    (4, 1, 3, False, 6.5, 3),
    (4, 0, 3, True, 6.5, 4),
]


@pytest.mark.parametrize("dof,fast,lm_iter,bounds,z_min,C", CASES)
def test_split_initialiser_against_the_resident_kernel(monkeypatch, dof, fast, lm_iter, bounds, z_min, C):
    simt_cluster_native.install(monkeypatch)
    pc, prob, inds, start = _case(dof, 48, 5, 6, bounds=bounds)
    if z_min > 1.0:                  # at the true pose, some points lie in front of z_min and some behind
        depth = _depths(pc, dof)
        assert (depth < z_min).any() and (depth > z_min).any()
    params = native.default_params(dof, lm_iter=lm_iter, fast_mode=fast, z_min=z_min)
    res = native.rslm(prob, inds, start, params, want_all=True)
    out = native.rslm_split(prob, inds, start, params, want_all=True, cluster_ctas=C)
    assert same(out["pose_all"], res["pose_all"])
    assert same(out["cost_all"], native.evaluate_cost_split(prob, out["pose_all"], dof, z_min, C))
    # a diverged fast-mode hypothesis has a NaN pose and cost in both; every other cost differs by summation order only
    finite = torch.isfinite(res["cost_all"])
    assert finite.float().mean() > 0.8 and torch.equal(finite, torch.isfinite(out["cost_all"]))
    rel = (out["cost_all"] - res["cost_all"])[finite].abs() / res["cost_all"][finite].abs().clamp(min=1e-30)
    assert rel.max() < 1e-5, rel.max()
    win = _check_select(out)
    assert torch.equal(win, _winner(res["cost_all"])) or \
        ((out["cost"] - res["cost"]).abs() / res["cost"].abs() < 1e-5).all()
    # an object alone = its row of the batch
    one = native.Problem(prob.x3d[1:2], prob.x2d[1:2], prob.w2d[1:2], prob.cam[1:2],
                         None if prob.lb is None else prob.lb[1:2], None if prob.ub is None else prob.ub[1:2],
                         prob.delta[1:2])
    alone = native.rslm_split(one, inds[:, 1:2].contiguous(), start[:, 1:2].contiguous(), params, want_all=True,
                              cluster_ctas=C)
    for k in ("pose_all", "cost_all"):
        assert same(alone[k], out[k][:, 1:2])
    assert same(alone["pose"], out["pose"][1:2]) and same(alone["cost"], out["cost"][1:2])
    # without want_all only the winners come back, the same ones
    lean = native.rslm_split(prob, inds, start, params, cluster_ctas=C)
    assert lean["pose_all"] is None and lean["cost_all"] is None
    assert same(lean["pose"], out["pose"]) and same(lean["cost"], out["cost"])


def test_nan_hypothesis_and_exact_tie(monkeypatch):
    """A hypothesis whose start is NaN has a NaN cost and wins its object (torch.min propagates NaN); a duplicated
    hypothesis ties exactly with its original and the earlier one wins."""
    simt_cluster_native.install(monkeypatch)
    pc, prob, inds, start = _case(6, 40, 6, 6)
    params = native.default_params(6, lm_iter=3, z_min=0.1)
    base = native.rslm_split(prob, inds, start, params, want_all=True, cluster_ctas=2)
    w = _check_select(base)
    last = inds.shape[0] - 1
    for b in range(3):                      # the last hypothesis repeats each object's winner
        inds[last, b] = inds[w[b], b]
        start[last, b] = start[w[b], b]
    start[2, 0] = float("nan")              # object 0: a NaN hypothesis
    out = native.rslm_split(prob, inds, start, params, want_all=True, cluster_ctas=2)
    res = native.rslm(prob, inds, start, params, want_all=True)
    assert same(out["pose_all"], res["pose_all"])
    win = _check_select(out)
    assert win[0] == 2 and math.isnan(float(out["cost"][0])) and out["pose"][0].isnan().all()
    for b in (1, 2):
        assert float(out["cost_all"][last, b]) == float(out["cost_all"][w[b], b])
        assert win[b] == w[b] < last
    assert _winner(res["cost_all"]).tolist() == win.tolist()


def _raw_call(prob, inds, start, params, C):
    """epnp_rslm_split_f32 on sentinel-filled outputs -> (rc, outputs)."""
    P, B, n = inds.shape
    D = start.shape[-1]
    outs = [torch.full(s, 1234.5) for s in ((B, D), (B,), (P, B, D), (P, B))]
    rc = capi.lib().epnp_rslm_split_f32(*prob.common_ptrs(), capi.iptr(inds), capi.ptr(start),
                                        *(capi.ptr(t) for t in outs), P, n, B, prob.N, ctypes.byref(params), C, None)
    return rc, outs


@pytest.mark.parametrize("build", ["single_cta", "no_cluster_fits"])
def test_without_clusters_the_call_is_refused_and_writes_nothing(monkeypatch, build):
    if build == "single_cta":
        simt_native.install(monkeypatch)
    else:
        simt_cluster_native.install(monkeypatch)
        monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "0")
    pc, prob, inds, start = _case(6, 40, 3, 6)
    params = native.default_params(6, lm_iter=3)
    rc, outs = _raw_call(prob, inds, start, params, 0)
    assert rc == -3                                         # EPNP_ERR_UNSUPPORTED
    assert all((t == 1234.5).all() for t in outs)
    with pytest.raises(native.NativeError, match="not supported"):
        native.rslm_split(prob, inds, start, params)


@pytest.mark.parametrize("cluster_split", [False, True])
def test_rslm_solver_routing(monkeypatch, cluster_split):
    """cluster_split=True: the split call exactly above the (lowered) resident limit, the resident call at or below it;
    the default: the resident call at every N."""
    simt_cluster_native.install(monkeypatch)
    calls = []
    for name in ("rslm", "rslm_split"):
        fn = getattr(native, name)
        monkeypatch.setattr(native, name, lambda *a, _fn=fn, _n=name, **k: calls.append(_n) or _fn(*a, **k))
    pc = make_problem(2, 40, seed=3, dof=6)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    solver = RSLMSolver(dof=6, num_points=6, num_proposals=4, num_iter=2, draws="torch", cluster_split=cluster_split)
    assert solver.cluster_split is cluster_split and RSLMSolver(dof=6).cluster_split is False
    results = {}
    for limit in (0, 39, 40, 10 ** 6):
        monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i, _l=limit: _l)
        calls.clear()
        torch.manual_seed(11)
        pose, none, cost = solver.solve(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun)
        assert none is None and torch.isfinite(pose).all() and torch.isfinite(cost).all()
        split = cluster_split and 40 > limit
        assert calls == ["rslm_split" if split else "rslm"], (limit, calls)
        results[limit] = (pose, cost)
    # the same draws: the split initialiser refines the same hypotheses; the winners' costs agree to summation order
    for limit in (0, 39):
        assert ((results[limit][1] - results[40][1]).abs() / results[40][1] < 1e-5).all()
