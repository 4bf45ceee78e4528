"""The camera-gradient kernels on the CPU: pnp_kernels.cu under the SIMT emulators, the resident kernels on the
single-CTA one (tests/simt_emul), the split kernels on the cluster one (tests/simt_cluster) with forced cluster sizes.
Held to the float64 oracle per object with the bound of test_camera_grad_gpu.py (whose helpers this file uses), and the
GN-plus kernels also to the reference's own autograd (tests/golden/cost_camera_grad); an object alone equals its row of
the batch (each object has its own CTA or cluster); the audit build checks that only rank 0 stores and that every rank
ends with rank 0's step and v; autograd hands the kernels' gradients to cam_mats and the bounds."""
import ctypes

import numpy as np
import pytest
import torch

import simt_cluster_native
import simt_native
import test_camera_grad_gpu as cg
import test_pose_grad_gpu as pg
from conftest import golden_bounds, load_golden
from oracle import pnp_oracle as orc
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import HuberPnPCost
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

AUDIT = ("-DEPNP_SPLIT_AUDIT",)


def _case(dof, N, P, B=3, bounds=False, seed=9):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.2)
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, P, 1)
    poses[..., :3] += 0.03 * torch.randn(B, P, 3, generator=gen)
    if dof == 6:
        q = poses[..., 3:] + 0.02 * torch.randn(B, P, 4, generator=gen)
        poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.05 * torch.randn(B, P, generator=gen)
    c = dict(pc, B=B, N=N, P=P, dof=dof, poses=poses, up=pg.upstream(B, P, gen), z_min=0.1, lb=None, ub=None,
             delta=orc.adaptive_delta(pc["x2d"], pc["w2d"], 0.1))
    if bounds:          # per-object bounds that clamp a share of the projections, none within BOUND_GAP of one
        c["lb"], c["ub"], margin = pg.bm.place_bounds(c["x3d"], poses, c["cam_mats"], 0.1, True)
        assert margin > pg.bm.BOUND_GAP, margin
    return c


def _check_cost(c, got, what):
    g64, fr = cg.camera_grads(c, torch.float64, census=True)
    g32, _ = cg.camera_grads(c, torch.float32)
    assert 0.01 < fr["outlier"] < 0.99 and (c["lb"] is None or fr["clamped"] > 0.01), fr
    assert got[0].abs().sum() > 0 and (c["lb"] is None or got[1].abs().sum() > 0 and got[2].abs().sum() > 0)
    cg.assert_per_object(got, g64, g32, what)


def _row(c, b):
    one = {k: (v[b:b + 1].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v)
           for k, v in c.items()}
    return dict(one, B=1)


@pytest.mark.parametrize("dof,N,P,bounds", [(6, 7, 1, False), (6, 513, 129, True), (4, 7, 129, True),
                                            (4, 513, 1, False)])
def test_resident_cost_kernel_against_float64(monkeypatch, dof, N, P, bounds):
    simt_native.install(monkeypatch)
    c = _case(dof, N, P, bounds=bounds)
    full = cg.run_kernel(c, PA=max(P - 1, 1))
    _check_cost(c, full, (dof, N, P))
    for b in (0, 2):
        for x, y in zip(cg.run_kernel(_row(c, b), PA=max(P - 1, 1)), full):
            assert x is None or torch.equal(x, y[b:b + 1])


@pytest.mark.parametrize("dof,N,P,ctas", [(6, 513, 129, 2), (6, 7, 3, 3), (4, 513, 1, 3), (4, 7, 129, 2)])
def test_split_cost_kernel_against_float64_and_resident(monkeypatch, dof, N, P, ctas):
    """N = 7 on 3 CTAs leaves ranks 1 and 2 without points; they still take part in both barriers."""
    simt_native.install(monkeypatch)
    c = _case(dof, N, P, bounds=(N == 513))
    res = cg.run_kernel(c)
    simt_cluster_native.install(monkeypatch)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)           # every N takes the split call
    split = cg.run_kernel(c, cluster_ctas=ctas)
    _check_cost(c, split, (dof, N, ctas))
    for a, b in zip(split, res):
        assert a is None or pg.bm.per_object(a, b).max() < 2e-5
    for b in (0, 2):
        for x, y in zip(cg.run_kernel(_row(c, b), cluster_ctas=ctas), split):
            assert x is None or torch.equal(x, y[b:b + 1])


def _gn_case(dof, N, B=3, bounds=False, seed=21):
    c = _case(dof, N, 1, B=B, bounds=bounds, seed=seed)
    c["pose"] = c["poses"][:, 0].contiguous()
    gp = torch.randn(B, 7 if dof == 6 else 4, generator=torch.Generator().manual_seed(seed))
    return c, gp


def _gn_run(c, gp, ctas=None):
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    want = (True,) + (c["lb"] is not None,) * 2
    return native.gn_plus_camera_backward(prob, c["pose"], gp, c["dof"], c["z_min"], cg.EPS, cg.HUBER_EPS, want=want,
                                          cluster_ctas=ctas or 0)


@pytest.mark.parametrize("dof,N,bounds", [(6, 7, False), (6, 513, True), (4, 7, True), (4, 513, False)])
def test_gn_plus_camera_kernels_against_float64(monkeypatch, dof, N, bounds):
    simt_native.install(monkeypatch)
    c, gp = _gn_case(dof, N, bounds=bounds)
    res = _gn_run(c, gp)
    c64, c32 = cg.gn_composite(c, gp, torch.float64), cg.gn_composite(c, gp, torch.float32)
    cg.assert_per_object(list(res), c64, c32, ("resident", dof, N))
    for b in (0, 2):
        for x, y in zip(_gn_run(_row(c, b), gp[b:b + 1]), res):
            assert x is None or torch.equal(x, y[b:b + 1])
    simt_cluster_native.install(monkeypatch)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)
    for ctas in (2, 3):
        split = _gn_run(c, gp, ctas)
        cg.assert_per_object(list(split), c64, c32, ("split", dof, N, ctas))
        for b in (0, 2):
            for x, y in zip(_gn_run(_row(c, b), gp[b:b + 1], ctas), split):
                assert x is None or torch.equal(x, y[b:b + 1])


@pytest.mark.parametrize("name", ["gn_dof6_tensor_bounds_outliers", "gn_dof4_tensor_bounds", "gn_dof6_below_zmin"])
def test_gn_plus_camera_kernels_against_reference_goldens(monkeypatch, name):
    """The reference's own float64 autograd of <g, pose (+) gn_step(pose)>, with the bound max(2e-4, 5 * the reference's
    float32 floor) per object; with outliers among the clamped points the bounds' gradient is not zero."""
    g = load_golden("cost_camera_grad/" + name)
    t = lambda k: torch.from_numpy(g[k]).float()
    lb, ub = golden_bounds(g)
    bounded = lb is not None
    simt_native.install(monkeypatch)
    prob = native.Problem(t("x3d"), t("x2d"), t("w2d"), t("cam_mats"), lb, ub, t("delta"))
    args = (prob, t("pose"), t("gplus"), int(g["dof"]), float(g["z_min"]), cg.EPS, cg.HUBER_EPS)
    res = native.gn_plus_camera_backward(*args, want=(True, bounded, bounded))
    simt_cluster_native.install(monkeypatch)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)
    split = native.gn_plus_camera_backward(*args, want=(True, bounded, bounded), cluster_ctas=2)
    refs = [g["grad_cam"]] + ([g["grad_lb"], g["grad_ub"]] if bounded else [])
    refs32 = [g["ref32_grad_cam"]] + ([g["ref32_grad_lb"], g["ref32_grad_ub"]] if bounded else [])
    for out in (res, split):
        for a, b, b32 in zip(out, refs, refs32):
            a = a.double().numpy()
            for o in range(b.shape[0]):
                if not np.abs(b[o]).any():
                    assert not np.abs(a[o]).any(), (name, o)
                    continue
                err = np.abs(a[o] - b[o]).max() / np.abs(b[o]).max()
                floor = np.abs(b32[o] - b[o]).max() / np.abs(b[o]).max()
                assert err < max(2e-4, 5 * floor), (name, o, err, floor)
    if name.endswith("_outliers"):
        assert res[1].abs().sum() > 0 and res[2].abs().sum() > 0


def test_audit_rank_zero_alone_stores_and_ranks_agree(monkeypatch):
    simt_cluster_native.install(monkeypatch, AUDIT)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)
    lib = simt_cluster_native.handle(AUDIT)
    counts = (ctypes.c_longlong * 16)()
    c = _case(6, 50, 5, B=2, bounds=True)
    lib.simt_audit_reset()
    cg.run_kernel(c, cluster_ctas=3)
    lib.simt_audit_read(counts)
    assert list(counts)[:8] == [c["B"] * 13] + [0] * 7 and list(counts)[8:] == [0] * 8
    g, gp = _gn_case(6, 50, B=2, bounds=True)
    try:
        for mode, seed in ((0, 1), (1, 1), (2, 5)):
            lib.simt_set_schedule(mode, seed)
            lib.simt_audit_reset()
            out = _gn_run(g, gp, 3)
            lib.simt_audit_read(counts)
            # rank 0 alone stores; H, g, cost, step and v carry rank 0's bits on every rank
            assert list(counts)[:8] == [g["B"] * 13] + [0] * 7 and list(counts)[8:] == [0] * 8, mode
            if mode == 0:
                base = out
            for a, b in zip(out, base):
                assert torch.equal(a, b), mode
    finally:
        lib.simt_set_schedule(0, 1)


def test_autograd_routes_camera_gradients_to_the_kernels(monkeypatch):
    """The cost with only the camera requiring grad has a grad_fn and gives the kernel's gradients, reduced to the
    shapes passed: a (3, 3) camera and (2,) bounds receive the sums over objects, (B, 2) bounds their rows."""
    simt_native.install(monkeypatch)
    c = _case(6, 40, 3, B=2, bounds=True)
    c["cam_mats"] = c["cam_mats"][:1].expand(2, 3, 3).contiguous()
    direct = cg.run_kernel(c)
    K = c["cam_mats"][0].clone().requires_grad_(True)
    lb = c["lb"].clone().requires_grad_(True)
    ub = c["ub"].clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=K, z_min=0.1, lb=lb, ub=ub)
    poses = c["poses"].transpose(0, 1).contiguous()
    cost = ag.evaluate_cost_autograd(c["x3d"], c["x2d"], c["w2d"], poses, camera, HuberPnPCost(delta=c["delta"]))
    assert cost.grad_fn is not None
    (cost * c["up"].T).sum().backward()
    assert torch.equal(K.grad, direct[0].sum(0)) and torch.equal(lb.grad, direct[1]) and torch.equal(ub.grad, direct[2])
    lb1 = c["lb"][0].clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=c["cam_mats"], z_min=0.1, lb=lb1, ub=float(c["ub"].max()) + 1e4)
    cost = ag.evaluate_cost_autograd(c["x3d"], c["x2d"], c["w2d"], poses, camera, HuberPnPCost(delta=c["delta"]))
    (cost * c["up"].T).sum().backward()
    assert lb1.grad.shape == (2,) and lb1.grad.abs().sum() > 0
