"""The pose-gradient kernels on the CPU: pnp_kernels.cu under the SIMT emulators, the resident kernel on the single-CTA
one (tests/simt_emul), the split kernel on the cluster one (tests/simt_cluster) with forced cluster sizes.  Held to the
oracle's float64 autograd per pose with the bound of test_pose_grad_gpu.py (whose helpers this file uses); bit-exact
properties; the audit build checks that rank 0 alone stores; results do not depend on the fiber schedule; autograd takes
the kernels for stacked hypotheses, resident and split."""
import ctypes

import pytest
import torch

import simt_cluster_native
import simt_native
import test_pose_grad_gpu as pg
from oracle import pnp_oracle as orc
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import HuberPnPCost
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

AUDIT = ("-DEPNP_SPLIT_AUDIT",)
TILE = pg.TILE


def _case(dof, N, P, B=2, bounds=False, nonunit=False, seed=9):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.2)
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, P, 1)
    poses[..., :3] += 0.03 * torch.randn(B, P, 3, generator=gen)
    if dof == 6:
        poses[..., 3:] += 0.02 * torch.randn(B, P, 4, generator=gen)
        if not nonunit:
            poses[..., 3:] /= poses[..., 3:].norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.05 * torch.randn(B, P, generator=gen)
    c = dict(pc, B=B, N=N, P=P, dof=dof, poses=poses, up=pg.upstream(B, P, gen), z_min=0.1, lb=None, ub=None,
             delta=orc.adaptive_delta(pc["x2d"], pc["w2d"], 0.1))
    if bounds:          # per-object bounds that clamp a share of the projections, none within BOUND_GAP of one
        c["lb"], c["ub"], margin = pg.bm.place_bounds(c["x3d"], poses, c["cam_mats"], 0.1, True)
        assert margin > pg.bm.BOUND_GAP, margin
    return c


def _check(c, got, what):
    g64, fr = pg.pose_grads(c, torch.float64, census=True)
    g32, _ = pg.pose_grads(c, torch.float32)
    assert 0.01 < fr["outlier"] < 0.99 and (c["lb"] is None or fr["clamped"] > 0.01), fr
    assert got.abs().sum() > 0
    pg.assert_per_pose(got, g64, g32, what)


@pytest.mark.parametrize("dof,N,bounds", [(6, 7, False), (6, 513, True), (4, 7, True), (4, 513, False)])
def test_resident_kernel_against_float64(monkeypatch, dof, N, bounds):
    simt_native.install(monkeypatch)
    c = _case(dof, N, TILE + 1, bounds=bounds, nonunit=(N == 7))
    full = pg.run_kernel(c)
    _check(c, full, (dof, N))
    # an object alone = its row of the batch; one pose alone = its row
    one = {k: (v[1:2].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v) for k, v in c.items()}
    assert torch.equal(pg.run_kernel(dict(one, B=1)), full[1:2])
    for p in (0, TILE - 1, TILE):
        assert torch.equal(pg.run_kernel(c, poses=c["poses"][:, p:p + 1].contiguous(), up=c["up"][:, p:p + 1].contiguous(),
                                         P=1), full[:, p:p + 1])


def test_plain_loader_equals_tma_path(monkeypatch):
    simt_native.install(monkeypatch)
    c = _case(6, 136, 5)
    full = pg.run_kernel(c)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], None, None, c["delta"])
    for k in ("x3d", "x2d", "w2d"):
        flat = torch.empty(c[k].numel() + 1)
        flat[1:] = c[k].reshape(-1)
        setattr(prob, k, flat[1:].view(c[k].shape))
        assert getattr(prob, k).data_ptr() % 16 != 0
    assert prob.x3d.data_ptr() % 16 != 0 and c["x3d"].data_ptr() % 16 == 0
    assert torch.equal(native.cost_pose_backward(prob, 6, 0.1, c["poses"], c["up"]), full)


@pytest.mark.parametrize("dof,N,P,ctas", [(6, 513, pg.SPLIT_TILE + 1, 2), (6, 7, 3, 3), (4, 513, TILE + 1, 3), (4, 7, 3, 2)])
def test_split_kernel_against_float64_and_resident(monkeypatch, dof, N, P, ctas):
    simt_native.install(monkeypatch)
    c = _case(dof, N, P, bounds=(N == 513), nonunit=(N == 7))
    res = pg.run_kernel(c)
    simt_cluster_native.install(monkeypatch)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)           # every N takes the split call
    split = pg.run_kernel(c, cluster_ctas=ctas)
    _check(c, split, (dof, N, ctas))
    assert pg.per_pose(split, res).max() < 2e-5
    assert torch.equal(pg.run_kernel(c, cluster_ctas=ctas), split)
    one = {k: (v[1:2].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v) for k, v in c.items()}
    assert torch.equal(pg.run_kernel(dict(one, B=1), cluster_ctas=ctas), split[1:2])


def test_rank_zero_alone_stores_and_schedule_does_not_matter(monkeypatch):
    simt_cluster_native.install(monkeypatch, AUDIT)
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)
    lib = simt_cluster_native.handle(AUDIT)
    c = _case(6, 50, TILE + 3, bounds=True)
    counts = (ctypes.c_longlong * 16)()
    try:
        lib.simt_set_schedule(0, 1)
        lib.simt_audit_reset()
        base = pg.run_kernel(c, cluster_ctas=3)
        lib.simt_audit_read(counts)
        assert list(counts)[:8] == [c["B"] * c["P"] * 7] + [0] * 7 and list(counts)[8:] == [0] * 8
        for mode, seed in ((1, 1), (2, 5)):
            lib.simt_set_schedule(mode, seed)
            assert torch.equal(pg.run_kernel(c, cluster_ctas=3), base), mode
    finally:
        lib.simt_set_schedule(0, 1)


def test_autograd_routes_pose_gradients_to_the_kernels(monkeypatch):
    """evaluate_cost_autograd on stacked hypotheses: the pose receives the kernel's gradient, with and without the
    correspondences requiring grad; above the (lowered) resident limit the split call."""
    dev = simt_cluster_native.install(monkeypatch)
    c = _case(6, 40, 3, B=2)
    camera = PerspectiveCamera(cam_mats=c["cam_mats"], z_min=0.1)
    cost_fun = HuberPnPCost(delta=c["delta"])
    direct = pg.run_kernel(c)
    for with_points in (False, True):
        x3d = c["x3d"].clone().requires_grad_(with_points)
        poses = c["poses"].transpose(0, 1).contiguous().requires_grad_(True)         # (S, B, D)
        cost = ag.evaluate_cost_autograd(x3d, c["x2d"], c["w2d"], poses, camera, cost_fun)
        (cost * c["up"].T).sum().backward()
        assert torch.equal(poses.grad, direct.transpose(0, 1))
        assert (x3d.grad is not None) == with_points
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "16")
    monkeypatch.setattr(native, "max_points", lambda dof, *a: 0)
    monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i: 0)
    poses = c["poses"].transpose(0, 1).contiguous().requires_grad_(True)
    cost = ag.evaluate_cost_autograd(c["x3d"], c["x2d"], c["w2d"], poses, camera, cost_fun)
    (cost * c["up"].T).sum().backward()
    assert torch.equal(poses.grad, pg.run_kernel(c).transpose(0, 1)) and pg.per_pose(poses.grad, direct.transpose(0, 1)).max() < 2e-5
    assert dev.type == "cpu"
