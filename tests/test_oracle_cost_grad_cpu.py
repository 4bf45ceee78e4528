"""Pins the oracle's autograd of the Monte-Carlo cost term to the reference's own float64 autograd
(tests/golden/cost_grad, written by oracle/make_golden_cost_grad.py): dL/d(x3d, x2d, w2d, delta) of
L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) through oracle.evaluate, at tensor and scalar bounds, 4DoF, depths below
z_min, both Huber branches and zero-weight rows.  The GPU backward matrix (test_backward_matrix_gpu.py) uses this
autograd as its float64 reference, so this is what ties the native backward to the reference."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc

NAMES = golden_names("cost_grad/")


def per_object_err(a, b):
    """max over objects of max|a - b| / max|b| within the object (leading axis = objects)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    return float((np.abs(a - b).max(1) / np.maximum(np.abs(b).max(1), 1e-300)).max())


def oracle_grads(g, dtype=torch.float64):
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    leaves = [t(k).requires_grad_(True) for k in ("x3d", "x2d", "w2d", "delta")]
    lb, ub = golden_bounds(g, dtype)
    cam = orc.Camera(t("cam_mats"), float(g["z_min"]), lb, ub)
    cost = orc.evaluate(*leaves[:3], t("poses"), cam, leaves[3])["cost"]
    (cost * t("upstream")).sum().backward()
    return cost.detach(), [x.grad for x in leaves]


def test_goldens_present():
    assert NAMES == sorted(["dof4", "dof6_below_zmin", "dof6_scalar_bounds", "dof6_small_delta", "dof6_tensor_bounds",
                            "dof6_zero_weights"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_cost_gradient_matches_reference_autograd(name):
    g = load_golden("cost_grad/" + name)
    cost, grads = oracle_grads(g)
    assert per_object_err(cost.T, g["ref64_cost"].T) < 1e-8
    for what, a in zip(("x3d", "x2d", "w2d", "delta"), grads):
        ref = g["grad_" + what]
        assert np.abs(ref).max() > 0, what
        assert per_object_err(a.numpy(), ref) < 1e-8, what


def test_cases_reach_their_branches():
    """Each golden exists for one branch of the backward: make sure the recorded inputs still reach it."""
    frac = lambda name, k: float(load_golden("cost_grad/" + name)[k])
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4"):
        assert 0.05 <= frac(name, "frac_clamped") <= 0.2, name
    assert 0.05 <= frac("dof6_below_zmin", "frac_below_zmin") <= 0.3
    g = load_golden("cost_grad/dof6_small_delta")
    x3d, x2d, w2d, poses = (torch.from_numpy(g[k]) for k in ("x3d", "x2d", "w2d", "poses"))
    u = orc.evaluate(x3d, x2d, w2d, poses, orc.Camera(torch.from_numpy(g["cam_mats"]), float(g["z_min"])),
                     torch.from_numpy(g["delta"]), want_jac=True)["residual"]
    # the robust rescale is sqrt(delta / s) < 1 exactly on the outlier branch: compare |residual| with |r|
    r = ((orc.evaluate(x3d, x2d, w2d, poses, orc.Camera(torch.from_numpy(g["cam_mats"]), float(g["z_min"])), 1e30,
                       want_jac=True)["residual"]))
    outlier = (u.abs() < r.abs() * (1 - 1e-12)).double().mean()
    assert 0.05 < float(outlier) < 0.995
    zw = load_golden("cost_grad/dof6_zero_weights")
    rows = (zw["w2d"] == 0).all(-1)                 # zero residual: the norm's gradient at 0 is 0 in torch
    assert rows.any() and ((zw["w2d"] == 0).sum(-1) == 1).any()
    for what in ("x3d", "x2d", "w2d"):
        assert (zw["grad_" + what][rows] == 0).all() and (zw["grad_" + what][~rows] != 0).any(), what
