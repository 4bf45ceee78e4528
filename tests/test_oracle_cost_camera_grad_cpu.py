"""Pins the oracle's autograd with respect to the CAMERA to the reference's own autograd (tests/golden/cost_camera_grad,
written by oracle/make_golden_cost_camera_grad.py): dL/d(cam_mats, lb, ub) of L = sum_{p, b} up[p, b] cost_b(pose[p, b])
through oracle.evaluate, and of L = <g, pose (+) gn_step(pose)> through oracle.gn_step / pose_add, at tensor and scalar
bounds, 4DoF, depths below z_min and both Huber branches.  The GPU and emulator tests of the camera-gradient kernels use
this autograd as their float64 reference, so this is what ties them to the reference."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc

NAMES = golden_names("cost_camera_grad/")


def oracle_camera_grad(g, dtype=torch.float64):
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    lb, ub = golden_bounds(g, dtype)
    K = t("cam_mats").requires_grad_(True)
    leaves = [K] + [b.requires_grad_(True) for b in (lb, ub) if torch.is_tensor(b)]
    cam = orc.Camera(K, float(g["z_min"]), lb, ub)
    if str(g["loss"]) == "cost":
        cost = orc.evaluate(t("x3d"), t("x2d"), t("w2d"), t("poses"), cam, t("delta"))["cost"]
        (cost * t("upstream")).sum().backward()
    else:
        pose = t("pose")
        step = orc.gn_step(t("x3d"), t("x2d"), t("w2d"), cam, t("delta"), pose, eps=1e-5)
        (orc.pose_add(pose, step) * t("gplus")).sum().backward()
    return [l.grad.numpy() for l in leaves]


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_goldens_present():
    assert NAMES == sorted(["dof4_tensor_bounds", "dof6_below_zmin", "dof6_scalar_bounds", "dof6_small_delta",
                            "dof6_tensor_bounds", "gn_dof4_tensor_bounds", "gn_dof6_below_zmin",
                            "gn_dof6_tensor_bounds", "gn_dof6_tensor_bounds_outliers"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_camera_gradient_matches_reference_autograd(name):
    g = load_golden("cost_camera_grad/" + name)
    got = oracle_camera_grad(g)
    refs = [g["grad_cam"]] + ([g["grad_lb"], g["grad_ub"]] if int(g["bounds"]) == 2 else [])
    assert len(got) == len(refs)
    got32 = oracle_camera_grad(g, torch.float32)
    refs32 = [g["ref32_grad_cam"]] + ([g["ref32_grad_lb"], g["ref32_grad_ub"]] if int(g["bounds"]) == 2 else [])
    for i, (a, b, a32, b32) in enumerate(zip(got, refs, got32, refs32)):
        if i > 0 and str(g["loss"]) == "gn" and not name.endswith("_outliers"):
            # the clamped points here are inliers: their clamped rows are masked and their Huber weight is 1, so no
            # residual of theirs reaches the step and the bounds get no gradient
            assert not np.abs(b).any() and not np.abs(a).any() and not np.abs(a32).any()
            continue
        assert np.abs(b).max() > 0
        for o in range(b.shape[0]):                     # per object
            if not np.abs(b[o]).any():                  # (a bound that clamps no outlier of this object)
                assert not np.abs(a[o]).any() and not np.abs(a32[o]).any(), (name, o)
                continue
            assert rel(a[o], b[o]) < 1e-8, (name, o)
            # the oracle in float32: what single precision alone moves, against the reference's own float32 floor
            assert rel(a32[o], b[o]) < max(2e-4, 5 * rel(b32[o], b[o])), (name, o)


def test_cases_reach_their_branches():
    frac = lambda name, k: float(load_golden("cost_camera_grad/" + name)[k])
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4_tensor_bounds", "gn_dof6_tensor_bounds",
                 "gn_dof4_tensor_bounds"):
        assert 0.03 <= frac(name, "frac_clamped") <= 0.2, name
    for name in ("dof6_below_zmin", "gn_dof6_below_zmin"):
        assert 0.05 <= frac(name, "frac_below_zmin") <= 0.3, name
    assert 0.05 < frac("dof6_small_delta", "frac_outlier") < 0.95
    # outliers among the clamped points: the bounds' gradient through pose_opt_plus is not zero
    g = load_golden("cost_camera_grad/gn_dof6_tensor_bounds_outliers")
    assert 0.03 <= float(g["frac_clamped"]) <= 0.2 and float(g["frac_outlier"]) > 0.05
    assert np.abs(g["grad_lb"]).max() > 0 and np.abs(g["grad_ub"]).max() > 0
