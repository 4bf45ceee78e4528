"""Pins the oracle's autograd of the cost with respect to the POSE to the reference's own autograd
(tests/golden/cost_pose_grad, written by oracle/make_golden_cost_pose_grad.py): dL/d pose of
L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) through oracle.evaluate, at tensor and scalar bounds, 4DoF, depths below
z_min and both Huber branches.  The GPU and emulator tests of the pose-gradient kernels use this autograd as their
float64 reference, so this is what ties them to the reference.

The reference differentiates the rotation 1 - 2 (jj + kk), ..., the oracle (as the forward kernels) ww + ii - jj - kk,
...: equal on the unit sphere, so at the goldens' unit quaternions the two gradients differ by a multiple of q only.
The translation (and the yaw) gradient is compared as it is, the quaternion gradient without its component along q."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc

NAMES = golden_names("cost_pose_grad/")


def oracle_pose_grad(g, dtype=torch.float64):
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    poses = t("poses").requires_grad_(True)
    lb, ub = golden_bounds(g, dtype)
    cam = orc.Camera(t("cam_mats"), float(g["z_min"]), lb, ub)
    cost = orc.evaluate(t("x3d"), t("x2d"), t("w2d"), poses, cam, t("delta"))["cost"]
    (cost * t("upstream")).sum().backward()
    return cost.detach().numpy(), poses.grad.numpy()


def comparable(grad, poses):
    """The pose gradient with the quaternion part projected on the tangent space of the unit sphere at q."""
    grad = np.array(grad, np.float64)
    if grad.shape[-1] == 7:
        q = poses[..., 3:] / np.linalg.norm(poses[..., 3:], axis=-1, keepdims=True)
        grad[..., 3:] -= q * (q * grad[..., 3:]).sum(-1, keepdims=True)
    return grad


def per_pose_err(a, b):
    """max over poses of max|a - b| / max|b| within one pose's gradient."""
    scale = np.maximum(np.abs(b).max(-1), 1e-300)
    return float((np.abs(a - b).max(-1) / scale).max())


def test_goldens_present():
    assert NAMES == sorted(["dof4_small_delta", "dof4_tensor_bounds", "dof6_below_zmin", "dof6_scalar_bounds",
                            "dof6_small_delta", "dof6_tensor_bounds"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_pose_gradient_matches_reference_autograd(name):
    g = load_golden("cost_pose_grad/" + name)
    cost, grad = oracle_pose_grad(g)
    assert np.abs(cost - g["ref64_cost"]).max() / np.abs(g["ref64_cost"]).max() < 1e-8
    ref = comparable(g["grad_pose"], g["poses"])
    live = np.abs(ref).max(-1) > 0                      # (poses with a zero upstream weight have a zero gradient)
    assert live.mean() > 0.5 and (np.abs(ref[..., 3:]).max(-1) > 0)[live].all()
    assert per_pose_err(comparable(grad, g["poses"]), ref) < 1e-8
    # the reference's own float32 autograd: what single precision alone moves
    _, grad32 = oracle_pose_grad(g, torch.float32)
    floor = per_pose_err(comparable(g["ref32_grad_pose"], g["poses"]), ref)
    assert per_pose_err(comparable(grad32, g["poses"]), ref) < max(2e-4, 5 * floor)


def test_quaternion_forms_differ_along_q_only():
    """What `comparable` removes is there and is radial: the raw quaternion gradients of the two forms differ, by a
    multiple of q."""
    g = load_golden("cost_pose_grad/dof6_tensor_bounds")
    _, grad = oracle_pose_grad(g)
    diff = grad[..., 3:] - g["grad_pose"][..., 3:]
    q = g["poses"][..., 3:]
    along = (diff * q).sum(-1, keepdims=True) * q
    assert np.abs(diff).max() > 1e-3 * np.abs(grad[..., 3:]).max()
    assert np.abs(diff - along).max() < 1e-8 * np.abs(grad[..., 3:]).max()
    assert np.abs(grad[..., :3] - g["grad_pose"][..., :3]).max() < 1e-8 * np.abs(grad[..., :3]).max()


def test_cases_reach_their_branches():
    frac = lambda name, k: float(load_golden("cost_pose_grad/" + name)[k])
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4_tensor_bounds"):
        assert 0.03 <= frac(name, "frac_clamped") <= 0.2, name
    assert 0.05 <= frac("dof6_below_zmin", "frac_below_zmin") <= 0.3
    for name in ("dof6_small_delta", "dof4_small_delta"):
        assert 0.05 < frac(name, "frac_outlier") < 0.95, name
