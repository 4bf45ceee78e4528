"""Pins the oracle's double backward of the Monte-Carlo cost term to the reference's own float64 autograd with
create_graph (tests/golden/cost_hvp, written by oracle/make_golden_cost_hvp.py): for L = sum_{p, b} up[p, b] *
cost_b(pose[p, b]) and a tangent v, d((dL/d inputs) . v) / d(x3d, x2d, w2d, delta, poses, cam_mats, lb, ub, up), at
tensor and scalar bounds, 4DoF, depths below z_min and both Huber branches, on stacked poses (P, B, D).  The GPU and
emulator tests of the Hessian-vector-product kernels (test_cost_hvp_gpu.py) use this double backward as their float64
reference, so this is what ties the native second order to the reference.

The oracle forms the rotation as the kernels do (ww + ii - jj - kk, ...); the reference's differentiable branch is
1 - 2 (jj + kk), ..., the same less (|q|^2 - 1) I.  So in 6DoF the golden's product (a), whose quaternion tangent is
orthogonal to q, is compared on every output but the quaternion rows, and product (b), without a quaternion tangent, on
the quaternion rows after removing their component along q.  The quaternion-quaternion block is held to the oracle
alone, by the GPU tests."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc

NAMES = golden_names("cost_hvp/")
INPUTS = ("x3d", "x2d", "w2d", "delta", "poses", "cam_mats", "lb", "ub")
TOL = 1e-8


def per_object_err(a, b, axis=0):
    """max over the leading `axis` + 1 axes' rows of max|a - b| / max|b| (0 where both are zero)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a, b = a.reshape(a.shape[:axis + 1] + (-1,)), b.reshape(b.shape[:axis + 1] + (-1,))
    den = np.abs(b).max(-1)
    num = np.abs(a - b).max(-1)
    return float(np.where(den > 0, num / np.maximum(den, 1e-300), num).max())


def oracle_hvp(g, tag):
    t = lambda k: torch.from_numpy(g[k]).to(torch.float64)
    lb, ub = golden_bounds(g, torch.float64)
    inputs = dict(x3d=t("x3d"), x2d=t("x2d"), w2d=t("w2d"), delta=t("delta"), poses=t("poses"),
                  cam_mats=t("cam_mats"), lb=lb, ub=ub)
    leaves = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in inputs.items()}
    up = t("upstream").requires_grad_(True)
    cam = orc.Camera(leaves["cam_mats"], float(g["z_min"]), leaves["lb"], leaves["ub"])
    cost = orc.evaluate(leaves["x3d"], leaves["x2d"], leaves["w2d"], leaves["poses"], cam, leaves["delta"])["cost"]
    keys = [k for k in INPUTS if torch.is_tensor(leaves[k])]
    grads = torch.autograd.grad((cost * up).sum(), [leaves[k] for k in keys], create_graph=True)
    tan = {k: t("tan_" + k) for k in keys}
    if tag == "b" and int(g["dof"]) == 6:
        tan["poses"][..., 3:] = 0.0
    dot = sum((gi * tan[k]).sum() for gi, k in zip(grads, keys))
    h = torch.autograd.grad(dot, [leaves[k] for k in keys] + [up], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = {k: z(hi, leaves[k]).detach().numpy() for hi, k in zip(h[:-1], keys)}
    out["up"] = z(h[-1], up).detach().numpy()
    return out


def off_q(rows, q):
    """quaternion rows without their component along q."""
    return rows - (rows * q).sum(-1, keepdims=True) / (q * q).sum(-1, keepdims=True) * q


def test_goldens_present():
    assert NAMES == sorted(["dof4", "dof6_below_zmin", "dof6_scalar_bounds", "dof6_small_delta",
                            "dof6_tensor_bounds"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_double_backward_matches_reference(name):
    g = load_golden("cost_hvp/" + name)
    dof = int(g["dof"])
    a = oracle_hvp(g, "a")
    for k, v in a.items():
        ref = g["hvp_a_" + k]
        assert np.abs(ref).max() > 0, k
        if k == "poses":                           # (P, B, D): per pose and object
            if dof == 6:
                assert per_object_err(v[..., :3], ref[..., :3], 1) < TOL, k
            else:
                assert per_object_err(v, ref, 1) < TOL, k
        elif k == "up":                            # (P, B): one value per pose, per object over its poses
            assert per_object_err(v.T, ref.T) < TOL, k
        else:
            assert per_object_err(v, ref) < TOL, k
    if dof == 6:
        q = g["poses"][..., 3:]
        rows = oracle_hvp(g, "b")["poses"][..., 3:]
        ref = off_q(g["hvp_b_poses"][..., 3:], q)
        assert np.abs(ref).max() > 0
        assert per_object_err(off_q(rows, q), ref, 1) < TOL


def test_cases_reach_their_branches():
    frac = lambda name, k: float(load_golden("cost_hvp/" + name)[k])
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4"):
        assert 0.05 <= frac(name, "frac_clamped") <= 0.2, name
    assert 0.05 <= frac("dof6_below_zmin", "frac_below_zmin") <= 0.3
    assert 0.05 < frac("dof6_small_delta", "frac_outlier") < 0.995
    for name in NAMES:
        assert frac(name, "huber_gap") > 1e-6, name
