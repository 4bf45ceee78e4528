"""Pins the oracle's double backward of the derivative-regularisation branch to the reference's own float64 autograd
with create_graph (tests/golden/gn_plus_hvp, written by oracle/make_golden_gn_plus_hvp.py): for L = <gplus,
pose_add(pose, gn_step(pose))> at a detached pose and a tangent u on every input, d((dL/d inputs) . u) / d(x3d, x2d,
w2d, delta, cam_mats, lb, ub, gplus), at tensor and scalar bounds, 4DoF, depths below z_min and both Huber branches.
The GPU and emulator tests of the Hessian-vector-product kernel (test_gn_plus_hvp_gpu.py) use this double backward as
their float64 reference, so this is what ties the native second order of pose_opt_plus to the reference."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc
from test_oracle_cost_hvp_cpu import per_object_err

NAMES = golden_names("gn_plus_hvp/")
INPUTS = ("x3d", "x2d", "w2d", "delta", "cam_mats", "lb", "ub")
TOL = 1e-8


def oracle_hvp(g):
    t = lambda k: torch.from_numpy(g[k]).to(torch.float64)
    lb, ub = golden_bounds(g, torch.float64)
    inputs = dict(x3d=t("x3d"), x2d=t("x2d"), w2d=t("w2d"), delta=t("delta"), cam_mats=t("cam_mats"), lb=lb, ub=ub)
    leaves = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in inputs.items()}
    gplus = t("gplus").requires_grad_(True)
    pose = t("pose")
    cam = orc.Camera(leaves["cam_mats"], float(g["z_min"]), leaves["lb"], leaves["ub"])
    plus = orc.pose_add(pose, orc.gn_step(leaves["x3d"], leaves["x2d"], leaves["w2d"], cam, leaves["delta"], pose))
    keys = [k for k in INPUTS if torch.is_tensor(leaves[k])]
    grads = torch.autograd.grad((plus * gplus).sum(), [leaves[k] for k in keys], create_graph=True)
    dot = sum((gi * t("tan_" + k)).sum() for gi, k in zip(grads, keys))
    h = torch.autograd.grad(dot, [leaves[k] for k in keys] + [gplus], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = {k: z(hi, leaves[k]).detach().numpy() for hi, k in zip(h[:-1], keys)}
    out["gplus"] = z(h[-1], gplus).detach().numpy()
    return out, plus.detach().numpy()


def test_goldens_present():
    assert NAMES == sorted(["dof4_tensor_bounds", "dof6", "dof6_below_zmin", "dof6_scalar_bounds", "dof6_small_delta",
                            "dof6_tensor_bounds"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_double_backward_matches_reference(name):
    g = load_golden("gn_plus_hvp/" + name)
    h, plus = oracle_hvp(g)
    assert per_object_err(plus, g["pose_opt_plus"]) < TOL
    for k, v in h.items():
        ref = g["hvp_" + k]
        if k not in ("lb", "ub"):           # the bounds reach the step only through clamped outliers' Huber weight
            assert np.abs(ref).max() > 0, k
        assert per_object_err(v, ref) < TOL, k


def test_cases_reach_their_branches():
    frac = lambda name, k: float(load_golden("gn_plus_hvp/" + name)[k])
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4_tensor_bounds"):
        assert frac(name, "frac_clamped") > 0.0, name
    assert 0.05 <= frac("dof6_below_zmin", "frac_below_zmin") <= 0.3
    assert 0.05 < frac("dof6_small_delta", "frac_outlier") < 0.995
    for name in NAMES:
        assert frac(name, "huber_gap") > 1e-6, name
