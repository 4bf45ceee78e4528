"""Pins the oracle's autograd through evaluate's residual, Jacobian and cost to the reference's own autograd
(tests/golden/evaluate_grad, written by oracle/make_golden_evaluate_grad.py): dL/d(x3d, x2d, w2d, delta, pose, cam_mats,
lb, ub) of L = <g_res, residual> + <g_jac, jacobian> + <g_cost, cost> through oracle.evaluate(want_jac=True), in 6DoF and
4DoF, with tensor, scalar and no bounds, depths below z_min, clip_jac=False, a stacked pose and both Huber branches.  The
GPU and emulator tests of epnp_evaluate_backward_f32 use this autograd as their float64 reference, so this is what ties
them to the reference.

As in test_oracle_cost_pose_grad_cpu.py, the quaternion gradient is compared without its component along q: the
reference's rotation and the oracle's (and the kernels') differ off the unit sphere only."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc
from test_oracle_cost_pose_grad_cpu import comparable

NAMES = golden_names("evaluate_grad/")
INPUTS = ("x3d", "x2d", "w2d", "delta", "pose", "cam_mats", "lb", "ub")


def oracle_evaluate_grad(g, dtype=torch.float64):
    """{input: gradient} of the golden's L through oracle.evaluate in `dtype` (bounds only when they are tensors)."""
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    leaves = {k: t(k).requires_grad_(True) for k in INPUTS[:6]}
    lb, ub = golden_bounds(g, dtype)
    if torch.is_tensor(lb):
        leaves["lb"], leaves["ub"] = lb.requires_grad_(True), ub.requires_grad_(True)
    cam = orc.Camera(leaves["cam_mats"], float(g["z_min"]), leaves.get("lb", lb), leaves.get("ub", ub))
    e = orc.evaluate(leaves["x3d"], leaves["x2d"], leaves["w2d"], leaves["pose"], cam, leaves["delta"], want_jac=True,
                     clip_jac=bool(g["clip_jac"]))
    ((e["residual"] * t("g_res")).sum() + (e["jac"] * t("g_jac")).sum() + (e["cost"] * t("g_cost")).sum()).backward()
    return {k: v.grad.numpy() for k, v in leaves.items()}


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_goldens_present():
    assert NAMES == sorted(["dof4_none", "dof4_tensor_bounds", "dof6_below_zmin", "dof6_no_clip", "dof6_scalar_bounds",
                            "dof6_small_delta", "dof6_stacked", "dof6_tensor_bounds"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_evaluate_gradient_matches_reference_autograd(name):
    g = load_golden("evaluate_grad/" + name)
    got, got32 = oracle_evaluate_grad(g), oracle_evaluate_grad(g, torch.float32)
    assert set(got) == {k for k in INPUTS if f"grad_{k}" in g}
    for k in got:
        ref, ref32, a, a32 = g[f"grad_{k}"], g[f"ref32_grad_{k}"], got[k], got32[k]
        if k == "pose":
            ref, ref32, a, a32 = (comparable(x, g["pose"]) for x in (ref, ref32, a, a32))
        # (delta reaches L only through outliers)
        assert np.abs(ref).max() > 0 or (k == "delta" and float(g["frac_outlier"]) == 0), (name, k)
        objs = ref.shape[-2] if k == "pose" else ref.shape[0]
        for o in range(objs):                           # per object
            pick = (lambda x: x[..., o, :]) if k == "pose" else (lambda x: x[o])
            b = pick(ref)
            if not np.abs(b).any():                     # (a bound that clamps nothing of this object)
                assert not np.abs(pick(a)).any(), (name, k, o)
                continue
            assert rel(pick(a), b) < 1e-8, (name, k, o, rel(pick(a), b))
            # the oracle in float32, against the reference's own float32 floor
            assert rel(pick(a32), b) < max(2e-4, 5 * rel(pick(ref32), b)), (name, k, o)


def test_cases_reach_their_branches():
    g = {n: load_golden("evaluate_grad/" + n) for n in NAMES}
    for name in ("dof6_tensor_bounds", "dof6_scalar_bounds", "dof4_tensor_bounds", "dof6_stacked"):
        assert 0.03 <= float(g[name]["frac_clamped"]) <= 0.2, name
    for name in ("dof6_below_zmin", "dof6_no_clip"):
        assert 0.05 <= float(g[name]["frac_below_zmin"]) <= 0.3, name
    for name in ("dof6_small_delta", "dof4_none", "dof6_below_zmin"):
        assert 0.05 < float(g[name]["frac_outlier"]) < 0.95, name
    assert int(g["dof6_no_clip"]["clip_jac"]) == 0 and g["dof6_stacked"]["pose"].shape[:2] == (3, 2)
    assert int(g["dof4_tensor_bounds"]["dof"]) == 4 and int(g["dof4_none"]["bounds"]) == 0
