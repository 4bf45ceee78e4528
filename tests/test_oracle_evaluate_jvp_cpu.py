"""Pins the oracle's forward-mode derivatives to the reference's own forward AD (tests/golden/evaluate_jvp, written by
oracle/make_golden_evaluate_jvp.py): the tangents of evaluate's residual, Jacobian and cost along a tangent of all eight
inputs (x3d, x2d, w2d, delta, the pose, cam_mats, tensor lb / ub), in 6DoF and 4DoF, with tensor, scalar and no bounds,
depths below z_min, clip_jac=False, a stacked pose and both Huber branches; and the tangent of pose_add(pose,
gn_step(pose)) with the pose held constant.  The GPU and emulator tests of epnp_evaluate_jvp_f32 and of the
pose_opt_plus tangent use this oracle as their float64 reference, so this is what ties them to the reference.  The
quaternion tangents are orthogonal to q, where the reference's rotation form and the oracle's have the same derivative."""
import numpy as np
import pytest
import torch

from conftest import golden_bounds, golden_names, load_golden
from oracle import pnp_oracle as orc

NAMES = golden_names("evaluate_jvp/")
INPUTS = ("x3d", "x2d", "w2d", "delta", "pose", "cam_mats", "lb", "ub")


def oracle_jvp(g, dtype=torch.float64):
    """{output: tangent} of the golden's evaluate (and pose_opt_plus) through the oracle in `dtype`."""
    t = lambda k: torch.from_numpy(g[k]).to(dtype)
    lb, ub = golden_bounds(g, dtype)
    names = [k for k in INPUTS if "t_" + k in g]
    z_min, clip = float(g["z_min"]), bool(g["clip_jac"])

    def unpack(args):
        a = dict(zip(names, args))
        return a, orc.Camera(a["cam_mats"], z_min, a.get("lb", lb), a.get("ub", ub))

    def f(*args):
        a, cam = unpack(args)
        e = orc.evaluate(a["x3d"], a["x2d"], a["w2d"], a["pose"], cam, a["delta"], want_jac=True, clip_jac=clip)
        return e["residual"], e["jac"], e["cost"]
    primals = tuple(t(k) for k in names)
    tangents = tuple(t("t_" + k) for k in names)
    out = dict(zip(("tan_residual", "tan_jac", "tan_cost"), torch.func.jvp(f, primals, tangents)[1]))
    if "tan_pose_opt_plus" in g:
        pose = t("pose")

        def plus(*args):
            a, cam = unpack(args)
            return orc.pose_add(pose, orc.gn_step(a["x3d"], a["x2d"], a["w2d"], cam, a["delta"], pose))
        keep = [i for i, k in enumerate(names) if k != "pose"]
        out["tan_pose_opt_plus"] = torch.func.jvp(
            lambda *a: plus(*[a[keep.index(i)] if i in keep else pose for i in range(len(names))]),
            tuple(primals[i] for i in keep), tuple(tangents[i] for i in keep))[1]
    return {k: v.numpy() for k, v in out.items()}


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_goldens_present():
    assert NAMES == sorted(["dof4_none", "dof4_tensor_bounds", "dof6_below_zmin", "dof6_no_clip", "dof6_scalar_bounds",
                            "dof6_small_delta", "dof6_stacked", "dof6_tensor_bounds"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_forward_mode_matches_reference(name):
    g = load_golden("evaluate_jvp/" + name)
    got, got32 = oracle_jvp(g), oracle_jvp(g, torch.float32)
    assert set(got) == {k for k in g if k.startswith("tan_")}
    for k in got:
        ref, ref32, a, a32 = g[k], g["ref32_" + k], got[k], got32[k]
        assert np.abs(ref).max() > 0, (name, k)
        ax = 1 if (g["pose"].ndim == 3 and k != "tan_pose_opt_plus") else 0      # the object axis
        for o in range(g["x3d"].shape[0]):              # per object (all its poses together when stacked)
            pick = lambda x: np.take(x, o, axis=ax)
            b = pick(ref)
            assert rel(pick(a), b) < 1e-8, (name, k, o, rel(pick(a), b))
            assert rel(pick(a32), b) < max(2e-4, 5 * rel(pick(ref32), b)), (name, k, o)
