#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/evaluate_jvp/*.npz: forward-mode derivatives recorded from the
UNMODIFIED reference (/root/reference/epropnp, torch CPU, torch.autograd.forward_ad in float64 and float32).

    python oracle/make_golden_evaluate_jvp.py      # needs /root/reference; run in the build container

The cases are those of make_golden_evaluate_grad.py (6DoF and 4DoF; tensor, scalar and no bounds; depths below z_min;
clip_jac=False; a stacked (3, B, D) pose; a small delta), read from its fixtures in tests/golden/evaluate_grad.  Every
input (x3d, x2d, w2d, delta, the pose, cam_mats and tensor lb / ub) gets a seeded random tangent; a quaternion tangent
is made orthogonal to q, because the reference differentiates its rotation in the form 1 - 2(jj + kk), which agrees with
the kernels' ww + xx - yy - zz on the unit sphere only to first order along it.  Recorded: the tangents of the residual,
Jacobian and cost of evaluate_pnp(out_residual=True, out_jacobian=True, out_cost=True); and, for the cases with one pose
per object, the tangent of pose_add(pose, gn_step(pose)) (LMSolver(eps=1e-5)) with the pose held constant, with respect
to the problem inputs.
"""
import glob
import os
import sys

import numpy as np
import torch
import torch.autograd.forward_ad as fwAD

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                      # noqa: E402  (puts the reference first on sys.path)
from make_golden_cost_grad import PerspectiveCamera, HuberPnPCost, evaluate_pnp      # noqa: E402
from epropnp.levenberg_marquardt import LMSolver         # noqa: E402  (reference)

SRC = os.path.join(mk.ROOT, "tests", "golden", "evaluate_grad")
OUT = os.path.join(mk.ROOT, "tests", "golden", "evaluate_jvp")
INPUTS = ("x3d", "x2d", "w2d", "delta", "pose", "cam_mats", "lb", "ub")
PROBLEM = ("x3d", "x2d", "w2d", "delta", "cam_mats", "lb", "ub")


def bounds_of(g):
    if int(g["bounds"]) == 0:
        return None, None
    lb, ub = g["lb"], g["ub"]
    if int(g["bounds"]) == 1:
        return float(lb), float(ub)
    return torch.from_numpy(lb), torch.from_numpy(ub)


def reference_jvp(g, tan, dtype, gn_plus):
    lb, ub = bounds_of(g)
    inp = dict(x3d=g["x3d"], x2d=g["x2d"], w2d=g["w2d"], delta=g["delta"], pose=g["pose"], cam_mats=g["cam_mats"])
    inp = {k: torch.from_numpy(v).to(dtype) for k, v in inp.items()}
    if torch.is_tensor(lb):
        inp["lb"], inp["ub"] = lb.to(dtype), ub.to(dtype)
    z_min, dof = float(g["z_min"]), int(g["dof"])
    out = {}
    with fwAD.dual_level():
        # the duals also require grad: the reference's clamps otherwise take their out= forms, which forward AD
        # does not support
        d = {k: fwAD.make_dual(v.clone().requires_grad_(True), tan[k].to(dtype)) for k, v in inp.items()}
        camera = PerspectiveCamera(cam_mats=d["cam_mats"], z_min=z_min, lb=d.get("lb", lb), ub=d.get("ub", ub))
        cost_fun = HuberPnPCost(delta=d["delta"], eps=1e-10)
        res, cost, jac = evaluate_pnp(d["x3d"], d["x2d"], d["w2d"], d["pose"], camera, cost_fun, out_residual=True,
                                      out_jacobian=True, out_cost=True, clip_jac=bool(g["clip_jac"]))
        for k, v in (("residual", res), ("jac", jac), ("cost", cost)):
            out["tan_" + k] = fwAD.unpack_dual(v).tangent.detach().numpy()
        if gn_plus:
            solver = LMSolver(dof=dof, eps=1e-5)
            pose = inp["pose"]                                                   # held constant
            step = solver.gn_step(d["x3d"], d["x2d"], d["w2d"], pose, camera, cost_fun)
            out["tan_pose_opt_plus"] = fwAD.unpack_dual(solver.pose_add(pose, step, camera)).tangent.detach().numpy()
    return out


def run_case(path, seed):
    name = os.path.basename(path)[:-4]
    g = dict(np.load(path))
    gen = torch.Generator().manual_seed(seed)
    tan = {}
    for k in INPUTS:
        if k in ("lb", "ub") and int(g["bounds"]) != 2:
            continue
        tan[k] = torch.randn(g[k].shape, generator=gen, dtype=torch.float64)
    tan["cam_mats"] *= 10.0                     # K is O(100): a tangent of a comparable relative size
    if int(g["dof"]) == 6:
        q = torch.from_numpy(g["pose"][..., 3:])
        tq = tan["pose"][..., 3:]
        tan["pose"][..., 3:] = tq - (tq * q).sum(-1, keepdim=True) * q / (q * q).sum(-1, keepdim=True)
    gn_plus = g["pose"].ndim == 2
    r64 = reference_jvp(g, tan, torch.float64, gn_plus)
    r32 = reference_jvp(g, tan, torch.float32, gn_plus)
    out = {k: g[k] for k in ("dof", "z_min", "clip_jac", "bounds", "x3d", "x2d", "w2d", "cam_mats", "delta", "pose",
                             "frac_below_zmin", "frac_clamped", "frac_outlier")}
    if int(g["bounds"]) != 0:
        out["lb"], out["ub"] = g["lb"], g["ub"]
    for k, v in tan.items():
        out["t_" + k] = v.numpy()
    for k in r64:
        out[k], out["ref32_" + k] = r64[k], r32[k]
    os.makedirs(OUT, exist_ok=True)
    dst = os.path.join(OUT, name + ".npz")
    np.savez_compressed(dst, **out)
    print(f"{name}: {sorted(r64)} -> {os.path.getsize(dst) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    for i, path in enumerate(sorted(glob.glob(os.path.join(SRC, "*.npz")))):
        run_case(path, 900 + i)


if __name__ == "__main__":
    main()
