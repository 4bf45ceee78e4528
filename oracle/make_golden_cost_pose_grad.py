#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/cost_pose_grad/*.npz: gradients of the PnP cost with respect to
the POSE, recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU autograd, float64 and float32).

    python oracle/make_golden_cost_pose_grad.py      # needs /root/reference; run in the build container

Every case evaluates L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) with the reference's evaluate_pnp(..., out_cost=True)
on stacked poses (P, B, D) that require grad, and stores dL/d pose.  Cases: per-object and scalar bounds that clamp
part of the projections, 4DoF, homogeneous depths below z_min, a small delta (both Huber branches).  Bounds and z_min
keep the margins of make_golden_cost_grad.py (whose helpers this file uses).

The quaternion.  With a pose that requires grad the reference builds the rotation as 1 - 2 (jj + kk), ...
(common.py:30-36); without, as ww + ii - jj - kk, ... (:37-41), which is what this project's forward kernels and its
oracle compute.  The two agree on the unit sphere and differ by (|q|^2 - 1) I off it, so their gradients at a unit
quaternion differ by a multiple of q and by nothing else.  The poses here are therefore normalised in float64 (not
rounded to float32), and tests/test_oracle_cost_pose_grad_cpu.py compares the translation gradient as it is and the
quaternion gradient after removing its component along q.  Off the unit sphere the two forms are different functions of
q; no case records one, because nothing of it could be compared.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                      # noqa: E402  (puts the reference first on sys.path)
from make_golden_cost_grad import PerspectiveCamera, HuberPnPCost, evaluate_pnp, make_problem      # noqa: E402

OUT = os.path.join(mk.ROOT, "tests", "golden", "cost_pose_grad")


def reference_grad(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min, dtype):
    c = lambda t: t.to(dtype).clone() if torch.is_tensor(t) else t
    ps = poses.to(dtype).clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=c(cam_mats), z_min=z_min, lb=c(lb), ub=c(ub))
    _, cost, _ = evaluate_pnp(c(x3d), c(x2d), c(w2d), ps, camera, HuberPnPCost(delta=c(delta)), out_cost=True)
    (cost * up.to(dtype)).sum().backward()
    return cost.detach(), ps.grad


def run_case(name, B, N, P, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0):
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    poses = mk.stacked_poses(p, P, dof, seed + 1, tz)
    if dof == 6:
        poses[..., 3:] /= poses[..., 3:].norm(dim=-1, keepdim=True)         # unit to float64 rounding
    up = mk.upstream(P, B, seed + 2)
    delta = (w2d.mean(dim=(-2, -1)) * x2d.var(dim=-2).sum(-1).sqrt() * relative_delta).float().double()
    if bounds == "tensor":
        lb = (x2d.amin(1) + bound_margin).float().double()
        ub = (x2d.amax(1) - bound_margin).float().double()
    elif bounds == "scalar":
        lb, ub = 110.5, 520.5
    else:
        lb = ub = None

    zh, u = mk.project_unclamped(x3d, poses, cam_mats)
    below = float((zh < z_min).double().mean())
    assert (zh - z_min).abs().min() > 1e-6, name
    clamped = 0.0
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=d) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        u_c = u * (zh / zh.clamp(min=z_min))[..., None]
        clamped = float(((u_c < lbt) | (u_c > ubt)).any(-1).double().mean())
        assert torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min() > 1e-3, name
    s = ((u - x2d) * w2d).norm(dim=-1)
    outlier = float((s > delta[:, None]).double().mean())

    cost64, g64 = reference_grad(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min, torch.float64)
    _, g32 = reference_grad(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min, torch.float32)
    out = dict(dof=dof, z_min=z_min, bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               poses=poses.numpy(), upstream=up.numpy(), ref64_cost=cost64.numpy(), grad_pose=g64.numpy(),
               ref32_grad_pose=g32.numpy(), frac_below_zmin=below, frac_clamped=clamped, frac_outlier=outlier)
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: B={B} N={N} P={P} dof={dof}  below z_min {below:.1%}  clamped {clamped:.1%}  "
          f"outlier pairs ~{outlier:.1%}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6_tensor_bounds", B=3, N=200, P=24, seed=51, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_scalar_bounds", B=3, N=128, P=16, seed=52, bounds="scalar")
    run_case("dof4_tensor_bounds", B=3, N=96, P=20, dof=4, seed=53, bounds="tensor", bound_margin=6.25)
    run_case("dof6_below_zmin", B=3, N=128, P=16, seed=54, z_min=4.7, tz=5.0)
    run_case("dof6_small_delta", B=3, N=160, P=20, seed=55, relative_delta=0.05, outlier_frac=0.1)
    run_case("dof4_small_delta", B=2, N=96, P=12, dof=4, seed=56, relative_delta=0.05, outlier_frac=0.1)


if __name__ == "__main__":
    main()
