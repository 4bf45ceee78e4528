#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/cost_camera_grad/*.npz: gradients with respect to the CAMERA
(cam_mats and tensor lb / ub), recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU autograd,
float64 and float32).

    python oracle/make_golden_cost_camera_grad.py      # needs /root/reference; run in the build container

Two losses.  "cost" cases: L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) of the reference's evaluate_pnp(...,
out_cost=True) on stacked poses (P, B, D), differentiated with respect to cam_mats (B, 3, 3) and lb / ub (B, 2): per-object
and scalar bounds that clamp part of the projections, 4DoF, depths below z_min, a small delta.  "gn" cases:
L = <g, pose (+) gn_step(pose)> through the reference's LMSolver.gn_step / pose_add at a detached pose (6DoF and 4DoF,
tensor bounds with and without outliers, below z_min).  Bounds and z_min keep the margins of make_golden_cost_grad.py
(whose helpers this file uses).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                      # noqa: E402  (puts the reference first on sys.path)
from make_golden_cost_grad import PerspectiveCamera, HuberPnPCost, evaluate_pnp, make_problem      # noqa: E402
from epropnp.levenberg_marquardt import LMSolver         # noqa: E402  (reference)

OUT = os.path.join(mk.ROOT, "tests", "golden", "cost_camera_grad")


def _leaves(cam_mats, lb, ub, dtype):
    leaf = lambda t: t.to(dtype).clone().requires_grad_(True) if torch.is_tensor(t) else t
    return leaf(cam_mats), leaf(lb), leaf(ub)


def _grads(K, lb, ub):
    g = lambda t: t.grad.numpy() if torch.is_tensor(t) else np.zeros(0)
    return g(K), g(lb), g(ub)


def cost_grad(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min, dtype):
    c = lambda t: t.to(dtype)
    K, lbl, ubl = _leaves(cam_mats, lb, ub, dtype)
    camera = PerspectiveCamera(cam_mats=K, z_min=z_min, lb=lbl, ub=ubl)
    _, cost, _ = evaluate_pnp(c(x3d), c(x2d), c(w2d), c(poses), camera, HuberPnPCost(delta=c(delta)), out_cost=True)
    (cost * c(up)).sum().backward()
    return _grads(K, lbl, ubl)


def gn_grad(x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, gplus, z_min, dof, dtype):
    c = lambda t: t.to(dtype)
    K, lbl, ubl = _leaves(cam_mats, lb, ub, dtype)
    camera = PerspectiveCamera(cam_mats=K, z_min=z_min, lb=lbl, ub=ubl)
    solver = LMSolver(dof=dof, eps=1e-5)
    cost_fun = HuberPnPCost(delta=c(delta), eps=1e-10)
    step = solver.gn_step(c(x3d), c(x2d), c(w2d), c(pose), camera, cost_fun)
    plus = solver.pose_add(c(pose), step, camera)
    (plus * c(gplus)).sum().backward()
    return _grads(K, lbl, ubl)


def _margins(name, x3d, x2d, w2d, poses, cam_mats, lb, ub, z_min, delta):
    zh, u = mk.project_unclamped(x3d, poses, cam_mats)
    below = float((zh < z_min).double().mean())
    assert (zh - z_min).abs().min() > 1e-6, name
    clamped = 0.0
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=torch.float64) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        u_c = u * (zh / zh.clamp(min=z_min))[..., None]
        clamped = float(((u_c < lbt) | (u_c > ubt)).any(-1).double().mean())
        assert torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min() > 1e-3, name
    outlier = float((((u - x2d) * w2d).norm(dim=-1) > delta[:, None]).double().mean())
    return below, clamped, outlier


def run_case(name, B, N, P, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0, loss="cost"):
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    poses = mk.stacked_poses(p, P, dof, seed + 1, tz)
    if dof == 6:
        poses[..., 3:] /= poses[..., 3:].norm(dim=-1, keepdim=True)
    delta = (w2d.mean(dim=(-2, -1)) * x2d.var(dim=-2).sum(-1).sqrt() * relative_delta).float().double()
    if bounds == "tensor":
        lb = (x2d.amin(1) + bound_margin).float().double()
        ub = (x2d.amax(1) - bound_margin).float().double()
    elif bounds == "scalar":
        lb, ub = 110.5, 520.5
    else:
        lb = ub = None
    below, clamped, outlier = _margins(name, x3d, x2d, w2d, poses, cam_mats, lb, ub, z_min, delta)
    out = dict(dof=dof, z_min=z_min, bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               frac_below_zmin=below, frac_clamped=clamped, frac_outlier=outlier, loss=loss)
    if loss == "cost":
        up = mk.upstream(P, B, seed + 2)
        args = (x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min)
        out.update(poses=poses.numpy(), upstream=up.numpy())
        g64, g32 = cost_grad(*args, torch.float64), cost_grad(*args, torch.float32)
    else:
        pose = poses[0]
        gplus = torch.from_numpy(np.random.RandomState(seed + 3).randn(*pose.shape))
        args = (x3d, x2d, w2d, cam_mats, lb, ub, delta, pose, gplus, z_min, dof)
        out.update(pose=pose.numpy(), gplus=gplus.numpy())
        g64, g32 = gn_grad(*args, torch.float64), gn_grad(*args, torch.float32)
    for k, a, b in zip(("cam", "lb", "ub"), g64, g32):
        out[f"grad_{k}"], out[f"ref32_grad_{k}"] = a, b
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: {loss} B={B} N={N} P={P} dof={dof}  below z_min {below:.1%}  clamped {clamped:.1%}  "
          f"outlier pairs ~{outlier:.1%}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6_tensor_bounds", B=3, N=200, P=24, seed=61, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_scalar_bounds", B=3, N=128, P=16, seed=62, bounds="scalar")
    run_case("dof4_tensor_bounds", B=3, N=96, P=20, dof=4, seed=63, bounds="tensor", bound_margin=6.25)
    run_case("dof6_below_zmin", B=3, N=128, P=16, seed=64, z_min=4.7, tz=5.0)
    run_case("dof6_small_delta", B=3, N=160, P=20, seed=65, relative_delta=0.05, outlier_frac=0.1)
    run_case("gn_dof6_tensor_bounds", B=3, N=200, P=1, seed=66, bounds="tensor", bound_margin=16.0, loss="gn")
    run_case("gn_dof4_tensor_bounds", B=3, N=96, P=1, dof=4, seed=67, bounds="tensor", bound_margin=6.25, loss="gn")
    run_case("gn_dof6_below_zmin", B=3, N=128, P=1, seed=68, z_min=4.7, tz=5.0, loss="gn")
    # outliers among the clamped points: the bounds reach the step through the Huber weight of the other coordinate
    run_case("gn_dof6_tensor_bounds_outliers", B=3, N=200, P=1, seed=69, bounds="tensor", bound_margin=16.0,
             relative_delta=0.05, outlier_frac=0.1, loss="gn")


if __name__ == "__main__":
    main()
