#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/gn_plus_hvp/*.npz: Hessian-vector products of the
derivative-regularisation branch, recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU, float64
autograd with create_graph=True).

    python oracle/make_golden_gn_plus_hvp.py      # needs /root/reference; run in the build container

Every case takes L = <gplus, pose_add(pose, gn_step(pose))> through the reference's LMSolver.gn_step / pose_add
(PerspectiveCamera, HuberPnPCost) at a detached pose, with x3d, x2d, w2d, delta (one per object), cam_mats, tensor
lb / ub and gplus as leaves; then g = dL/d(inputs) with create_graph and, for a tangent u on every input, d(g . u) /
d(inputs, gplus).  The pose is a constant, so the rotation-form caveat of the cost goldens does not arise.  Cases: 6DoF
and 4DoF; no, scalar and tensor bounds that clamp part of the projections; depths below z_min; a small delta for both
Huber branches.  Bounds, z_min and the Huber threshold keep the margins of make_golden_cost_grad.py (whose helpers
this file uses).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                      # noqa: E402  (puts the reference first on sys.path)
from make_golden_cost_grad import PerspectiveCamera, HuberPnPCost, make_problem      # noqa: E402
from epropnp.levenberg_marquardt import LMSolver         # noqa: E402  (reference)

OUT = os.path.join(mk.ROOT, "tests", "golden", "gn_plus_hvp")
NAMES = ("x3d", "x2d", "w2d", "delta", "cam_mats", "lb", "ub")


def hvp(inputs, pose, gplus, z_min, dof, tangents):
    """d((dL/d inputs) . u) / d(inputs, gplus) by the reference's autograd; tensor bounds are inputs, float ones not."""
    leaves = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in inputs.items()}
    gp = gplus.clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=leaves["cam_mats"], z_min=z_min, lb=leaves["lb"], ub=leaves["ub"])
    solver = LMSolver(dof=dof, eps=1e-5)
    cost_fun = HuberPnPCost(delta=leaves["delta"], eps=1e-10)
    step = solver.gn_step(leaves["x3d"], leaves["x2d"], leaves["w2d"], pose, camera, cost_fun)
    plus = solver.pose_add(pose, step, camera)
    keys = [k for k in NAMES if torch.is_tensor(leaves[k])]
    g = torch.autograd.grad((plus * gp).sum(), [leaves[k] for k in keys], create_graph=True)
    dot = sum((gi * tangents[k]).sum() for gi, k in zip(g, keys))
    h = torch.autograd.grad(dot, [leaves[k] for k in keys] + [gp], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = {k: z(hi, leaves[k]).detach().numpy() for hi, k in zip(h[:-1], keys)}
    out["gplus"] = z(h[-1], gp).detach().numpy()
    return out, plus.detach().numpy()


def run_case(name, B, N, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0):
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    pose = mk.stacked_poses(p, 1, dof, seed + 1, tz)[0]
    if dof == 6:
        pose[..., 3:] /= pose[..., 3:].norm(dim=-1, keepdim=True)
    delta = (w2d.mean(dim=(-2, -1)) * x2d.var(dim=-2).sum(-1).sqrt() * relative_delta).float().double()
    if bounds == "tensor":
        lb = (x2d.amin(1) + bound_margin).float().double()
        ub = (x2d.amax(1) - bound_margin).float().double()
    elif bounds == "scalar":
        lb, ub = 110.5, 520.5
    else:
        lb = ub = None

    zh, u = mk.project_unclamped(x3d, pose[None], cam_mats)
    zh, u = zh[0], u[0]
    assert (zh - z_min).abs().min() > 1e-6, name
    u_c = u * (zh / zh.clamp(min=z_min))[..., None]
    clamped = 0.0
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=d) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        gap = torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min()
        assert gap > 1e-3, (name, float(gap))
        clamped = float(((u_c < lbt) | (u_c > ubt)).any(-1).double().mean())
        u_c = torch.minimum(torch.maximum(u_c, lbt), ubt)
    s = ((u_c - x2d) * w2d).norm(dim=-1)
    huber_gap = float(((s - delta[:, None]).abs() / delta[:, None]).min())
    assert huber_gap > 1e-6, (name, huber_gap)

    g = torch.Generator().manual_seed(seed + 3)
    rnd = lambda shape: torch.randn(shape, generator=g, dtype=d)
    gplus = rnd(pose.shape)
    inputs = dict(x3d=x3d, x2d=x2d, w2d=w2d, delta=delta, cam_mats=cam_mats, lb=lb, ub=ub)
    tan = {k: rnd(v.shape) for k, v in inputs.items() if torch.is_tensor(v)}
    tan["cam_mats"] *= 10.0
    h, plus = hvp(inputs, pose, gplus, z_min, dof, tan)

    out = dict(dof=dof, z_min=z_min, relative_delta=relative_delta,
               bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               pose=pose.numpy(), gplus=gplus.numpy(), pose_opt_plus=plus, huber_gap=huber_gap,
               frac_below_zmin=float((zh < z_min).double().mean()), frac_clamped=clamped,
               frac_outlier=float((s > delta[:, None]).double().mean()))
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
    for k, v in tan.items():
        out["tan_" + k] = v.numpy()
    for k, v in h.items():
        out["hvp_" + k] = v
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: B={B} N={N} dof={dof}  below z_min {out['frac_below_zmin']:.1%}  clamped {clamped:.1%}  "
          f"outliers {out['frac_outlier']:.1%}  Huber gap {huber_gap:.1e}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6", B=3, N=160, seed=81, outlier_frac=0.05)
    # outliers among the clamped points: the bounds reach the step through the Huber weight of the other coordinate
    run_case("dof6_tensor_bounds", B=3, N=200, seed=82, bounds="tensor", bound_margin=60.0, relative_delta=0.05,
             outlier_frac=0.1)
    run_case("dof6_scalar_bounds", B=3, N=128, seed=83, bounds="scalar")
    run_case("dof4_tensor_bounds", B=3, N=96, dof=4, seed=84, bounds="tensor", bound_margin=6.25, relative_delta=0.05,
             outlier_frac=0.1)
    run_case("dof6_below_zmin", B=3, N=128, seed=85, z_min=4.7, tz=5.0)
    run_case("dof6_small_delta", B=3, N=160, seed=86, relative_delta=0.05, outlier_frac=0.1)


if __name__ == "__main__":
    main()
