#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/evaluate_grad/*.npz: gradients through evaluate_pnp's residual,
Jacobian and cost, recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU autograd, float64 and
float32).

    python oracle/make_golden_evaluate_grad.py      # needs /root/reference; run in the build container

L = sum g_res * residual + sum g_jac * jacobian + sum g_cost * cost of the reference's evaluate_pnp(out_residual=True,
out_jacobian=True, out_cost=True) with seeded random upstream gradients, differentiated with respect to x3d, x2d, w2d,
delta, the pose, cam_mats and tensor lb / ub.  Cases: 6DoF and 4DoF; tensor, scalar and no bounds; depths below z_min;
clip_jac=False; a stacked (3, B, D) pose; a small delta (outliers).  Poses come from make_golden_cost_grad.py's helper,
their quaternions normalised again in float64; bounds and z_min keep its margins.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                      # noqa: E402  (puts the reference first on sys.path)
from make_golden_cost_grad import PerspectiveCamera, HuberPnPCost, evaluate_pnp, make_problem      # noqa: E402

OUT = os.path.join(mk.ROOT, "tests", "golden", "evaluate_grad")
INPUTS = ("x3d", "x2d", "w2d", "delta", "pose", "cam_mats", "lb", "ub")


def grads(inp, ups, z_min, clip_jac, dtype):
    """The reference's autograd of L in `dtype` -> {input: gradient} for the inputs that are tensors."""
    leaves = {k: (v.to(dtype).clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in inp.items()}
    camera = PerspectiveCamera(cam_mats=leaves["cam_mats"], z_min=z_min, lb=leaves["lb"], ub=leaves["ub"])
    cost_fun = HuberPnPCost(delta=leaves["delta"], eps=1e-10)
    res, cost, jac = evaluate_pnp(leaves["x3d"], leaves["x2d"], leaves["w2d"], leaves["pose"], camera, cost_fun,
                                  out_residual=True, out_jacobian=True, out_cost=True, clip_jac=clip_jac)
    g_res, g_jac, g_cost = (u.to(dtype) for u in ups)
    ((res * g_res).sum() + (jac * g_jac).sum() + (cost * g_cost).sum()).backward()
    return {k: v.grad.numpy() for k, v in leaves.items() if torch.is_tensor(v)}


def run_case(name, B, N, P=None, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0, clip_jac=True):
    """P = None: one pose per object, (B, D); else a stacked (P, B, D) pose."""
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    poses = mk.stacked_poses(p, P or 1, dof, seed + 1, tz)
    if dof == 6:            # unit to float64 rounding: the reference's rotation form and the oracle's then agree
        poses[..., 3:] /= poses[..., 3:].norm(dim=-1, keepdim=True)
    pose = poses if P else poses[0]
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
    u_c = u * (zh / zh.clamp(min=z_min))[..., None]
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=d) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        clamped = float(((u_c < lbt) | (u_c > ubt)).any(-1).double().mean())
        assert torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min() > 1e-3, name
        u_c = torch.minimum(torch.maximum(u_c, lbt), ubt)
    s = ((u_c - x2d) * w2d).norm(dim=-1)
    outlier = float((s > delta[:, None]).double().mean())
    assert (s - delta[:, None]).abs().min() > 1e-6, name          # no pair on the Huber kink
    lead = tuple(pose.shape[:-1])
    g = torch.Generator().manual_seed(seed + 2)
    ups = (torch.randn(lead + (2 * N,), generator=g, dtype=d), torch.randn(lead + (2 * N, dof), generator=g, dtype=d),
           torch.randn(lead, generator=g, dtype=d))
    inp = dict(x3d=x3d, x2d=x2d, w2d=w2d, delta=delta, pose=pose, cam_mats=cam_mats, lb=lb, ub=ub)
    g64, g32 = grads(inp, ups, z_min, clip_jac, d), grads(inp, ups, z_min, clip_jac, torch.float32)
    out = dict(dof=dof, z_min=z_min, clip_jac=int(clip_jac),
               bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               pose=pose.numpy(), g_res=ups[0].numpy(), g_jac=ups[1].numpy(), g_cost=ups[2].numpy(),
               frac_below_zmin=below, frac_clamped=clamped, frac_outlier=outlier)
    for k in g64:
        out[f"grad_{k}"], out[f"ref32_grad_{k}"] = g64[k], g32[k]
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: B={B} N={N} pose {lead} dof={dof}  below z_min {below:.1%}  clamped {clamped:.1%}  "
          f"outliers {outlier:.1%}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6_tensor_bounds", B=3, N=96, seed=81, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_scalar_bounds", B=3, N=64, seed=82, bounds="scalar")
    run_case("dof4_tensor_bounds", B=3, N=64, dof=4, seed=83, bounds="tensor", bound_margin=6.25)
    run_case("dof4_none", B=3, N=48, dof=4, seed=84, relative_delta=0.2, outlier_frac=0.1)
    run_case("dof6_below_zmin", B=3, N=64, seed=85, z_min=4.7, tz=5.0)
    run_case("dof6_no_clip", B=3, N=64, seed=86, bounds="tensor", bound_margin=16.0, z_min=4.7, tz=5.0,
             clip_jac=False)
    run_case("dof6_stacked", B=2, N=48, P=3, seed=87, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_small_delta", B=3, N=80, seed=88, relative_delta=0.05, outlier_frac=0.1)


if __name__ == "__main__":
    main()
