#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/cost_grad/*.npz: gradients of the Monte-Carlo cost term,
recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU, float64 autograd).

    python oracle/make_golden_cost_grad.py      # needs /root/reference; run in the build container

Every case evaluates L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) with the reference's
evaluate_pnp(..., out_cost=True) through PerspectiveCamera and HuberPnPCost on stacked poses (P, B, D), and stores
dL/d(x3d, x2d, w2d, delta), with delta a leaf of its own (one value per object).  The upstream weights have mixed signs
and exact zeros.  The cases reach the branches the native backward (epnp_cost_backward_f32) takes: per-object tensor
bounds and scalar bounds that clamp part of the projections, 4DoF, homogeneous depths below z_min, a small delta (both
Huber branches), and rows with zero weights.  Bounds and z_min are placed so that no projection or depth lies within
a margin of them: at an exact tie torch.max / clamp split or pass the gradient in ways this file does not pin.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, "/root/reference")
sys.path.append(os.path.join(ROOT, "epro-pnp_b200"))     # after the reference: `epropnp` must resolve to /root/reference
warnings.filterwarnings("ignore")

import epropnp.camera as ref_camera                    # noqa: E402  (reference)
from epropnp.camera import PerspectiveCamera           # noqa: E402
from epropnp.common import evaluate_pnp                # noqa: E402
from epropnp.cost_fun import HuberPnPCost               # noqa: E402
from epropnp_b200.synth import make_problem            # noqa: E402

assert "/root/reference" in os.path.abspath(ref_camera.__file__)

OUT = os.path.join(ROOT, "tests", "golden", "cost_grad")


def stacked_poses(p, P, dof, seed, tz=None):
    """P poses per object around the ground truth (P, B, D); tz: replace the depth of every pose (z_min case)."""
    g = torch.Generator().manual_seed(seed)
    B = p["pose_gt"].shape[0]
    poses = p["pose_gt"].double()[None].repeat(P, 1, 1)
    poses[..., :3] += 0.05 * torch.randn(P, B, 3, generator=g, dtype=torch.float64)
    if dof == 6:
        q = poses[..., 3:] + 0.05 * torch.randn(P, B, 4, generator=g, dtype=torch.float64)
        poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.1 * torch.randn(P, B, generator=g, dtype=torch.float64)
    if tz is not None:
        poses[..., 2] = tz + 0.05 * torch.randn(P, B, generator=g, dtype=torch.float64)
    return poses.float().double()           # fp32-representable: the fp32 kernels see the same poses


def upstream(P, B, seed):
    g = torch.Generator().manual_seed(seed)
    up = torch.randn(P, B, generator=g, dtype=torch.float64)
    up[torch.rand(P, B, generator=g) < 0.15] = 0.0
    return up


def project_unclamped(x3d, pose, cam_mats):
    """(homogeneous depth zh, projection before the bounds) of every (pose, point), float64, no clamps."""
    from epropnp.common import quaternion_to_rot_mat, yaw_to_rot_mat
    R = yaw_to_rot_mat(pose[..., 3]) if pose.shape[-1] == 4 else quaternion_to_rot_mat(pose[..., 3:])
    xh = (x3d @ R.transpose(-1, -2) + pose[..., None, :3]) @ cam_mats.transpose(-1, -2)
    return xh[..., 2], xh[..., :2] / xh[..., 2:3]


def run_case(name, B, N, P, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0, zero_w=False):
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    if zero_w:          # whole rows and single components with zero weight
        w2d[:, ::7] = 0.0
        w2d[:, 3::11, 1] = 0.0
    poses = stacked_poses(p, P, dof, seed + 1, tz)
    up = upstream(P, B, seed + 2)
    delta = (w2d.mean(dim=(-2, -1)) * x2d.var(dim=-2).sum(-1).sqrt() * relative_delta).float().double()
    if bounds == "tensor":
        lb = (x2d.amin(1) + bound_margin).float().double()
        ub = (x2d.amax(1) - bound_margin).float().double()
    elif bounds == "scalar":
        lb, ub = 110.5, 520.5
    else:
        lb = ub = None

    zh, u = project_unclamped(x3d, poses, cam_mats)
    below = float((zh < z_min).double().mean())
    assert (zh - z_min).abs().min() > 1e-6, name
    clamped = 0.0
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=d) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        u_c = u * (zh / zh.clamp(min=z_min))[..., None]                 # the projection with the z clamp applied
        clamped = float(((u_c < lbt) | (u_c > ubt)).any(-1).double().mean())
        gap = torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min()
        assert gap > 1e-3, (name, float(gap))

    leaf = lambda t: t.clone().requires_grad_(True)
    t3, t2, tw, td = leaf(x3d), leaf(x2d), leaf(w2d), leaf(delta)
    lbr = lb.clone() if torch.is_tensor(lb) else lb
    ubr = ub.clone() if torch.is_tensor(ub) else ub
    camera = PerspectiveCamera(cam_mats=cam_mats, z_min=z_min, lb=lbr, ub=ubr)
    cost_fun = HuberPnPCost(delta=td)
    _, cost, _ = evaluate_pnp(t3, t2, tw, poses, camera, cost_fun, out_cost=True)
    (cost * up).sum().backward()

    s = ((u - x2d) * w2d).norm(dim=-1)          # residual norm without clamps: only used for the branch census
    out = dict(dof=dof, z_min=z_min, relative_delta=relative_delta,
               bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               poses=poses.numpy(), upstream=up.numpy(), ref64_cost=cost.detach().numpy(),
               grad_x3d=t3.grad.numpy(), grad_x2d=t2.grad.numpy(), grad_w2d=tw.grad.numpy(),
               grad_delta=td.grad.numpy(), frac_below_zmin=below, frac_clamped=clamped)
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    outl = float((s > delta[:, None]).double().mean())
    print(f"{name}: B={B} N={N} P={P} dof={dof}  below z_min {below:.1%}  clamped {clamped:.1%}  "
          f"outlier pairs ~{outl:.1%}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6_tensor_bounds", B=3, N=200, P=48, seed=41, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_scalar_bounds", B=3, N=128, P=32, seed=42, bounds="scalar")
    run_case("dof4", B=3, N=96, P=40, dof=4, seed=43, bounds="tensor", bound_margin=6.0)
    run_case("dof6_below_zmin", B=3, N=128, P=32, seed=44, z_min=4.7, tz=5.0)
    run_case("dof6_small_delta", B=3, N=160, P=40, seed=45, relative_delta=0.05, outlier_frac=0.1)
    run_case("dof6_zero_weights", B=2, N=96, P=24, seed=46, zero_w=True, outlier_frac=0.1)


if __name__ == "__main__":
    main()
