#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/cost_hvp/*.npz: Hessian-vector products of the Monte-Carlo cost
term, recorded from the UNMODIFIED reference (/root/reference/epropnp, torch CPU, float64 autograd with
create_graph=True).

    python oracle/make_golden_cost_hvp.py      # needs /root/reference; run in the build container

Every case takes L = sum_{p, b} up[p, b] * cost_b(pose[p, b]) through the reference's evaluate_pnp(..., out_cost=True)
(PerspectiveCamera, HuberPnPCost) on stacked poses (P, B, D), with x3d, x2d, w2d, delta (one per object), the poses,
cam_mats, tensor lb / ub and the upstream weights as leaves; then g = dL/d(inputs) with create_graph and, for a tangent
v, d(g . v)/d(inputs, up).  The cases, poses, upstream weights and margins are those of make_golden_cost_grad.py
(tensor / scalar bounds that clamp part of the projections, 4DoF, depths below z_min, a small delta for both Huber
branches) less the zero-weight rows, where the second derivative of the residual norm at 0 is not defined.

When the pose requires grad the reference forms the rotation as 1 - 2 (jj + kk), ..., which is the raw form
ww + ii - jj - kk, ... minus (|q|^2 - 1) I: the two agree in value and first derivative on the unit sphere only for
directions orthogonal to q.  So each case records two products:
  a) v with every part random and its quaternion part orthogonal to q: every output except the quaternion rows is
     comparable with the raw form;
  b) v without a quaternion part: the quaternion rows are comparable after removing their component along q.
(In 4DoF both forms are the same and every output of (a) is comparable.)  The quaternions are normalised in float64:
these goldens pin the float64 oracle only, and a float32-rounded unit quaternion is off the sphere by some 1e-7.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_cost_grad as mk                     # noqa: E402  (puts the reference first on sys.path)

from epropnp.camera import PerspectiveCamera           # noqa: E402  (reference)
from epropnp.common import evaluate_pnp                # noqa: E402
from epropnp.cost_fun import HuberPnPCost               # noqa: E402
from epropnp_b200.synth import make_problem            # noqa: E402

warnings.filterwarnings("ignore")
OUT = os.path.join(mk.ROOT, "tests", "golden", "cost_hvp")
NAMES = ("x3d", "x2d", "w2d", "delta", "poses", "cam_mats", "lb", "ub")


def hvp(inputs, up, z_min, tangents):
    """d((dL/d inputs) . v) / d(inputs, up) by the reference's autograd; tensor bounds are inputs, float ones not."""
    leaves = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in inputs.items()}
    upl = up.clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=leaves["cam_mats"], z_min=z_min, lb=leaves["lb"], ub=leaves["ub"])
    _, cost, _ = evaluate_pnp(leaves["x3d"], leaves["x2d"], leaves["w2d"], leaves["poses"], camera,
                              HuberPnPCost(delta=leaves["delta"]), out_cost=True)
    keys = [k for k in NAMES if torch.is_tensor(leaves[k])]
    g = torch.autograd.grad((cost * upl).sum(), [leaves[k] for k in keys], create_graph=True)
    dot = sum((gi * tangents[k]).sum() for gi, k in zip(g, keys))
    h = torch.autograd.grad(dot, [leaves[k] for k in keys] + [upl], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = {k: z(hi, leaves[k]).detach().numpy() for hi, k in zip(h[:-1], keys)}
    out["up"] = z(h[-1], upl).detach().numpy()
    return out


def run_case(name, B, N, P, dof=6, seed=0, bounds=None, bound_margin=8.0, z_min=0.1, tz=None, relative_delta=0.5,
             outlier_frac=0.0):
    p = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outlier_frac)
    d = torch.float64
    x3d, x2d, w2d, cam_mats = (p[k].to(d) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    poses = mk.stacked_poses(p, P, dof, seed + 1, tz)
    if dof == 6:            # unit in float64: off the sphere the two rotation forms differ by (|q|^2 - 1) I
        poses[..., 3:] /= poses[..., 3:].norm(dim=-1, keepdim=True)
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
    assert (zh - z_min).abs().min() > 1e-6, name
    u_c = u * (zh / zh.clamp(min=z_min))[..., None]
    if lb is not None:
        lbt, ubt = (torch.as_tensor(b, dtype=d) for b in (lb, ub))
        lbt, ubt = (b.unsqueeze(-2) if b.dim() else b for b in (lbt, ubt))
        gap = torch.minimum((u_c - lbt).abs(), (u_c - ubt).abs()).min()
        assert gap > 1e-3, (name, float(gap))
        u_c = torch.minimum(torch.maximum(u_c, lbt), ubt)
    s = ((u_c - x2d) * w2d).norm(dim=-1)
    huber_gap = float(((s - delta[:, None]).abs() / delta[:, None]).min())
    assert huber_gap > 1e-6, (name, huber_gap)

    g = torch.Generator().manual_seed(seed + 3)
    rnd = lambda shape: torch.randn(shape, generator=g, dtype=d)
    inputs = dict(x3d=x3d, x2d=x2d, w2d=w2d, delta=delta, poses=poses, cam_mats=cam_mats, lb=lb, ub=ub)
    tan = {k: rnd(v.shape) for k, v in inputs.items() if torch.is_tensor(v)}
    tan["cam_mats"] *= 10.0
    if dof == 6:                                            # quaternion tangent orthogonal to q
        q, vq = poses[..., 3:], tan["poses"][..., 3:]
        tan["poses"][..., 3:] = vq - (vq * q).sum(-1, keepdim=True) / (q * q).sum(-1, keepdim=True) * q
    tan_b = {k: v.clone() for k, v in tan.items()}
    tan_b["poses"][..., 3:] = 0.0 if dof == 6 else tan_b["poses"][..., 3:]
    ha, hb = hvp(inputs, up, z_min, tan), hvp(inputs, up, z_min, tan_b)

    out = dict(dof=dof, z_min=z_min, relative_delta=relative_delta,
               bounds=dict(none=0, scalar=1, tensor=2)["none" if bounds is None else bounds],
               x3d=x3d.numpy(), x2d=x2d.numpy(), w2d=w2d.numpy(), cam_mats=cam_mats.numpy(), delta=delta.numpy(),
               poses=poses.numpy(), upstream=up.numpy(), huber_gap=huber_gap,
               frac_below_zmin=float((zh < z_min).double().mean()),
               frac_outlier=float((s > delta[:, None]).double().mean()))
    if lb is not None:
        out["lb"], out["ub"] = (np.asarray(b, dtype=np.float64) for b in (lb, ub))
        out["frac_clamped"] = float((u_c != u * (zh / zh.clamp(min=z_min))[..., None]).any(-1).double().mean())
    for k, v in tan.items():
        out["tan_" + k] = v.numpy()
    for tag, h in (("a", ha), ("b", hb)):
        for k, v in h.items():
            out[f"hvp_{tag}_{k}"] = v
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: B={B} N={N} P={P} dof={dof}  below z_min {out['frac_below_zmin']:.1%}  "
          f"clamped {out.get('frac_clamped', 0.0):.1%}  outliers {out['frac_outlier']:.1%}  "
          f"Huber gap {huber_gap:.1e}  -> {os.path.getsize(path) / 1024:.0f} KiB")


def main():
    torch.set_num_threads(4)
    run_case("dof6_tensor_bounds", B=3, N=200, P=48, seed=41, bounds="tensor", bound_margin=16.0, outlier_frac=0.05)
    run_case("dof6_scalar_bounds", B=3, N=128, P=32, seed=42, bounds="scalar")
    run_case("dof4", B=3, N=96, P=40, dof=4, seed=43, bounds="tensor", bound_margin=6.0)
    run_case("dof6_below_zmin", B=3, N=128, P=32, seed=44, z_min=4.7, tz=5.0)
    run_case("dof6_small_delta", B=3, N=160, P=40, seed=45, relative_delta=0.05, outlier_frac=0.1)


if __name__ == "__main__":
    main()
