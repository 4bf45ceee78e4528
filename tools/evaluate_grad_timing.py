#!/usr/bin/env python
"""Forward + backward through evaluate_pnp(out_residual, out_jacobian, out_cost) on the GPU: the native path (the
forward kernel and epnp_evaluate_backward_f32) against the torch composite the reference runs
(PerspectiveCamera.project + HuberPnPCost.compute under autograd), at (S, B, N) = (1, 32, 4096) -- LMSolver.gn_step on
a dense map -- (64, 32, 512) and (64, 32, 4096) -- a reprojection loss on a stack of hypotheses.  Gradients with respect
to x3d, x2d, w2d and the pose; the loss is <g_res, residual> + <g_jac, jacobian> + <g_cost, cost> with fixed upstreams.
Both arms' gradients are also compared with the composite's in float64 on the same inputs.

    python tools/evaluate_grad_timing.py [--reps 15] [--out RESULT.json]

Each time is the median of `reps` steps timed one by one with CUDA events after three warm-up steps, the arms
alternating, with the minimum and maximum; the peak memory is torch.cuda.max_memory_allocated over one step above what
was allocated before it.  The card's name and power limit are read in the same run and stored beside the numbers.
Fails without a CUDA device: there is nothing to measure on a CPU."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "epro-pnp_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from camera_grad_timing import card, measure, rel  # noqa: E402

HUBER_EPS = 1e-10


def setup(S, B, N, dev, seed=3):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp_b200 import native
    from epropnp_b200.synth import make_problem
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, outlier_frac=0.1).items()}
    g = torch.Generator(device=dev).manual_seed(seed)
    pose = pc["pose_gt"][None].repeat(S, 1, 1)
    pose[..., :3] += 0.02 * torch.randn(S, B, 3, generator=g, device=dev)
    pose = pose if S > 1 else pose[0]
    lead = pose.shape[:-1]
    ups = (torch.randn(lead + (2 * N,), generator=g, device=dev), torch.randn(lead + (2 * N, 6), generator=g, device=dev),
           torch.randn(lead, generator=g, device=dev))
    leaves = [pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d")] + [pose.clone().requires_grad_(True)]
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.1)
    cost_fun = HuberPnPCost(delta=native.adaptive_delta(pc["x2d"], pc["w2d"], 0.1), eps=HUBER_EPS)
    return leaves, camera, cost_fun, ups


def arms(leaves, camera, cost_fun, ups):
    from epropnp.common import evaluate_pnp

    def native_step():
        r, c, j = evaluate_pnp(*leaves, camera, cost_fun, out_residual=True, out_jacobian=True, out_cost=True)
        return torch.autograd.grad((r * ups[0]).sum() + (j * ups[1]).sum() + (c * ups[2]).sum(), leaves)

    def composite_step():
        x3d, x2d, w2d, pose = leaves
        x2d_proj, jac_cam = camera.project(x3d, pose, out_jac=True, clip_jac=True)
        r, c, j = cost_fun.compute(x2d_proj, x2d, w2d, jac_cam=jac_cam, out_residual=True, out_cost=True,
                                   out_jacobian=True)
        return torch.autograd.grad((r * ups[0]).sum() + (j * ups[1]).sum() + (c * ups[2]).sum(), leaves)
    return dict(native=native_step, composite=composite_step)


def float64_grads(leaves, camera, cost_fun, ups):
    """The composite's gradients in float64 on the same inputs: the reference both arms are held to."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    d = torch.float64
    leaves64 = [t.detach().to(d).requires_grad_(True) for t in leaves]
    cam64 = PerspectiveCamera(cam_mats=camera.cam_mats.to(d), z_min=camera.z_min)
    cf64 = HuberPnPCost(delta=cost_fun.delta.to(d), eps=HUBER_EPS)
    grads = arms(leaves64, cam64, cf64, [u.to(d) for u in ups])["composite"]()
    return [g.float() for g in grads]


def peak_bytes(step, dev):
    torch.cuda.synchronize(dev)
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    out = step()
    torch.cuda.synchronize(dev)
    peak = torch.cuda.max_memory_allocated(dev) - base
    del out
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    result = dict(card=card(), shapes=[])
    for S, B, N in ((1, 32, 4096), (64, 32, 512), (64, 32, 4096)):
        inputs = setup(S, B, N, dev)
        steps = arms(*inputs)
        row, live = measure(steps, dev, args.reps)
        row.update(S=S, B=B, N=N)
        for k, f in live.items():
            row[k + "_peak_MB"] = peak_bytes(f, dev) / 2 ** 20
        if len(live) == 2:
            ref = float64_grads(*inputs)
            for k, f in live.items():       # largest |error| of each input's gradient over its largest |value|
                row[k + "_vs_float64_grad_rel_max"] = rel(f(), ref)
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
        del inputs, steps, live
        torch.cuda.empty_cache()
    print(json.dumps(result["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
