#!/usr/bin/env python
"""Forward + backward of evaluate_pnp(out_cost=True) with respect to a stack of poses: the native kernels
(epnp_evaluate_cost_f32 + epnp_cost_pose_backward_f32, or their cluster-split forms) against the torch composite
(PerspectiveCamera.project + HuberPnPCost.compute under autograd), at

    (S, B, N) = (1, 1024, 512), (512, 32, 512), (1, 256, 4096)      both
                (512, 32, 16384)                                      native; the composite is tried and what happens reported

    python tools/pose_grad_timing.py [--reps 15] [--out RESULT.json]

Each number is the median of `reps` steps timed one by one with CUDA events after three warm-up steps, the two arms
alternating.  The card's name and power limit are read in the same run and stored beside the numbers.  Fails without a
CUDA device: there is nothing to measure on a CPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "epro-pnp_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

SHAPES = [(1, 1024, 512), (512, 32, 512), (1, 256, 4096), (512, 32, 16384)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return dict(name=name, power_limit=power)
    except Exception:
        return dict(name=torch.cuda.get_device_name(0), power_limit="not measured")


def arms(S, B, N, dev):
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp_b200.synth import make_problem
    pc = make_problem(B, N, seed=1, outlier_frac=0.1)
    x3d, x2d, w2d = (pc[k].to(dev) for k in ("x3d", "x2d", "w2d"))
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"].to(dev))
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(x2d, w2d)
    poses = pc["pose_init"].to(dev)[None].repeat(S, 1, 1)
    poses[..., :3] += 0.02 * torch.randn(S, B, 3, device=dev)
    poses.requires_grad_(True)

    def native_step():
        cost = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_cost=True)[1]
        return torch.autograd.grad(cost.sum(), poses)[0]

    def composite_step():
        proj, _ = camera.project(x3d, poses, out_jac=False)
        cost = cost_fun.compute(proj, x2d, w2d, out_cost=True)[1]
        return torch.autograd.grad(cost.sum(), poses)[0]
    return native_step, composite_step


def timed(step, dev):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    step()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pose_grad_timing: no CUDA device; nothing measured")
    assert args.reps >= 10, "the median of at least 10 steps"
    dev = torch.device("cuda:0")
    result = dict(card=card(), reps=args.reps, shapes=[])
    for S, B, N in SHAPES:
        native_step, composite_step = arms(S, B, N, dev)
        row = dict(S=S, B=B, N=N)
        steps = {"native": native_step, "composite": composite_step}
        try:
            for _ in range(3):
                composite_step()
            torch.cuda.synchronize(dev)
        except torch.OutOfMemoryError as e:
            row["composite"] = "did not run: " + str(e).split(".")[0]
            del steps["composite"]
            torch.cuda.empty_cache()
        for _ in range(3):
            native_step()
        times = {k: [] for k in steps}
        for _ in range(args.reps):
            for k, f in steps.items():
                times[k].append(timed(f, dev))
        for k, v in times.items():
            row[k + "_ms_median"] = statistics.median(v)
            row[k + "_ms_min_max"] = (min(v), max(v))
        if "composite" in steps:
            g_n, g_c = native_step(), composite_step()
            row["native_vs_composite_rel_max"] = float((g_n - g_c).abs().max() / g_c.abs().max())
        result["shapes"].append(row)
        print(json.dumps(row))
    print(json.dumps(result["card"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(result, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
