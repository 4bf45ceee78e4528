#!/usr/bin/env python
"""Eager calls against CUDA-graph replay of the same step, at the small static batches where launch and Python overhead
dominate:

    train6   the 6DoF training step of EPro-PnP-6DoF/lib/train.py: B = 32 objects, N = 512 points, M = 512 samples,
             RSLMSolver(num_proposals=4) with force_init_solve=True, pose_opt_plus, MonteCarloPoseLoss, backward
    det4     a Det-shaped 4-DoF inference: B = 64 objects, N = 256 points, RSLM init with P = 64, monte_carlo_forward

    python tools/graph_replay_timing.py [--steps 200] [--out RESULT.json]

Each step is timed with CUDA events over `steps` back-to-back steps after a warm-up, five rounds, eager and replay
alternating; the median round is reported per step.  The card's name and power limit are read in the same run and
printed beside the numbers.  Needs a CUDA device; without one it reports every number as not measured."""
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return dict(name=name, power_limit=power)
    except Exception:
        return dict(name=torch.cuda.get_device_name(0), power_limit="not measured")


def workload(kind, dev):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP4DoF, EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    from epropnp_b200.synth import make_problem

    if kind == "train6":
        B, N, M, I, P, dof = 32, 512, 512, 4, 4, 6
    else:
        B, N, M, I, P, dof = 64, 256, 128, 4, 64, 4
    pc = make_problem(B, N, seed=1, dof=dof)
    inp = {k: pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats", "pose_gt")}
    camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
    solver = LMSolver(dof=dof, num_iter=10, init_solver=RSLMSolver(dof=dof, num_points=16, num_proposals=P, num_iter=3))
    if kind == "train6":
        layer = EProPnP6DoF(mc_samples=M, num_iter=I, solver=solver)
        loss_fn = MonteCarloPoseLoss().to(dev)
        leaves = tuple(inp[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))

        def step():
            x3d, x2d, w2d = leaves
            for t in leaves:
                t.grad = None
            cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
            cost_fun.set_param(x2d.detach(), w2d)
            _, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(
                x3d, x2d, w2d, camera, cost_fun, pose_init=inp["pose_gt"], force_init_solve=True,
                with_pose_opt_plus=True)
            loss = loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - inp["pose_gt"]).abs().sum()
            loss.backward()
        what = f"6DoF training step B={B} N={N} M={M} RSLM P={P}"
    else:
        layer = EProPnP4DoF(mc_samples=M, num_iter=I, solver=solver)

        def step():
            cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
            cost_fun.set_param(inp["x2d"], inp["w2d"])
            layer.monte_carlo_forward(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun)
        what = f"4DoF inference B={B} N={N} M={M} RSLM P={P}"
    return what, step


def time_steps(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    result = dict(card="not measured", workloads={})
    if not torch.cuda.is_available():
        for kind in ("train6", "det4"):
            result["workloads"][kind] = dict(eager_ms="not measured", replay_ms="not measured")
        print(json.dumps(result, indent=1))
        return
    dev = torch.device("cuda:0")
    result["card"] = card()
    for kind in ("train6", "det4"):
        what, step = workload(kind, dev)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for _ in range(10):
            step()
            g.replay()
        eager, replay = [], []
        for _ in range(5):
            eager.append(time_steps(step, args.steps))
            replay.append(time_steps(g.replay, args.steps))
        e, r = statistics.median(eager), statistics.median(replay)
        result["workloads"][kind] = dict(what=what, eager_ms=round(e, 4), replay_ms=round(r, 4),
                                         speedup=round(e / r, 2), eager_rounds_ms=[round(x, 4) for x in eager],
                                         replay_rounds_ms=[round(x, 4) for x in replay], steps_per_round=args.steps)
        print(f"{what}: eager {e:.3f} ms/step, replay {r:.3f} ms/step ({e / r:.2f}x) on {result['card']['name']} "
              f"at power limit {result['card']['power_limit']}", flush=True)
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
