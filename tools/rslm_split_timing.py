#!/usr/bin/env python
"""CUDA-event timing of the cluster-split RSLM initialiser (epnp_rslm_split_f32) at N = 16 384, n = 16, lm_iter = 3.

At each (B, N, P) it times
  * split      the initialiser: refine, score on the clusters, select (three launches);
  * composed   the same work from existing calls: gathered (P B, n, .) mini-problems -> lm_solve -> evaluate_cost_split
               -> torch.min;
  * train      the reference's 6DoF training step (EPro-PnP-6DoF/lib/train.py: RSLM P hypotheses inside LMSolver(5)
               inside EProPnP6DoF(512, 4), pose_opt_plus, Monte-Carlo pose loss, backward) with force_init_solve=True
               on the split initialiser, and with force_init_solve=False (what runs at this N without it).
Each is the median of --reps timed calls (min - max beside it) after warm-up.  The card's name and power limit are read
in the same run.  The two initialisers' winners must agree or be cost-equivalent (1e-4); the script exits 1 otherwise.

    python tools/rslm_split_timing.py [--reps 15] [--shapes 32,16384,4 256,16384,4 32,16384,64]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "epro-pnp_b200")]

import torch  # noqa: E402

from epropnp.camera import PerspectiveCamera  # noqa: E402
from epropnp.cost_fun import AdaptiveHuberPnPCost  # noqa: E402
from epropnp.epropnp import EProPnP6DoF  # noqa: E402
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver  # noqa: E402
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss  # noqa: E402
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_problem  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return dict(median_ms=ms[len(ms) // 2], min_ms=ms[0], max_ms=ms[-1], reps=reps)


def shape_run(B, N, P, n, reps, dev):
    pc = make_problem(B, N, seed=B + P, dof=6, outlier_frac=0.2)
    d = {k: v.to(dev) for k, v in pc.items()}
    delta = native.adaptive_delta(d["x2d"], d["w2d"], 0.1)
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], None, None, delta)
    inds, start = native.rslm_draw(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], P, n, 6, seed=5)
    params = native.default_params(6, lm_iter=3, z_min=0.1)
    rows = torch.arange(B, device=dev)[None, :, None]
    li = inds.long()

    def composed():
        mini = native.Problem(prob.x3d[rows, li].reshape(P * B, n, 3), prob.x2d[rows, li].reshape(P * B, n, 2),
                              prob.w2d[rows, li].reshape(P * B, n, 2), prob.cam.repeat(P, 1, 1), None, None,
                              prob.delta.repeat(P))
        pose_all = native.lm_solve(mini, start.reshape(P * B, 7), params)["pose_opt"].reshape(P, B, 7)
        cost_all = native.evaluate_cost_split(prob, pose_all, 6, params.z_min)
        cost, win = cost_all.min(dim=0)
        return pose_all[win, torch.arange(B, device=dev)], cost

    out = dict(B=B, N=N, P=P, n=n)
    out["split"] = timed(lambda: native.rslm_split(prob, inds, start, params), reps)
    out["composed"] = timed(composed, reps)
    a = native.rslm_split(prob, inds, start, params)
    _, c_comp = composed()
    rel = ((a["cost"] - c_comp).abs() / c_comp.abs())
    out["winner_cost_rel_max"] = float(rel.max())
    out["winners_cost_equivalent"] = bool((rel < 1e-4).all())

    camera = PerspectiveCamera(cam_mats=d["cam_mats"])
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    rslm = RSLMSolver(dof=6, num_points=n, num_proposals=P, num_iter=3, cluster_split=True)
    layer = EProPnP6DoF(mc_samples=512, num_iter=4, solver=LMSolver(dof=6, num_iter=5, init_solver=rslm))
    loss_fn = MonteCarloPoseLoss().to(dev)
    leaves = tuple(d[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))

    def step(force):
        x3d, x2d, w2d = leaves
        for t in leaves:
            t.grad = None
        cost_fun.set_param(x2d.detach(), w2d)
        _, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=d["pose_gt"],
                                                                    force_init_solve=force, with_pose_opt_plus=True)
        (loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - d["pose_gt"]).abs().sum()).backward()

    out["train_force_init_solve"] = timed(lambda: step(True), reps)
    out["train_no_init_solve"] = timed(lambda: step(False), reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--shapes", nargs="*", default=["32,16384,4", "256,16384,4", "32,16384,64"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rslm_split_timing: no CUDA device (timings are only taken on the GPU)")
    dev = torch.device("cuda:0")
    res = dict(card=card(), shapes=[])
    for s in args.shapes:
        B, N, P = (int(x) for x in s.split(","))
        r = shape_run(B, N, P, 16, args.reps, dev)
        res["shapes"].append(r)
        print(json.dumps(r), flush=True)
    res["card_after"] = card()
    print(json.dumps(dict(card=res["card"], card_after=res["card_after"])))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    sys.exit(0 if all(r["winners_cost_equivalent"] for r in res["shapes"]) else 1)


if __name__ == "__main__":
    main()
