#!/usr/bin/env python
"""What the second-order pass through the cost costs: a create_graph training step (MonteCarloPoseLoss, then a
gradient-norm loss on the correspondences) against the first-order step, and the point-major and pose-major
Hessian-vector-product kernels (epnp_cost_hvp_f32) against the first-order cost_backward_kernel / cost_pose_backward
at the same shape.  CUDA events over many repetitions after a warm-up; prints one JSON line with the device name and
power limit.

    python tools/cost_hvp_timing.py [--reps 50]"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "epro-pnp_b200")]

import torch  # noqa: E402

from epropnp.camera import PerspectiveCamera  # noqa: E402
from epropnp.cost_fun import AdaptiveHuberPnPCost  # noqa: E402
from epropnp.epropnp import EProPnP6DoF  # noqa: E402
from epropnp.levenberg_marquardt import LMSolver  # noqa: E402
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss  # noqa: E402
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_noise, make_problem  # noqa: E402

SHAPES = [("6dof_train", 32, 512, 512), ("det_like", 1024, 64, 128)]


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def measure(B, N, M, reps, dev):
    pc = make_problem(B, N, seed=1)
    noise = tuple(t.to(dev) for t in make_noise(B, M, seed=2))
    layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=5))
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"].to(dev))
    x3d = pc["x3d"].to(dev)
    loss_fn = MonteCarloPoseLoss().to(dev)

    def step(second):
        x2d = pc["x2d"].to(dev).requires_grad_(True)
        w2d = pc["w2d"].to(dev).requires_grad_(True)
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d.detach(), w2d.detach())
        _, _, _, _, logw, cost_init = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=pc["pose_init"].to(dev), force_init_solve=False,
            with_cost=True, amis_noise=noise)
        loss = loss_fn(logw, cost_init, 1.0).sum()
        if not second:
            loss.backward()
            return
        gx, gw = torch.autograd.grad(loss, (x2d, w2d), create_graph=True)
        (loss + (gx * gx).sum() + (gw * gw).sum()).backward()

    out = dict(B=B, N=N, M=M, step_first_ms=timed(lambda: step(False), reps),
               step_second_ms=timed(lambda: step(True), reps))
    # the kernels alone: M samples plus the cost_init pose per object
    prob = native.Problem(x3d, pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          torch.full((B,), 0.5, device=dev))
    poses = pc["pose_init"].to(dev)[:, None].repeat(1, M + 1, 1).contiguous()
    grad = torch.randn(B, M + 1, device=dev)
    t = dict(x3d=torch.randn(B, N, 3, device=dev), x2d=torch.randn(B, N, 2, device=dev),
             w2d=torch.randn(B, N, 2, device=dev), delta=torch.randn(B, device=dev))
    tp = dict(pose=torch.randn(B, M + 1, 7, device=dev))
    pts = (True, True, True, True, False, False, False, False, False)
    pose_out = (False, False, False, False, True, True, False, False, False)
    out["cost_backward_ms"] = timed(lambda: native.cost_backward(prob, 6, 0.1, poses, grad), reps)
    out["hvp_point_ms"] = timed(lambda: native.cost_hvp(prob, 6, 0.1, poses, grad, t, pts), reps)
    out["cost_pose_backward_ms"] = timed(lambda: native.cost_pose_backward(prob, 6, 0.1, poses, grad), reps)
    out["hvp_pose_ms"] = timed(lambda: native.cost_hvp(prob, 6, 0.1, poses, grad, tp, pose_out), reps)
    return out


def few_poses(B, N, P, reps, dev):
    """The pose-major kernel where it is weakest: thread per pose, so B * P threads stream N points each."""
    pc = make_problem(B, N, seed=3)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          torch.full((B,), 0.5, device=dev))
    poses = pc["pose_init"].to(dev)[:, None].repeat(1, P, 1).contiguous()
    grad = torch.randn(B, P, device=dev)
    tp = dict(pose=torch.randn(B, P, 7, device=dev))
    pose_out = (False, False, False, False, True, True, False, False, False)
    pts = (True, True, True, True, False, False, False, False, False)
    t = dict(x3d=torch.randn(B, N, 3, device=dev))
    return dict(B=B, N=N, P=P, cost_pose_backward_ms=timed(lambda: native.cost_pose_backward(prob, 6, 0.1, poses, grad),
                                                           reps),
                hvp_pose_ms=timed(lambda: native.cost_hvp(prob, 6, 0.1, poses, grad, tp, pose_out), reps),
                hvp_point_ms=timed(lambda: native.cost_hvp(prob, 6, 0.1, poses, grad, t, pts), reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res = dict(device=q, reps=args.reps, shapes={name: measure(B, N, M, args.reps, dev) for name, B, N, M in SHAPES},
               few_poses=[few_poses(B, 16384, P, args.reps, dev) for B, P in ((2, 1), (2, 3), (32, 3))])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
