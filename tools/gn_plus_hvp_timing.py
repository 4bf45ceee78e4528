#!/usr/bin/env python
"""What second order through pose_opt_plus costs: a 6DoF training step (MonteCarloPoseLoss + loss_t / loss_r on
pose_opt_plus, train.py:178-193) with a create_graph gradient-norm penalty on the native kernels, against the same
first-order step and against the penalised step on the torch composite (EPNP_NATIVE_GN_STEP=0); and the
Hessian-vector-product kernel (epnp_gn_plus_hvp_f32) against gn_plus_backward + gn_plus_camera_backward at the same
shape.  CUDA events over many repetitions after a warm-up; prints one JSON line with the device name and power limit.

    python tools/gn_plus_hvp_timing.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "epro-pnp_b200")]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from epropnp.camera import PerspectiveCamera  # noqa: E402
from epropnp.cost_fun import HuberPnPCost  # noqa: E402
from epropnp.epropnp import EProPnP6DoF  # noqa: E402
from epropnp.levenberg_marquardt import LMSolver  # noqa: E402
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss  # noqa: E402
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_noise, make_problem  # noqa: E402
from oracle import pnp_oracle as orc  # noqa: E402

SHAPES = [(32, 512, 512), (32, 16384, 512)]


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
    loss_fn = MonteCarloPoseLoss().to(dev)
    gt = pc["pose_gt"].to(dev)
    delta0 = orc.adaptive_delta(pc["x2d"], pc["w2d"], 0.5).to(dev)

    def step(second):
        leaves = [pc[k].to(dev).requires_grad_(True) for k in ("x3d", "x2d", "w2d")]
        delta, cam = delta0.clone().requires_grad_(True), pc["cam_mats"].to(dev).requires_grad_(True)
        x3d, x2d, w2d = leaves
        _, _, plus, _, logw, cost_init = layer.monte_carlo_forward(
            x3d, x2d, w2d, PerspectiveCamera(cam_mats=cam), HuberPnPCost(delta=delta), pose_init=pc["pose_init"].to(dev),
            force_init_solve=False, with_pose_opt_plus=True, with_cost=True, amis_noise=noise)
        dot = (plus[:, 3:] * gt[:, 3:]).sum(-1)
        loss = (loss_fn(logw, cost_init, 1.0) + F.smooth_l1_loss(plus[:, :3], gt[:, :3], beta=0.05)
                + (1 - dot * dot).mean())
        ins = leaves + [delta, cam]
        if not second:
            loss.backward()
            return
        g = torch.autograd.grad(loss, ins, create_graph=True)
        (loss + sum((gi * gi).sum() for gi in g)).backward()

    out = dict(B=B, N=N, M=M)
    os.environ["EPNP_NATIVE_GN_STEP"] = "1"
    out["step_first_ms"] = timed(lambda: step(False), reps)
    out["step_second_native_ms"] = timed(lambda: step(True), reps)
    os.environ["EPNP_NATIVE_GN_STEP"] = "0"
    out["step_second_composite_ms"] = timed(lambda: step(True), reps)
    os.environ["EPNP_NATIVE_GN_STEP"] = "1"
    # the kernels alone, every output
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          delta0)
    pose, gp = pc["pose_gt"].to(dev), torch.randn(B, 7, device=dev)
    t = dict(x3d=torch.randn(B, N, 3, device=dev), x2d=torch.randn(B, N, 2, device=dev),
             w2d=torch.randn(B, N, 2, device=dev), delta=torch.randn(B, device=dev),
             cam=10 * torch.randn(B, 3, 3, device=dev))
    args = (prob, pose, gp, 6, 0.1, 1e-5, 1e-10)
    split = N > native.max_points(6)
    gnb = native.gn_plus_backward_split if split else native.gn_plus_backward
    out["gn_plus_backward_plus_camera_ms"] = timed(
        lambda: (gnb(*args), native.gn_plus_camera_backward(*args, want=(True, False, False))), reps)
    want = (True, True, True, True, True, False, False, True)
    out["gn_plus_hvp_ms"] = timed(lambda: native.gn_plus_hvp(*args, t, want), reps)
    want_pts = (True, True, True, True, False, False, False, True)
    out["gn_plus_hvp_points_only_ms"] = timed(lambda: native.gn_plus_hvp(*args, t, want_pts), reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print(json.dumps(dict(device=q, reps=args.reps, shapes=[measure(B, N, M, args.reps, dev) for B, N, M in SHAPES])))


if __name__ == "__main__":
    main()
