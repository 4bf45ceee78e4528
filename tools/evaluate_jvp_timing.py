#!/usr/bin/env python
"""What forward mode costs: the Jacobian-vector-product kernel (epnp_evaluate_jvp_f32, every tangent part given)
against the forward evaluate_full_kernel (epnp_evaluate_f32) and its backward (epnp_evaluate_backward_f32, every
upstream and gradient) at three shapes, all three outputs; then the Monte-Carlo log-weights' tangent (d cost alone at
M stacked poses) pose-major, and point-major (the residual asked for too, which forces that form), against the fused
LM + AMIS forward.  CUDA events over many repetitions after a warm-up; prints one JSON line with the device name and power limit.

    python tools/evaluate_jvp_timing.py [--reps 30]"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "epro-pnp_b200")]

import torch  # noqa: E402

from epropnp_b200 import native, ops  # noqa: E402
from epropnp_b200.synth import make_noise, make_problem  # noqa: E402

SHAPES = [("B32_N512", 32, 512), ("B1024_N64", 1024, 64), ("B1_N16384", 1, 16384)]


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


def _case(B, N, S, dev):
    pc = make_problem(B, N, seed=1)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          torch.full((B,), 2.0, device=dev))
    poses = pc["pose_gt"].to(dev).unsqueeze(0).repeat(S, 1, 1).contiguous()
    gen = torch.Generator().manual_seed(3)
    t = dict(x3d=torch.randn(B, N, 3, generator=gen), x2d=torch.randn(B, N, 2, generator=gen),
             w2d=torch.randn(B, N, 2, generator=gen), delta=torch.randn(B, generator=gen),
             pose=torch.randn(S, B, 7, generator=gen), cam=torch.randn(B, 3, 3, generator=gen))
    return pc, prob, poses, {k: v.to(dev) for k, v in t.items()}


def measure_eval(B, N, reps, dev):
    _, prob, poses, t = _case(B, N, 1, dev)
    g_r, g_j, g_c = (torch.randn(1, B, 2 * N, device=dev), torch.randn(1, B, 2 * N, 6, device=dev),
                     torch.randn(1, B, device=dev))
    fwd = timed(lambda: native.evaluate_full(prob, poses[0], 6, 0.1, 1e-10, True, True, True, True), reps)
    bwd = timed(lambda: native.evaluate_backward(prob, poses, 6, 0.1, 1e-10, True, g_r, g_j, g_c,
                                                 want=(True,) * 6 + (False, False)), reps)
    jvp = timed(lambda: native.evaluate_jvp(prob, poses, 6, 0.1, 1e-10, True, t, (True, True, True)), reps)
    return dict(forward_ms=round(fwd, 4), backward_ms=round(bwd, 4), jvp_ms=round(jvp, 4))


def measure_logw(B, N, M, reps, dev):
    pc, prob, poses, t = _case(B, N, M, dev)
    t.pop("pose")
    noise = tuple(x.to(dev) for x in make_noise(B, M, seed=2))
    ints, floats = ops.param_lists(None, 6, mc_samples=M, lm_iter=5)
    args = ops.problem_args(prob.x3d, prob.x2d, prob.w2d, prob.cam, None, None, prob.delta)
    fused = timed(lambda: ops.lm_amis_fused(*args, pc["pose_init"].to(dev), None, *noise, 0, None, ints, floats, True,
                                            False, False), reps)
    pose_major = timed(lambda: native.evaluate_jvp(prob, poses, 6, 0.1, 1e-10, True, t, (False, False, True)), reps)
    point_major = timed(lambda: native.evaluate_jvp(prob, poses, 6, 0.1, 1e-10, True, t, (True, False, True)), reps)
    return dict(fused_forward_ms=round(fused, 4), logw_jvp_pose_major_ms=round(pose_major, 4),
                logw_jvp_point_major_with_residual_ms=round(point_major, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("evaluate_jvp_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    out = dict(device=q, evaluate={n: measure_eval(B, N, a.reps, dev) for n, B, N in SHAPES},
               logw_B32_N512_M512=measure_logw(32, 512, 512, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
