#!/usr/bin/env python
"""The camera gradients' cost on the GPU: the native camera backwards against the torch composite that computes the same
gradients (PerspectiveCamera.project + HuberPnPCost.compute under autograd), at

    evaluate_pnp(out_cost=True) on a (S, B, N) = (512, 32, 512) stack, forward + backward with respect to cam_mats and
        per-object lb / ub
    the camera backward of the 6DoF training step (lib/train.py: the Monte-Carlo log-weights, cost_init and pose_opt_plus)
        at B = 32, M = 512 and N = 512, 16 384: the inputs of one forward, then the cost and GN-plus camera backwards
        (native) or the autograd of the same three terms (composite); the composite is tried and what happens reported
    the whole training step (forward + backward) at the same sizes with and without the camera requiring grad

    python tools/camera_grad_timing.py [--reps 15] [--out RESULT.json]

Each number is the median of `reps` steps timed one by one with CUDA events after three warm-up steps, the arms
alternating, with the minimum and maximum.  The card's name and power limit are read in the same run and stored beside
the numbers.  Fails without a CUDA device: there is nothing to measure on a CPU."""
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

EPS, HUBER_EPS = 1e-5, 1e-10


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return dict(name=name, power_limit=power)
    except Exception:
        return dict(name=torch.cuda.get_device_name(0), power_limit="not measured")


def timed(step, dev):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    step()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b)


def measure(steps, dev, reps):
    """steps: {arm: callable}.  Arms that run out of memory in the warm-up are reported, not timed."""
    row, live = {}, {}
    for k, f in steps.items():
        try:
            for _ in range(3):
                f()
            torch.cuda.synchronize(dev)
            live[k] = f
        except torch.OutOfMemoryError as e:
            row[k] = "did not run: " + str(e).split(".")[0]
            torch.cuda.empty_cache()
    times = {k: [] for k in live}
    for _ in range(reps):
        for k, f in live.items():
            times[k].append(timed(f, dev))
    for k, v in times.items():
        row[k + "_ms_median"] = statistics.median(v)
        row[k + "_ms_min_max"] = (min(v), max(v))
    return row, live


def rel(a, b):
    return float(max((x - y).abs().max() / y.abs().max().clamp(min=1e-30) for x, y in zip(a, b)))


def problem(B, N, dev, seed=1):
    from epropnp_b200.synth import make_problem
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, outlier_frac=0.1,
                                                grid2d=round(N ** 0.5) ** 2 == N).items()}
    lo, hi = pc["x2d"].amin(1), pc["x2d"].amax(1)
    border = 30 * (hi - lo) / (round(N ** 0.5) - 1)                    # lib/train.py:169-174
    return pc, lo - border, hi + border


def stack_arms(S, B, N, dev):
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    pc, lb0, ub0 = problem(B, N, dev)
    K = pc["cam_mats"].clone().requires_grad_(True)
    lb, ub = lb0.clone().requires_grad_(True), ub0.clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=K, z_min=0.1, lb=lb, ub=ub)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    poses = pc["pose_init"][None].repeat(S, 1, 1)
    poses[..., :3] += 0.02 * torch.randn(S, B, 3, device=dev)

    def native_step():
        cost = evaluate_pnp(pc["x3d"], pc["x2d"], pc["w2d"], poses, camera, cost_fun, out_cost=True)[1]
        return torch.autograd.grad(cost.sum(), [K, lb, ub])

    def composite_step():
        proj, _ = camera.project(pc["x3d"], poses, out_jac=False)
        cost = cost_fun.compute(proj, pc["x2d"], pc["w2d"], out_cost=True)[1]
        return torch.autograd.grad(cost.sum(), [K, lb, ub])
    return dict(native=native_step, composite=composite_step)


def train_arms(B, N, M, dev):
    """The camera backward of one training step: inputs from one forward, then the native or the composite backward."""
    from epropnp import autograd as ag
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    from epropnp_b200 import native
    pc, lb0, ub0 = problem(B, N, dev)
    K0 = pc["cam_mats"][0]
    init = RSLMSolver(dof=6, num_points=16, num_proposals=64, num_iter=3, cluster_split=True)
    layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=5, init_solver=init))
    mc_loss = MonteCarloPoseLoss().to(dev)

    def step(camera_grad):
        K = K0.clone().requires_grad_(camera_grad)
        lb, ub = lb0.clone().requires_grad_(camera_grad), ub0.clone().requires_grad_(camera_grad)
        camera = PerspectiveCamera(cam_mats=K[None].expand(B, -1, -1), z_min=0.01, lb=lb, ub=ub)
        x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
        cost_fun.set_param(x2d, w2d)
        pose_opt, _, plus, samples, logw, cost_tgt = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=pc["pose_gt"], force_init_solve=True, with_pose_opt_plus=True,
            amis_seed=7)
        loss = mc_loss(logw, cost_tgt, torch.tensor(1.0, device=dev)) + (plus - pc["pose_gt"]).square().sum()
        return loss, [x3d, x2d, w2d] + ([K, lb, ub] if camera_grad else []), (pose_opt, plus, samples, logw, cost_tgt,
                                                                              cost_fun)

    # one forward: the samples, pose_opt and the upstream gradients the camera backward receives
    loss, leaves, (pose_opt, plus, samples, logw, cost_tgt, cost_fun) = step(True)
    g_logw, g_cost, g_plus = torch.autograd.grad(loss, [logw, cost_tgt, plus])
    delta = cost_fun.delta.detach()
    K = K0[None].expand(B, -1, -1).contiguous()
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], K, lb0, ub0, delta)
    samples_bm = samples.detach().transpose(0, 1).contiguous()
    poses = torch.cat((pc["pose_gt"][:, None], samples_bm), 1)                 # (B, M + 1, 7)
    up = torch.cat((g_cost.reshape(B, 1), -g_logw.T), 1)

    def native_backward():
        a = native.cost_camera_backward(prob, 6, 0.01, samples_bm, -g_logw.T.contiguous(), pc["pose_gt"][:, None],
                                        g_cost.reshape(B, 1))
        b = native.gn_plus_camera_backward(prob, pose_opt.detach(), g_plus, 6, 0.01, EPS, HUBER_EPS)
        return [x + y for x, y in zip(a, b)]

    def composite_backward():
        leaf = lambda t: t.clone().requires_grad_(True)
        Kc, lbc, ubc = leaf(K), leaf(lb0), leaf(ub0)
        camera = PerspectiveCamera(cam_mats=Kc, z_min=0.01, lb=lbc, ub=ubc)
        from epropnp.cost_fun import HuberPnPCost
        hub = HuberPnPCost(delta=delta, eps=HUBER_EPS)
        proj, _ = camera.project(pc["x3d"], poses.transpose(0, 1), out_jac=False)
        cost = hub.compute(proj, pc["x2d"], pc["w2d"], out_cost=True)[1]               # (M + 1, B)
        solver = LMSolver(dof=6, eps=EPS)
        pose = pose_opt.detach()
        pl = solver.pose_add(pose, ag.gn_step_autograd(solver, pc["x3d"], pc["x2d"], pc["w2d"], pose, camera, hub),
                             camera)
        return torch.autograd.grad((cost * up.T).sum() + (pl * g_plus).sum(), [Kc, lbc, ubc])

    def full(camera_grad):
        def f():
            loss, leaves, _ = step(camera_grad)
            return torch.autograd.grad(loss, leaves)
        return f
    return (dict(native=native_backward, composite=composite_backward),
            dict(step_with_camera_grad=full(True), step_without_camera_grad=full(False)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("camera_grad_timing: no CUDA device; nothing measured")
    assert args.reps >= 10, "the median of at least 10 steps"
    dev = torch.device("cuda:0")
    result = dict(card=card(), reps=args.reps, rows=[])
    S, B, N = 512, 32, 512
    arms = stack_arms(S, B, N, dev)
    row, live = measure(arms, dev, args.reps)
    if "composite" in live:
        row["native_vs_composite_rel_max"] = rel(live["native"](), live["composite"]())
    result["rows"].append(dict(what="evaluate_pnp forward + camera backward", S=S, B=B, N=N, **row))
    print(json.dumps(result["rows"][-1]))
    for N in (512, 16384):
        torch.manual_seed(0)
        backward, whole = train_arms(32, N, 512, dev)
        row, live = measure(backward, dev, args.reps)
        if "composite" in live:
            row["native_vs_composite_rel_max"] = rel(live["native"](), live["composite"]())
        result["rows"].append(dict(what="training step: camera backward", B=32, N=N, M=512, **row))
        print(json.dumps(result["rows"][-1]))
        row, _ = measure(whole, dev, args.reps)
        result["rows"].append(dict(what="training step: forward + backward", B=32, N=N, M=512, **row))
        print(json.dumps(result["rows"][-1]))
        torch.cuda.empty_cache()
    print(json.dumps(result["card"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(result, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
