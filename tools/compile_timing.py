#!/usr/bin/env python
"""The layer's step eagerly, under torch.compile (default mode and mode="reduce-overhead") and as a manual CUDA-graph
replay, at the shapes of tools/graph_replay_timing.py:

    train6   the 6DoF training step: B = 32, N = 512, M = 512, RSLMSolver(num_proposals=4), force_init_solve=True,
             pose_opt_plus, MonteCarloPoseLoss, backward
    det4     a Det-shaped 4-DoF inference: B = 64, N = 256, M = 128, RSLM init with P = 64, monte_carlo_forward

    python tools/compile_timing.py [--steps 100] [--rounds 5] [--parent DIR] [--out RESULT.json]

Each variant is timed with CUDA events over `steps` back-to-back steps after a warm-up, `rounds` rounds with the
variants alternating; the median and the range of the rounds are reported.  torch.compile compiles the forward and the
loss; backward() runs outside, on the compiled backward graph.

--parent DIR: a directory holding another version's `epropnp` package (for example the parent commit's
epro-pnp_b200/epropnp, from `git archive`).  It is imported under another name beside this tree's and its eager step
alternates with this tree's in the same rounds, so the two eager paths (the operators against the autograd.Function
classes they replaced) are compared on one card in one run.  The native library is this tree's for both.

The card's name and power limit are read in the same run.  Needs a CUDA device; without one every number is reported
as not measured."""
import argparse
import importlib.util
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "epro-pnp_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from graph_replay_timing import card, time_steps  # noqa: E402


def load_package(path, name):
    """Import the `epropnp` package at `path` as `name` (its relative imports resolve inside it)."""
    spec = importlib.util.spec_from_file_location(name, os.path.join(path, "__init__.py"),
                                                  submodule_search_locations=[path])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    for sub in ("camera", "cost_fun", "epropnp", "levenberg_marquardt", "monte_carlo_pose_loss"):
        importlib.import_module(f"{name}.{sub}")
    return mod


def workload(kind, dev, pkg="epropnp"):
    """-> (description, fwd, backward): fwd() returns the loss (train6) or the pose (det4); the step is fwd() then,
    for train6, loss.backward()."""
    m = lambda sub: sys.modules[f"{pkg}.{sub}"]
    from epropnp_b200.synth import make_problem
    if kind == "train6":
        B, N, M, I, P, dof = 32, 512, 512, 4, 4, 6
    else:
        B, N, M, I, P, dof = 64, 256, 128, 4, 64, 4
    pc = make_problem(B, N, seed=1, dof=dof)
    inp = {k: pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats", "pose_gt")}
    camera = m("camera").PerspectiveCamera(cam_mats=inp["cam_mats"])
    lmm = m("levenberg_marquardt")
    solver = lmm.LMSolver(dof=dof, num_iter=10,
                          init_solver=lmm.RSLMSolver(dof=dof, num_points=16, num_proposals=P, num_iter=3))
    if kind == "train6":
        layer = m("epropnp").EProPnP6DoF(mc_samples=M, num_iter=I, solver=solver)
        loss_fn = m("monte_carlo_pose_loss").MonteCarloPoseLoss().to(dev)
        leaves = tuple(inp[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))

        def fwd():
            x3d, x2d, w2d = leaves
            cost_fun = m("cost_fun").AdaptiveHuberPnPCost(relative_delta=0.5)
            cost_fun.set_param(x2d.detach(), w2d)
            _, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(
                x3d, x2d, w2d, camera, cost_fun, pose_init=inp["pose_gt"], force_init_solve=True,
                with_pose_opt_plus=True)
            return loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - inp["pose_gt"]).abs().sum()

        def clear():
            for t in leaves:
                t.grad = None
        return f"6DoF training step B={B} N={N} M={M} RSLM P={P}", fwd, clear
    layer = m("epropnp").EProPnP4DoF(mc_samples=M, num_iter=I, solver=solver)

    def fwd():
        cost_fun = m("cost_fun").AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(inp["x2d"], inp["w2d"])
        return layer.monte_carlo_forward(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun)[0]
    return f"4DoF inference B={B} N={N} M={M} RSLM P={P}", fwd, None


def make_step(fwd, clear):
    if clear is None:
        return fwd

    def step():
        clear()
        fwd().backward()
    return step


def graph_step(step):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g.replay


def summary(rounds):
    return dict(median_ms=round(statistics.median(rounds), 4), min_ms=round(min(rounds), 4),
                max_ms=round(max(rounds), 4), rounds_ms=[round(x, 4) for x in rounds])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--parent", default=None, help="directory of another version's epropnp package (eager A/B)")
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    kinds = ("train6", "det4")
    if not torch.cuda.is_available():
        print(json.dumps(dict(card="not measured", workloads={k: "not measured" for k in kinds}), indent=1))
        return
    import epropnp.camera, epropnp.cost_fun, epropnp.epropnp, epropnp.levenberg_marquardt  # noqa: F401,E401
    import epropnp.monte_carlo_pose_loss  # noqa: F401
    if args.parent:
        load_package(args.parent, "epropnp_parent")
    # Python floats (Huber and solver constants, loss weights) specialised: unspecialised, they would become CPU scalar
    # inputs whose arithmetic inductor compiles to host C++ kernels
    torch._dynamo.config.specialize_float = True
    dev = torch.device("cuda:0")
    result = dict(card=card(), steps_per_round=args.steps, workloads={})
    for kind in kinds:
        what, fwd, clear = workload(kind, dev)
        variants = dict(eager=make_step(fwd, clear))
        if args.parent:
            variants["eager_parent"] = make_step(*workload(kind, dev, "epropnp_parent")[1:])
        for mode in ("default", "reduce-overhead"):
            _, f, c = workload(kind, dev)
            variants[f"compile_{mode}"] = make_step(torch.compile(f, mode=mode), c)
        _, f, c = workload(kind, dev)
        variants["graph_replay"] = graph_step(make_step(f, c))
        for step in variants.values():                  # compile and warm every variant before any timing
            for _ in range(10):
                step()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, step in variants.items():
                times[k].append(time_steps(step, args.steps))
        entry = dict(what=what, **{k: summary(v) for k, v in times.items()})
        if args.parent:
            entry["eager_vs_parent"] = round(entry["eager"]["median_ms"] / entry["eager_parent"]["median_ms"], 4)
        result["workloads"][kind] = entry
        print(f"{what} on {result['card']['name']} at power limit {result['card']['power_limit']}: " +
              ", ".join(f"{k} {v['median_ms']:.3f} ms" for k, v in entry.items() if isinstance(v, dict)), flush=True)
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
