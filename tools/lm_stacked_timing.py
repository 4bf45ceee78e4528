#!/usr/bin/env python
"""What stacked starts save: the LM / GN solve from S starts per object in one call (epnp_lm_solve_stacked_f32, each
object's points staged once per CTA of up to 8 hypothesis warps) against the replicate-and-flatten call a caller makes
without it (the correspondences copied S times, epnp_lm_solve_f32 on S B objects), on the same inputs.  The flattened
call is timed twice: on inputs replicated beforehand (the solve alone) and with the replication in the timed call (what
the caller pays).  6DoF LM with 10 iterations and 4DoF fast-mode GN with 5, B = 1024, N = 512 at S = 2, 8, 32 and
N = 4096 at S = 8; pose_opt and cost asked for.  The three calls alternate in one process, CUDA events over `--reps`
calls per round, median of `--rounds` rounds; the outputs are checked bit for bit first.  Prints one JSON line with the
device name and power limit.

    python tools/lm_stacked_timing.py [--reps 20] [--rounds 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "epro-pnp_b200")]

import torch  # noqa: E402

from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_problem  # noqa: E402

B = 1024
SHAPES = [(512, 2), (512, 8), (512, 32), (4096, 8)]
MODES = {"dof6_lm10": (6, dict(lm_iter=10)), "dof4_gn5_fast": (4, dict(lm_iter=5, fast_mode=1))}


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def replicate(prob, S):
    rep = lambda v: v.unsqueeze(0).expand((S,) + v.shape).reshape((S * v.shape[0],) + v.shape[1:])
    return native.Problem(rep(prob.x3d), rep(prob.x2d), rep(prob.w2d), rep(prob.cam), None, None, rep(prob.delta))


def measure(dof, overrides, N, S, reps, rounds, dev):
    pc = make_problem(B, N, seed=N + S, dof=dof)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          torch.full((B,), 2.0, device=dev))
    pose = pc["pose_init"].to(dev)
    gen = torch.Generator().manual_seed(S)
    starts = pose.unsqueeze(0) + 0.05 * torch.randn((S,) + pose.shape, generator=gen).to(dev)
    p = native.default_params(dof, **overrides)
    flat = replicate(prob, S)
    stacked = lambda: native.lm_solve_stacked(prob, starts, p, want_cost=True)
    flattened = lambda: native.lm_solve(flat, starts.reshape(S * B, -1), p, want_cost=True)
    with_copy = lambda: native.lm_solve(replicate(prob, S), starts.reshape(S * B, -1), p, want_cost=True)
    a, b = stacked(), flattened()
    same = all(torch.equal(a[k].reshape(b[k].shape).view(torch.int32), b[k].view(torch.int32))
               for k in ("pose_opt", "cost"))
    for fn in (stacked, flattened, with_copy):
        fn()
    torch.cuda.synchronize()
    t = {"stacked": [], "flat_solve": [], "flat_with_copy": []}
    for _ in range(rounds):
        for k, fn in zip(t, (stacked, flattened, with_copy)):
            t[k].append(timed(fn, reps))
    ms = {k + "_ms": round(statistics.median(v), 4) for k, v in t.items()}
    spread = {k + "_range_ms": [round(min(v), 4), round(max(v), 4)] for k, v in t.items()}
    return dict(ms, **spread, speedup_vs_flat_solve=round(ms["flat_solve_ms"] / ms["stacked_ms"], 3),
                speedup_vs_flat_with_copy=round(ms["flat_with_copy_ms"] / ms["stacked_ms"], 3), bit_identical=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lm_stacked_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    out = dict(device=q, B=B)
    for name, (dof, overrides) in MODES.items():
        out[name] = {f"N{N}_S{S}": measure(dof, overrides, N, S, a.reps, a.rounds, dev) for N, S in SHAPES}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
