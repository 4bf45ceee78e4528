"""Times the host-buffer solve from scratch (epnp_solve_host_f32 / epnp_solve_split_host_f32) on the GPU against doing
the same work without its pipeline, at three shapes:
    det    EPro-PnP-Det inference: 4DoF, N = 256, RSLM (P = 64, n = 16, 3 iterations), LM 5 in fast mode, no AMIS
    6dof   EPro-PnP-6DoF test: dense 64 x 64 maps, EPnP on the 0.8 quantile, GN(3), no AMIS
    split  N = 16 384 on the split form: EPnP, LM 5 + AMIS 512 x 4
Arms, alternated round by round on the current stream, each timed with CUDA events around the whole call:
    host0 / host8   the host call with n_chunks = 0 / 8 (pinned host inputs and outputs)
    serial          copy-in to device tensors, the device composition, copy-out, all on one stream
    device          the device composition alone on device-resident inputs
Every arm's outputs are first checked bit for bit against the device composition.  Prints one JSON line with the card's
name and power limit, medians and min / max in ms.

    python tools/solve_host_timing.py [--rounds 15] [--out /tmp/solve_host_timing.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "epro-pnp_b200"))
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_problem  # noqa: E402

DEV = torch.device("cuda", 0)
SHAPES = {
    "det": dict(B=2047, N=256, dof=4, grid2d=False, init=lambda: native.rslm_spec(4, 16, 64, 3, seed=9, fast_mode=1),
                params=dict(lm_iter=5, fast_mode=1, mc_samples=0), split=False),
    "6dof": dict(B=255, N=4096, dof=6, grid2d=True, init=lambda: native.epnp_spec(0.8),
                 params=dict(lm_iter=3, fast_mode=1, mc_samples=0), split=False),
    "split": dict(B=64, N=16384, dof=6, grid2d=False, init=lambda: native.epnp_spec(0.8),
                  params=dict(lm_iter=5, mc_samples=512, mc_iter=4), split=True),
}
KEYS = ("pose_opt", "pose_cov", "cost", "logw", "pose_samples")


def composition(prob, init, p, split):
    if init.kind == native.capi.INIT_RSLM:
        inds, start = native.rslm_draw(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.num_proposals, init.num_points,
                                       p.dof, eps=init.rslm.eps, seed=init.seed)
        pose0 = (native.rslm_split if split else native.rslm)(prob, inds, start, init.rslm)["pose"]
    else:
        pose0 = (native.epnp_init_split if split else native.epnp_init)(prob.x3d, prob.x2d, prob.w2d, prob.cam,
                                                                         init.conf_quantile)
    if p.mc_samples == 0:
        return native.lm_solve(prob, pose0, p, want_cov=True, want_cost=True)
    fused = native.lm_amis_fused_split if split else native.lm_amis_fused
    return fused(prob, pose0, p, seed=1, want_cost=True, want_cost_init=False)


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_shape(name, cfg, rounds):
    B, N, dof = cfg["B"], cfg["N"], cfg["dof"]
    pc = make_problem(B, N, seed=5, dof=dof, grid2d=cfg["grid2d"])
    delta = native.adaptive_delta(pc["x2d"].to(DEV), pc["w2d"].to(DEV), 0.1)
    host = {k: pc[k].contiguous().pin_memory() for k in ("x3d", "x2d", "w2d", "cam_mats")}
    host["delta"] = delta.cpu().pin_memory()
    init, p = cfg["init"](), native.default_params(dof, **cfg["params"])
    split = cfg["split"]
    call = native.solve_split_host if split else native.solve_host
    ws = torch.empty(native.solve_workspace_bytes(B, N, p, init), dtype=torch.uint8, device=DEV)
    dev_in = {k: torch.empty(v.shape, dtype=v.dtype, device=DEV) for k, v in host.items()}
    for k in dev_in:
        dev_in[k].copy_(host[k])
    prob = native.Problem(dev_in["x3d"], dev_in["x2d"], dev_in["w2d"], dev_in["cam_mats"], None, None, dev_in["delta"])
    ref = composition(prob, init, p, split)
    outs = {}

    def host_arm(n_chunks):
        def run():
            outs[n_chunks] = call(host, p, ws, init=init, n_chunks=n_chunks, seed=1, out=outs.get(n_chunks))
        return run

    pinned_out = {k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True) for k, v in ref.items()
                  if v is not None and k in KEYS}

    def serial():
        for k in dev_in:                                   # one stream: copy-in, the composition, copy-out
            dev_in[k].copy_(host[k], non_blocking=True)
        res = composition(prob, init, p, split)
        for k, t in pinned_out.items():
            t.copy_(res[k], non_blocking=True)

    def device():
        composition(prob, init, p, split)

    arms = dict(host0=host_arm(0), host8=host_arm(8), serial=serial, device=device)
    for fn in arms.values():                               # warm-up, then bit-identity before any timing
        fn()
    torch.cuda.synchronize()
    for n_chunks in (0, 8):
        for k, t in pinned_out.items():
            assert torch.equal(outs[n_chunks][k], ref[k].cpu()), (name, n_chunks, k)
    for k, t in pinned_out.items():
        assert torch.equal(t, ref[k].cpu()), (name, "serial", k)
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times[a].append(e0.elapsed_time(e1))
    stat = lambda v: dict(median=sorted(v)[len(v) // 2], min=min(v), max=max(v))
    return dict(B=B, N=N, dof=dof, init="rslm" if init.kind == native.capi.INIT_RSLM else "epnp",
                mc_samples=p.mc_samples, split=split, ms={a: stat(v) for a, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("solve_host_timing needs a CUDA device")
    res = dict(card=torch.cuda.get_device_name(DEV), power_limit=power_limit(),
               shapes={name: run_shape(name, cfg, args.rounds) for name, cfg in SHAPES.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
