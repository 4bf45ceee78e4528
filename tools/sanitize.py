#!/usr/bin/env python
"""Small driver for compute-sanitizer: one call of every kernel family on tiny problems (6DoF / 4DoF,
TMA and plain loaders, bounded / unbounded, AMIS-only, fused, cost, full evaluate, backward)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
import torch  # noqa: E402
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_problem  # noqa: E402

dev = torch.device("cuda:0")
failed = []


def check(what, ok, detail=""):
    """A failed comparison is reported by name (and the run goes on, so the sanitizer sees every kernel)."""
    if not bool(ok):
        failed.append(what)
        print(f"CHECK FAILED: {what} {detail}", flush=True)


def maxdiff(a, b):
    return f"max |diff| = {(a.double() - b.double()).abs().max().item():.3e}"


for dof, N, B, bounded in ((6, 64, 5, False), (6, 130, 3, True), (6, 51, 4, False), (4, 64, 4, True)):
    pc = make_problem(B, N, seed=dof + N, dof=dof)
    d = {k: v.to(dev) for k, v in pc.items()}
    delta = native.adaptive_delta(d["x2d"], d["w2d"], 0.5)
    lb = ub = None
    if bounded:
        lb = d["x2d"].min(1).values + 5
        ub = d["x2d"].max(1).values - 5
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], lb, ub, delta)
    D = 7 if dof == 6 else 4
    p = native.default_params(dof, mc_samples=128, mc_iter=4)
    lm = native.lm_solve(prob, d["pose_init"], p, want_cov=True, want_cost=True, want_plus=True, want_cost_init=True)
    s, w, _ = native.amis(prob, lm["pose_opt"], lm["pose_cov"], p, seed=1, want_proposals=True)
    out = native.lm_amis_fused(prob, d["pose_init"], p, seed=1, want_cost=True)
    c = native.evaluate_cost(prob, out["pose_samples"].transpose(0, 1).contiguous()[:9], dof, 0.1)
    native.evaluate_full(prob, d["pose_init"], dof, 0.1, 1e-10, True, True, True, True)
    g = native.cost_backward(prob, dof, 0.1, out["pose_samples"], torch.randn(B, 128, device=dev),
                             d["pose_init"].reshape(B, 1, D), torch.randn(B, 1, device=dev))
    if True:
        ep = native.mc_epilogue(out["logw"], out["pose_samples"], out["pose_opt"], cost_target=torch.rand(B, device=dev),
                                want_lse=True, want_loss=True, want_weights=True, want_score=True)
        native.mc_lse_backward(out["logw"], ep["lse"], torch.randn(B, device=dev))
        # push kernel with this device standing in for two "peers" (second copies of the full-batch buffers)
        full_lw = [torch.zeros(B + 3, 128, device=dev) for _ in range(3)]
        full_ps = [torch.zeros(B + 3, D, device=dev) for _ in range(3)]
        native.lm_amis_fused_push(prob, d["pose_init"], p, full_ps[0][2:2 + B], full_lw[0][2:2 + B], full_lw[1:], full_ps[1:],
                                  seed=1, obj_offset=2, want_cost=True, want_cov=True)
        torch.cuda.synchronize()
        tag = f"dof={dof} N={N}"
        check(f"{tag}: peer 1 log-weights == local", torch.equal(full_lw[1][2:2 + B], full_lw[0][2:2 + B]))
        check(f"{tag}: peer 2 poses == local", torch.equal(full_ps[2][2:2 + B], full_ps[0][2:2 + B]))
        same = native.lm_amis_fused(prob, d["pose_init"], p, seed=1, obj_offset=2)          # the Philox stream is keyed by the GLOBAL index
        check(f"{tag}: push kernel == plain kernel", torch.equal(full_lw[0][2:2 + B], same["logw"]), maxdiff(full_lw[0][2:2 + B], same["logw"]))
        check(f"{tag}: rows of other ranks untouched", not full_lw[1][:2].any() and not full_lw[1][2 + B:].any())
        P, n = 5, 6
        inds = torch.stack([torch.stack([torch.randperm(N, device=dev)[:n] for _ in range(B)]) for _ in range(P)])
        native.rslm(prob, inds, d["pose_init"][None].repeat(P, 1, 1), native.default_params(dof, lm_iter=2), want_all=True)
        di, ds = native.rslm_draw(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], 9, n, dof, seed=3)
        check(f"{tag}: drawn subsets in range and distinct",
              di.min() >= 0 and di.max() < N and (di.sort(-1).values[..., 1:] != di.sort(-1).values[..., :-1]).all())
        native.rslm(prob, di, ds, native.default_params(dof, lm_iter=2))
        bounded = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], 0.0, 640.0, prob.delta)
        native.rslm_split(bounded, di, ds, native.default_params(dof, lm_iter=2), want_all=True, cluster_ctas=2)
        native.gn_plus_backward(prob, out["pose_opt"], torch.randn(B, D, device=dev), dof, 0.1, 1e-5, 1e-10)
        gp = torch.randn(B, D, device=dev)
        cam = [native.cost_camera_backward(bounded, dof, 0.1, out["pose_samples"], torch.randn(B, 128, device=dev),
                                           d["pose_init"].reshape(B, 1, D), torch.randn(B, 1, device=dev)),
               native.gn_plus_camera_backward(bounded, out["pose_opt"], gp, dof, 0.1, 1e-5, 1e-10)]
        ev = native.evaluate_backward(bounded, out["pose_samples"][:, :3].transpose(0, 1).contiguous(), dof, 0.1, 1e-10,
                                      True, torch.randn(3, B, 2 * N, device=dev),
                                      torch.randn(3, B, 2 * N, dof, device=dev), torch.randn(3, B, device=dev))
        torch.cuda.synchronize()
        check(f"{tag}: finite camera gradients", all(torch.isfinite(t).all() for g3 in cam for t in g3))
        check(f"{tag}: finite residual / Jacobian gradients", all(torch.isfinite(t).all() for t in ev))
    torch.cuda.synchronize()
    check(f"dof={dof} N={N}: finite log-weights", torch.isfinite(out["logw"]).all())
    check(f"dof={dof} N={N}: finite gradients", all(torch.isfinite(t).all() for t in g))
# objects beyond one SM: the cluster-split camera backwards (distributed shared memory, cluster barriers)
for dof in (6, 4):
    N, B, D = native.max_points(dof) + 1, 2, 7 if dof == 6 else 4
    d = {k: v.to(dev) for k, v in make_problem(B, N, seed=5 + dof, dof=dof, outlier_frac=0.1).items()}
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], d["x2d"].min(1).values + 5,
                          d["x2d"].max(1).values - 5, native.adaptive_delta(d["x2d"], d["w2d"], 0.5))
    poses = d["pose_init"][:, None].repeat(1, 3, 1)
    cam = [native.cost_camera_backward(prob, dof, 0.1, poses, torch.randn(B, 3, device=dev), d["pose_init"][:, None],
                                       torch.randn(B, 1, device=dev), cluster_ctas=ctas) for ctas in (2, 3)]
    cam += [native.gn_plus_camera_backward(prob, d["pose_init"], torch.randn(B, D, device=dev), dof, 0.1, 1e-5, 1e-10,
                                           cluster_ctas=2)]
    torch.cuda.synchronize()
    check(f"dof={dof} N={N}: finite split camera gradients", all(torch.isfinite(t).all() for g3 in cam for t in g3))
# long point set: the 8-warp LM kernel and the 512-thread AMIS kernel
pc = make_problem(2, 2052, seed=3)
d = {k: v.to(dev) for k, v in pc.items()}
prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], None, None, native.adaptive_delta(d["x2d"], d["w2d"], 0.5))
out = native.lm_amis_fused(prob, d["pose_init"], native.default_params(6, lm_iter=3, mc_samples=64, mc_iter=2), seed=1, want_cost=True)
torch.cuda.synchronize()
check("N=2052: finite log-weights", torch.isfinite(out["logw"]).all())
print("sanitize driver finished" + (f" with {len(failed)} failed checks" if failed else ", all checks passed"))
sys.exit(1 if failed else 0)
