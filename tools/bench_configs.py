#!/usr/bin/env python
"""Device-timed throughput of the BASELINE.json configs that are not the headline bench line
(parity-test shapes, measured for the record):  #2 LM-only, #3 LM+AMIS at B=1024, #4 dense N=4096."""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
import torch  # noqa: E402
from epropnp_b200 import native  # noqa: E402
from epropnp_b200.synth import make_problem  # noqa: E402


# EPNP_BENCH_CONFIGS_TOY=1 shrinks every size (tests/test_bench_dryrun_cpu.py drives this script on the SIMT-emulated
# library to check that it runs; the numbers mean nothing then)
TOY = os.environ.get("EPNP_BENCH_CONFIGS_TOY") == "1"


def b(x):       # objects
    return max(2, x // 512) if TOY else x


def bs(*xs):
    return tuple(sorted({b(x) for x in xs}))


def n(x):       # correspondences per object
    return max(9, x // 32) if TOY else x


def m(x):       # Monte-Carlo samples / stacked poses
    return 8 if TOY else x


def timed(fn, iters=20, warm=3):
    if TOY:
        iters, warm = 1, 1
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev)


def main():
    dev = torch.device(os.environ.get("EPNP_BENCH_DEVICE", "cuda"), 0)
    out = []

    def setup(B, N, rel, **kw):
        pc = make_problem(B, N, seed=11, **kw)
        d = {k: v.to(dev) for k, v in pc.items()}
        delta = native.adaptive_delta(d["x2d"], d["w2d"], rel)
        return native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], None, None, delta), d["pose_init"]

    for B in bs(1024, 4096, 16384):
        prob, p0 = setup(B, n(512), 0.5)
        p = native.default_params(6, lm_iter=10)
        ms = timed(lambda: native.lm_solve(prob, p0, p, want_cov=True, want_cost=True))
        out.append(dict(config="#2 LM(10) only, N=512", B=B, ms=ms, objects_per_s=B / ms * 1e3,
                        hbm_gbs=B * 14580 / ms / 1e6))
    for B in bs(1024, 4096):
        prob, p0 = setup(B, n(512), 0.5)
        p = native.default_params(6, lm_iter=10, mc_samples=m(512), mc_iter=2 if TOY else 4)
        ms = timed(lambda: native.lm_amis_fused(prob, p0, p, seed=1))
        out.append(dict(config="#3 LM(10)+AMIS(4x128), N=512", B=B, ms=ms, objects_per_s=B / ms * 1e3,
                        hbm_gbs=B * 30964 / ms / 1e6))
    for B in bs(256, 1024):
        prob, p0 = setup(B, 16 if TOY else 4096, 0.1, grid2d=True)
        p = native.default_params(6, lm_iter=3, fast_mode=1, z_min=0.01, mc_samples=m(512), mc_iter=2 if TOY else 4)
        ms = timed(lambda: native.lm_amis_fused(prob, p0, p, seed=1), iters=10)
        out.append(dict(config="#4 dense GN(3)+AMIS(4x128), N=4096", B=B, ms=ms, objects_per_s=B / ms * 1e3,
                        hbm_gbs=B * 131316 / ms / 1e6))
        ms = timed(lambda: native.lm_solve(prob, p0, p, want_cov=True), iters=10)
        out.append(dict(config="#4 dense GN(3) only (test-time path, lib/test.py:209-211), N=4096", B=B, ms=ms,
                        objects_per_s=B / ms * 1e3, hbm_gbs=B * 114932 / ms / 1e6))
    # detection variant (EPro-PnP-Det/configs/epropnp_det_basic.py:98-111): EProPnP4DoF, 8 heads x 32 points = 256
    # correspondences per object, LM(10) + AMIS(4x128), in-kernel von Mises / uniform yaw sampler
    for B in bs(1024, 4096):
        prob, p0 = setup(B, n(256), 0.5, dof=4)
        p = native.default_params(4, lm_iter=10, mc_samples=m(512), mc_iter=2 if TOY else 4)
        ms = timed(lambda: native.lm_amis_fused(prob, p0, p, seed=1))
        out.append(dict(config="Det: EProPnP4DoF LM(10)+AMIS(4x128), N=256", B=B, ms=ms, objects_per_s=B / ms * 1e3,
                        hbm_gbs=B * (28 * 256 + 36 + 4 + 16 + 16 + 64 + 4 + 20 * 512) / ms / 1e6))
    # training step: fused forward + native Monte-Carlo cost backward (513 poses per object)
    for B in bs(1024, 4096):
        prob, p0 = setup(B, n(512), 0.5)
        p = native.default_params(6, lm_iter=10, mc_samples=m(512), mc_iter=2 if TOY else 4)
        fw = native.lm_amis_fused(prob, p0, p, seed=1, want_cov=False)
        gl = torch.randn(B, m(512), device=dev)
        gc = torch.randn(B, 1, device=dev)
        ms_b = timed(lambda: native.cost_backward(prob, 6, 0.1, fw["pose_samples"], gl, p0.reshape(B, 1, 7), gc))
        ms_f = timed(lambda: native.lm_amis_fused(prob, p0, p, seed=1, want_cov=False))
        out.append(dict(config="training step: fused forward + MC-cost backward, N=512, M=512", B=B, ms_forward=ms_f,
                        ms_backward=ms_b, objects_per_s=B / (ms_f + ms_b) * 1e3,
                        backward_pose_point_pairs_per_s=B * 513 * 512 / ms_b * 1e3))
    S = m(128)
    prob, p0 = setup(b(4096), n(512), 0.5)
    poses = p0[None].repeat(S, 1, 1).contiguous()
    ms = timed(lambda: native.evaluate_cost(prob, poses, 6, 0.1))
    out.append(dict(config="evaluate_pnp cost, 128 poses x 4096 objects x 512 pts", B=4096, ms=ms,
                    pose_point_pairs_per_s=S * 4096 * 512 / ms * 1e3))
    # random-sample LM initialiser (RSLMSolver.solve = centre-based translation in torch + epnp_rslm_draw_f32 +
    # epnp_rslm_f32), demo-notebook and detection configurations; draws='torch' = the reference's torch.multinomial / randn.  (The reference's own formulation -- gather + P*B tiny
    # solves + stacked evaluate_pnp -- on the same kernels measured slower and is gone.)
    if os.environ.get("EPNP_BENCH_RSLM"):
        sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
        from epropnp.camera import PerspectiveCamera
        from epropnp.cost_fun import AdaptiveHuberPnPCost
        from epropnp.levenberg_marquardt import RSLMSolver
        for dof, B, N, npts, P, K in ((6, b(256), 64, 8, 128, 5), (4, b(512), 64, 16, 64, 3), (6, b(4096), n(512), 16, 64, 3),
                                      (6, b(4096), n(512), 8, 128, 3)):
            P = max(2, P // 32) if TOY else P
            pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=3, dof=dof).items()}
            camera = PerspectiveCamera(cam_mats=pc["cam_mats"])
            cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
            cost_fun.set_param(pc["x2d"], pc["w2d"])
            solver = RSLMSolver(dof=dof, num_points=npts, num_proposals=P, num_iter=K)
            row = dict(config=f"RSLM init, dof={dof}, N={N}, {P} proposals x {npts} points x LM({K})", B=B)
            # the draws alone (torch.multinomial on P*B rows of N weights + the start orientations): torch work of the
            # reference's own algorithm (levenberg_marquardt.py:306-324) that both paths share
            rows = pc["w2d"].mean(dim=-1).unsqueeze(0).expand(P, B, N).reshape(P * B, N)
            row["ms_setup_torch"] = timed(lambda: (torch.multinomial(rows, npts), solver._starting_hypotheses(pc["x3d"], pc["x2d"], camera)), iters=10)
            row["ms_setup_native"] = timed(lambda: native.rslm_draw(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], P, npts, dof, seed=1), iters=10)
            row["ms_solve"] = timed(lambda: solver.solve(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun), iters=10)
            solver_t = RSLMSolver(dof=dof, num_points=npts, num_proposals=P, num_iter=K, draws="torch")
            row["ms_solve_torch_draws"] = timed(lambda: solver_t.solve(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun), iters=10)
            inds = torch.multinomial(rows, npts).reshape(P, B, npts)
            start = solver._starting_hypotheses(pc["x3d"], pc["x2d"], camera)
            prob_r = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], camera.cam_mats, camera.lb, camera.ub, cost_fun.delta)
            par_r = solver.native_params(camera, cost_fun, False)
            row["ms_kernel"] = timed(lambda: native.rslm(prob_r, inds, start, par_r), iters=10)
            row["hypotheses_per_s"] = P * B / row["ms_kernel"] * 1e3
            out.append(row)
    # derivative-regularisation branch: pose_opt_plus forward + backward, torch composite vs native kernel
    if os.environ.get("EPNP_BENCH_GN_PLUS"):
        sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
        from epropnp import autograd as ag
        from epropnp.camera import PerspectiveCamera
        from epropnp.cost_fun import AdaptiveHuberPnPCost
        from epropnp.levenberg_marquardt import LMSolver
        for B in bs(1024, 4096):
            pc = {k: v.to(dev) for k, v in make_problem(B, n(512), seed=5).items()}
            x3d, w2d = pc["x3d"].clone().requires_grad_(True), pc["w2d"].clone().requires_grad_(True)
            camera = PerspectiveCamera(cam_mats=pc["cam_mats"])
            cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
            solver = LMSolver(dof=6, num_iter=10)
            row = dict(config="pose_opt_plus forward + backward (derivative regularisation), N=512", B=B)

            def step():
                x3d.grad = w2d.grad = None
                cost_fun.set_param(pc["x2d"], w2d)        # delta depends on w2d: part of every training step's graph
                ag.pose_plus_autograd(solver, x3d, pc["x2d"], w2d, pc["pose_init"], camera, cost_fun).square().sum().backward()
            for flag, key in (("0", "ms_composite"), ("1", "ms_native")):
                os.environ["EPNP_NATIVE_GN_STEP"] = flag
                row[key] = timed(step, iters=10)
            os.environ["EPNP_NATIVE_GN_STEP"] = "1"
            out.append(row)
    # the step after the path: Monte-Carlo pose loss forward + backward and the Det MC score, torch composite on the
    # layer's (M, B) views vs the native one-pass epilogue
    if os.environ.get("EPNP_BENCH_MC_EPILOGUE"):
        sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
        from epropnp import monte_carlo_pose_loss as mcl
        for B, D in ((b(4096), 7), (b(4096), 4)):
            logw = (torch.randn(B, m(512), device=dev) * 3).transpose(0, 1).requires_grad_(True)
            samples = torch.randn(B, m(512), D, device=dev).transpose(0, 1)
            opt, ct = torch.randn(B, D, device=dev), torch.rand(B, device=dev)
            loss_fn = mcl.MonteCarloPoseLoss().to(dev).eval()
            row = dict(config=f"MC pose loss fwd+bwd and MC te-score on (512, {B}) log-weights, D={D}", B=B,
                       bytes_min=B * 512 * 4 * 3 + B * 512 * D * 4)

            def step():
                logw.grad = None
                loss_fn(logw, ct, 1.0).backward()
                mcl.mc_score_te(samples, opt, logw.detach())
            for flag, key in (("0", "ms_composite"), ("1", "ms_native")):
                os.environ["EPNP_NATIVE_MC_EPILOGUE"] = flag
                row[key] = timed(step, iters=20)
            os.environ["EPNP_NATIVE_MC_EPILOGUE"] = "1"
            out.append(row)
    # the 6DoF test-time path (EPro-PnP-6DoF/lib/test.py:178-211): EPnP on the 20 % most confident points, then GN(3);
    # host_cv2_ms is the reference's own per-object loop on the same objects (device -> host copy, np.quantile mask,
    # cv2 EPnP, scipy quaternion, host -> device copy), where OpenCV is installed
    if os.environ.get("EPNP_BENCH_EPNP"):
        sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
        from epropnp.camera import PerspectiveCamera
        from epropnp.cost_fun import AdaptiveHuberPnPCost
        from epropnp.epnp import EPnPSolver
        from epropnp.levenberg_marquardt import LMSolver
        card = dict(card=torch.cuda.get_device_name(dev), power_limit_w=power_limit(dev)) if dev.type == "cuda" else {}
        N = 16 if TOY else 4096
        for B in bs(256, 1024):
            pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=13, grid2d=True).items()}
            camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.01)
            cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
            cost_fun.set_param(pc["x2d"], pc["w2d"])
            solver = LMSolver(dof=6, num_iter=3, init_solver=EPnPSolver(conf_quantile=0.8))
            row = dict(config=f"6DoF test-time path: EPnP init (q=0.8) + GN(3), N={N}", B=B, **card)
            row["ms_epnp"] = timed(lambda: native.epnp_init(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], 0.8), iters=10)
            row["ms_epnp_gn3"] = timed(lambda: solver.solve(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun,
                                                            fast_mode=True), iters=10)
            host = host_cv2_epnp_ms(pc, 0.8)
            if host is not None:
                row["host_cv2_ms"] = host
            out.append(row)
    # objects larger than one SM holds: the cluster-split fused call at out_res = 128 (N = 16,384), and at N = 4,096 the
    # split form on two CTAs next to the resident 512-thread kernel on the same inputs (the DSMEM experiment of DESIGN
    # section 9.2: one object on two SMs against one object per SM)
    if os.environ.get("EPNP_BENCH_SPLIT"):
        card = dict(card=torch.cuda.get_device_name(dev), power_limit_w=power_limit(dev)) if dev.type == "cuda" else {}
        B = b(256)
        for N, ctas in ((16 if TOY else 16384, 0), (16 if TOY else 4096, 2)):
            prob, p0 = setup(B, N, 0.1, grid2d=True)
            p = native.default_params(6, lm_iter=3, fast_mode=1, z_min=0.01, mc_samples=m(512), mc_iter=2 if TOY else 4)
            c = ctas or native.split_ctas(6, N, p.mc_samples, p.mc_iter)
            row = dict(config=f"dense GN(3)+AMIS(4x128), N={N}, cluster-split", B=B, cluster_ctas=c, **card)
            row["ms_split"] = timed(lambda: native.lm_amis_fused_split(prob, p0, p, seed=1, cluster_ctas=ctas), iters=10)
            if N <= native.max_points(6, p.mc_samples, p.mc_iter):
                row["ms_resident"] = timed(lambda: native.lm_amis_fused(prob, p0, p, seed=1), iters=10)
            row["ms_lm_only"] = timed(lambda: native.lm_solve(prob, p0, p, want_cov=True), iters=10)
            row["objects_per_s_split"] = B / row["ms_split"] * 1e3
            out.append(row)
    for r in out:
        print(json.dumps(r))


def power_limit(dev):
    """The card's power limit in W (read-only nvidia-smi query), None when it cannot be read."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def host_cv2_epnp_ms(pc, q, reps=3):
    """Wall time of the reference's per-object EPnP loop (lib/test.py:178-194) on the objects of `pc`, None without
    OpenCV."""
    try:
        import cv2
        import numpy as np
        from scipy.spatial.transform import Rotation
    except ImportError:
        return None
    import time
    dev = pc["x3d"].device

    def loop():
        x3d, x2d, w2d, K = (pc[k].cpu().numpy() for k in ("x3d", "x2d", "w2d", "cam_mats"))
        pose = np.empty((x3d.shape[0], 7), np.float32)
        for b in range(x3d.shape[0]):
            conf = w2d[b].mean(-1)
            m = conf >= np.quantile(conf, q)
            _, rvec, tvec = cv2.solvePnP(x3d[b][m], x2d[b][m], K[b], None, flags=cv2.SOLVEPNP_EPNP)
            pose[b, :3] = tvec[:, 0]
            pose[b, 3:] = Rotation.from_rotvec(rvec[:, 0]).as_quat()[[3, 0, 1, 2]]
        return torch.from_numpy(pose).to(dev)
    ts = []
    for _ in range(reps):
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        loop()
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


if __name__ == "__main__":
    main()
