"""Cluster-split Monte-Carlo forward and stacked-pose cost (epnp_lm_amis_fused_split_f32, epnp_evaluate_cost_split_f32):
objects with more points than one SM holds, each spread over a thread-block cluster of 2..8 CTAs.  Against the fp64
oracle, against the resident kernels where both run, for determinism and batch independence, end to end through the
drop-in classes, and for the refusals that remain."""
import numpy as np
import pytest
import torch

from conftest import err_stats, err_vs, record_parity
from epropnp_b200 import native
from epropnp_b200.synth import make_noise, make_problem

pytestmark = pytest.mark.gpu


def _setup(dev, dof, B, N, M, seed, rel=0.1, z_min=0.01):
    dense = dof == 6 and int(round(N ** 0.5)) ** 2 == N          # a coordinate map where N is a square
    pc = make_problem(B, N, seed=seed, dof=dof, grid2d=dense)
    n3, c2, r = make_noise(B, M, seed=seed + 1, dof=dof)
    if dof == 4:                     # injected yaw draws themselves (noise_rot (B, M))
        r = torch.rand(B, M, generator=torch.Generator().manual_seed(seed + 2)) * (2 * np.pi) - np.pi
    noise = (n3, c2, r)
    delta = native.adaptive_delta(pc["x2d"].to(dev), pc["w2d"].to(dev), rel)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None,
                          delta)
    return pc, noise, prob


def _oracle_amis(pc, noise, pose, cov, dof, M, I, dtype, z_min, rel):
    """The oracle's AMIS loop started from the kernel's own LM solution, so an LM flip cannot leak into the comparison."""
    from oracle import pnp_oracle as orc
    t = lambda k: pc[k].to(dtype)
    cam = orc.Camera(t("cam_mats"), z_min)
    delta = orc.adaptive_delta(t("x2d"), t("w2d"), rel)
    B, S = pc["x3d"].shape[0], M // I
    n3, c2, r = noise
    nz = (n3.reshape(B, I, S, 3).permute(1, 2, 0, 3).to(dtype), c2.reshape(B, I, S).permute(1, 2, 0).to(dtype))
    if dof == 6:
        nz += (r.reshape(B, I, S, 4).permute(1, 2, 0, 3).to(dtype),)
        return orc.amis_6dof(t("x3d"), t("x2d"), t("w2d"), cam, delta, pose.to(dtype), cov.to(dtype), nz, M, I)
    nz += (r.reshape(B, I, S).permute(1, 2, 0).to(dtype),)
    return orc.amis_4dof(t("x3d"), t("x2d"), t("w2d"), cam, delta, pose.to(dtype), cov.to(dtype), nz, M, I)


def check_split_against_oracle(dev, dof, B, N, M, I, ctas, seed, k=5, record=None, against_resident=False):
    """Split fused call (cluster_ctas = ctas, 0 = automatic) with injected noise: samples and log-weights within
    DESIGN section 2's bound max(1e-4, k * floor) of the fp64 oracle, floor = what fp32 rounding alone moves the oracle.
    against_resident: the resident kernel on the same inputs must meet the same bound, and both share the LM kernel."""
    z_min, rel = 0.01, 0.1
    pc, noise, prob = _setup(dev, dof, B, N, M, seed, rel, z_min)
    p = native.default_params(dof, lm_iter=3, fast_mode=1, z_min=z_min, mc_samples=M, mc_iter=I)
    nz = tuple(t.to(dev) for t in noise)
    out = native.lm_amis_fused_split(prob, pc["pose_init"].to(dev), p, noise=nz, want_cost=True, cluster_ctas=ctas)
    pose_k, cov_k = out["pose_opt"].cpu(), out["pose_cov"].cpu()
    r64 = _oracle_amis(pc, noise, pose_k, cov_k, dof, M, I, torch.float64, z_min, rel)
    r32 = _oracle_amis(pc, noise, pose_k, cov_k, dof, M, I, torch.float32, z_min, rel)
    floor_w, floor_s = err_vs(r32["logw"], r64["logw"]), err_vs(r32["samples"], r64["samples"])
    runs = [("split", out)]
    if against_resident:
        res = native.lm_amis_fused(prob, pc["pose_init"].to(dev), p, noise=nz, want_cost=True)
        assert torch.equal(res["pose_opt"], out["pose_opt"]) and torch.equal(res["pose_cov"], out["pose_cov"])
        runs.append(("resident", res))
    for what, o in runs:
        lw = o["logw"].transpose(0, 1).cpu().numpy()
        smp = o["pose_samples"].transpose(0, 1).cpu().numpy()
        assert np.isfinite(lw).all(), what
        assert err_vs(smp, r64["samples"]) < max(1e-4, k * floor_s), what
        assert err_vs(lw, r64["logw"]) < max(1e-4, k * floor_w), what
    if record:
        lw = out["logw"].transpose(0, 1).cpu().numpy()
        smp = out["pose_samples"].transpose(0, 1).cpu().numpy()
        record_parity(record, cluster_ctas=ctas or native.split_ctas(dof, N, M, I), logw_vs_f64=err_stats(lw, r64["logw"]),
                      samples_vs_f64=err_stats(smp, r64["samples"]), f32_vs_f64_logw=err_stats(r32["logw"], r64["logw"]))
    return out


def check_cost_split(dev, dof, B, N, S, ctas, seed):
    """evaluate_cost_split against the fp64 oracle, and against the resident cost kernel where N allows it."""
    from oracle import pnp_oracle as orc
    pc, _, prob = _setup(dev, dof, B, N, 8, seed)
    g = torch.Generator().manual_seed(seed)
    poses = pc["pose_init"][None].repeat(S, 1, 1)
    poses[..., :3] += 0.02 * torch.randn(S, B, 3, generator=g)
    if dof == 6:
        poses[..., 3:] = torch.nn.functional.normalize(poses[..., 3:] + 0.05 * torch.randn(S, B, 4, generator=g), dim=-1)
    else:
        poses[..., 3] += 0.1 * torch.randn(S, B, generator=g)
    cost = native.evaluate_cost_split(prob, poses.to(dev), dof, 0.01, cluster_ctas=ctas).cpu()
    d = torch.float64
    cam = orc.Camera(pc["cam_mats"].to(d), 0.01)
    ref = orc.evaluate(pc["x3d"].to(d), pc["x2d"].to(d), pc["w2d"].to(d), poses.to(d), cam,
                       prob.delta.cpu().to(d))["cost"]
    assert err_vs(cost.numpy(), ref.numpy()) < 1e-5
    if N <= native.max_points(dof):
        res = native.evaluate_cost(prob, poses.to(dev), dof, 0.01).cpu()
        assert err_vs(cost.numpy(), res.numpy()) < 1e-5
    return cost


# ------------------------------------------------------------------------------------------------
def test_split_against_oracle_dense_128(cuda_device):
    """out_res = 128: N = 16,384 points per object, beyond what one SM holds; the automatic cluster size."""
    assert 16384 > native.max_points(6, 512, 4) and native.split_ctas(6, 16384, 512, 4) >= 2
    check_split_against_oracle(cuda_device, 6, 4, 16384, 512, 4, 0, seed=3, record="split/6dof_B4_N16384_M512")


def test_split_against_oracle_4dof(cuda_device):
    check_split_against_oracle(cuda_device, 4, 4, 10004, 512, 4, 0, seed=5, record="split/4dof_B4_N10004_M512")


def test_split_c2_against_resident_dense_kernel(cuda_device):
    """At N = 4,096 both forms run: the split one on two CTAs against the resident 512-thread kernel (the same LM
    kernel, so the same solution), both within the oracle bound."""
    check_split_against_oracle(cuda_device, 6, 8, 4096, 512, 4, 2, seed=7, against_resident=True,
                               record="split/6dof_B8_N4096_C2")


@pytest.mark.parametrize("ctas", [0, 8])
def test_split_deterministic_and_batch_independent(cuda_device, ctas):
    """Same seed, same bits; and an object solved alone with its obj_offset equals the same object inside a batch of
    257 (Philox keyed by obj_offset + object; the cluster size depends on N only)."""
    dev, B, N, M, I = cuda_device, 257, 16384, 512, 4
    pc = make_problem(B, N, seed=9, grid2d=True)
    x = {k: v.to(dev) for k, v in pc.items()}
    prob = native.Problem(x["x3d"], x["x2d"], x["w2d"], x["cam_mats"], None, None,
                          native.adaptive_delta(x["x2d"], x["w2d"], 0.1))
    p = native.default_params(6, lm_iter=3, fast_mode=1, z_min=0.01, mc_samples=M, mc_iter=I)
    a = native.lm_amis_fused_split(prob, x["pose_init"], p, seed=11, cluster_ctas=ctas)
    b = native.lm_amis_fused_split(prob, x["pose_init"], p, seed=11, cluster_ctas=ctas)
    for k in ("pose_opt", "pose_samples", "logw"):
        assert torch.equal(a[k], b[k]), k
    assert torch.isfinite(a["logw"]).all()
    for i in (0, 128, 256):
        one = native.Problem(x["x3d"][i:i + 1], x["x2d"][i:i + 1], x["w2d"][i:i + 1], x["cam_mats"][i:i + 1], None, None,
                             prob.delta[i:i + 1])
        o = native.lm_amis_fused_split(one, x["pose_init"][i:i + 1], p, seed=11, obj_offset=i, cluster_ctas=ctas)
        for k in ("pose_opt", "pose_samples", "logw"):
            assert torch.equal(o[k][0], a[k][i]), (i, k)


def test_cost_split_against_resident_and_oracle(cuda_device):
    n_res = native.max_points(6)
    check_cost_split(cuda_device, 6, 3, 4096, 700, 0, seed=13)
    check_cost_split(cuda_device, 6, 3, n_res, 700, 5, seed=14)
    check_cost_split(cuda_device, 4, 3, 4100, 600, 3, seed=15)
    check_cost_split(cuda_device, 6, 2, 16384, 1100, 0, seed=16)


def test_dropin_monte_carlo_forward_and_backward_at_16384(cuda_device):
    """EProPnP6DoF.monte_carlo_forward on 16,384-point objects (pose_init given, force_init_solve=False): finite
    log-weights; the training backward's gradients equal cost_backward applied to the returned samples."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    dev, B, N, M, I = cuda_device, 2, 16384, 512, 4
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=17, grid2d=True).items()}
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    layer = EProPnP6DoF(mc_samples=M, num_iter=I, solver=LMSolver(dof=6, num_iter=3))
    with torch.no_grad():
        pose_opt, _, _, samples, logw, cost_init = layer.monte_carlo_forward(
            pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun, pose_init=pc["pose_init"], force_init_solve=False,
            fast_mode=True, amis_seed=5)
    assert samples.shape == (M, B, 7) and logw.shape == (M, B) and torch.isfinite(logw).all()
    assert torch.isfinite(pose_opt).all() and torch.isfinite(cost_init).all()
    x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
    _, _, _, samples_g, logw_g, cost_init_g = layer.monte_carlo_forward(
        x3d, x2d, w2d, camera, cost_fun, pose_init=pc["pose_init"], force_init_solve=False, fast_mode=True, amis_seed=5)
    assert torch.equal(logw_g.detach(), logw) and torch.equal(samples_g, samples)
    loss = torch.logsumexp(logw_g, dim=0).sum() + cost_init_g.sum()
    gx3d, gx2d, gw2d = torch.autograd.grad(loss, [x3d, x2d, w2d])
    g_logw = torch.softmax(logw, dim=0).transpose(0, 1).contiguous()
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, cost_fun.delta)
    ref = native.cost_backward(prob, 6, 0.01, samples.transpose(0, 1).contiguous(), -g_logw,
                               pc["pose_init"].reshape(B, 1, 7), torch.ones(B, 1, device=dev), want=(True, True, True, False))
    for a, b in zip((gx3d, gx2d, gw2d), ref[:3]):
        assert torch.isfinite(a).all() and err_vs(a.cpu(), b.cpu()) < 1e-6
    # evaluate_pnp(out_cost=True) at this N takes the split cost kernel, with and without autograd
    # (the no-grad forward's cost_init comes from the LM kernel, the training forward's from the split cost kernel)
    c = evaluate_pnp(pc["x3d"], pc["x2d"], pc["w2d"], pc["pose_init"], camera, cost_fun, out_cost=True)[1]
    assert torch.equal(c, cost_init_g.detach()) and err_vs(c.cpu(), cost_init.cpu()) < 1e-5
    cg = evaluate_pnp(x3d, x2d, w2d, pc["pose_init"], camera, cost_fun, out_cost=True)[1]
    assert torch.equal(cg.detach(), c)


def test_refusals(cuda_device):
    """Above epnp_max_points_split the split calls refuse; below it the flows the split path does not cover (RSLM init,
    the resident entry points) keep their shared-memory refusal; a cluster size outside [minimum, 8] is a bad argument."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
    dev = cuda_device
    p = native.default_params(6, lm_iter=3, fast_mode=1, mc_samples=512, mc_iter=4)

    def prob_of(N, B=1):
        z = lambda *s: torch.zeros(*s, device=dev)
        return native.Problem(z(B, N, 3), z(B, N, 2), z(B, N, 2), torch.eye(3, device=dev)[None].repeat(B, 1, 1), None,
                              None, 1.0), z(B, 7)
    big, pose = prob_of(native.max_points_split(6, 512, 4) + 64)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.lm_amis_fused_split(big, pose, p)
    big_c, _ = prob_of(native.max_points_split(6) + 64)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.evaluate_cost_split(big_c, pose[None], 6, 0.1)
    mid, pose = prob_of(16384)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.lm_amis_fused(mid, pose, p)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.evaluate_cost(mid, pose[None], 6, 0.1)
    for bad in (1, 9):
        with pytest.raises(native.NativeError, match="bad argument"):
            native.lm_amis_fused_split(mid, pose, p, cluster_ctas=bad)
    pc = {k: v.to(dev) for k, v in make_problem(1, 16384, seed=19, grid2d=True).items()}
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    layer = EProPnP6DoF(mc_samples=512, num_iter=4, solver=LMSolver(dof=6, num_iter=3, init_solver=RSLMSolver(dof=6)))
    with pytest.raises(native.NativeError, match="shared memory"):
        layer.monte_carlo_forward(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun)
