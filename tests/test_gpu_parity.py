"""GPU parity tests: the sm_90a kernels, called through the C ABI (epropnp_b200.native -> ctypes),
against (1) golden vectors produced by the unmodified reference, (2) the CPU oracle on seeded inputs at
sizes it finishes in seconds, and (3) size-independent properties at BASELINE.json's full size.

Tolerances.  BASELINE.json asks for <= 1e-4 rel in fp32.  "rel" is measured against the scale of the
tensor: err = max|a - b| / max|b|  (conftest.err_vs).  The reference itself, re-run with different
rounding (its own fp64 run with the identical noise), moves by `floor` = err(ref32, ref64); no fp32
implementation can be closer to ref32 than that, so every bound below is max(1e-4, k * floor) with k
stated at the assert.  At the north-star size (N = 512) floor < 1e-4 and the plain 1e-4 bound applies.
"""
import numpy as np
import pytest
import torch

from conftest import assert_lm_parity, err_stats, err_vs, golden_bounds, golden_names, load_golden, record_parity
from epropnp_b200 import native
from epropnp_b200.synth import make_noise, make_problem

pytestmark = pytest.mark.gpu


def _params(g, **kw):
    return native.default_params(int(g["dof"]), lm_iter=int(g["lm_iter"]), fast_mode=int(g["fast_mode"]),
                                 z_min=float(g["z_min"]), **kw)


def _problem(g, dev):
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    lb, ub = golden_bounds(g)
    if torch.is_tensor(lb):
        lb, ub = lb.to(dev), ub.to(dev)
    return native.Problem(t("x3d"), t("x2d"), t("w2d"), t("cam_mats"), lb, ub, t("delta")), t("pose_init")


def _noise(g, dev):
    B = int(g["B"])
    n3 = torch.from_numpy(np.transpose(g["noise_normal"], (2, 0, 1, 3)).reshape(B, -1, 3).copy()).to(dev)
    c2 = torch.from_numpy(np.transpose(g["noise_chi2"], (2, 0, 1)).reshape(B, -1).copy()).to(dev)
    n4 = torch.from_numpy(np.transpose(g["noise_rot"], (2, 0, 1, 3)).reshape(B, -1, 4).copy()).to(dev)
    return n3, c2, n4


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", golden_names())
def test_golden_evaluate(cuda_device, name):
    g = load_golden(name)
    prob, pose0 = _problem(g, cuda_device)
    dof = int(g["dof"])
    if float(g["fixed_delta"]) < 0:
        d = native.adaptive_delta(prob.x2d, prob.w2d, float(g["relative_delta"]))
        assert err_vs(d.cpu().numpy(), g["delta"]) < 1e-5
    poses = torch.from_numpy(g["eval_poses"]).to(cuda_device)
    cost = native.evaluate_cost(prob, poses, dof, float(g["z_min"]))
    assert err_vs(cost.cpu().numpy(), g["ref64_eval_cost_multi"]) < 2e-5
    res, c, jac = native.evaluate_full(prob, pose0, dof, float(g["z_min"]), 1e-10, not bool(g["fast_mode"]),
                                       True, True, True)
    assert err_vs(res.cpu().numpy(), g["ref64_eval_residual"]) < 2e-4
    assert err_vs(jac.cpu().numpy(), g["ref64_eval_jac"]) < 2e-5
    assert err_vs(c.cpu().numpy(), g["ref64_eval_cost"]) < 2e-5


@pytest.mark.parametrize("name", golden_names())
def test_golden_lm_solve(cuda_device, name):
    g = load_golden(name)
    prob, pose0 = _problem(g, cuda_device)
    out = native.lm_solve(prob, pose0, _params(g), want_cov=True, want_cost=True, want_plus=True, want_cost_init=True)
    floor = err_vs(g["ref32_lm_pose"], g["ref64_lm_pose"])
    tol = max(1e-4, 3 * floor)                                             # k = 3
    pose, cst = out["pose_opt"].cpu().numpy(), out["cost"].cpu().numpy()
    assert_lm_parity(pose, cst, g["ref32_lm_pose"], g["ref64_lm_cost"], tol, what=name + " vs ref32")
    assert_lm_parity(pose, cst, g["ref64_lm_pose"], g["ref64_lm_cost"], tol, what=name + " vs ref64")
    assert_lm_parity(out["pose_opt_plus"].cpu().numpy(), cst, g["ref64_lm_pose_plus"], g["ref64_lm_cost"], tol,
                     what=name + " pose_plus")
    assert err_vs(out["cost"].cpu().numpy(), g["ref64_lm_cost"]) < max(1e-4, 3 * err_vs(g["ref32_lm_cost"], g["ref64_lm_cost"]))
    assert err_vs(out["pose_cov"].cpu().numpy(), g["ref64_lm_cov"]) < max(2e-3, 3 * err_vs(g["ref32_lm_cov"], g["ref64_lm_cov"]))
    assert err_vs(out["cost_init"].cpu().numpy(), g["ref64_eval_cost"]) < 2e-5
    record_parity(f"lm/{name}", pose_vs_ref64=err_stats(pose, g["ref64_lm_pose"]), pose_vs_ref32=err_stats(pose, g["ref32_lm_pose"]),
                  cost_vs_ref64=err_stats(cst, g["ref64_lm_cost"]), cov_vs_ref64=err_stats(out["pose_cov"].cpu().numpy(), g["ref64_lm_cov"]),
                  ref32_vs_ref64_pose_rel=floor)


def _check_amis(samples, logw, props, g, record=None):
    smp = samples.transpose(0, 1).cpu().numpy()
    lw = logw.transpose(0, 1).cpu().numpy()
    assert np.isfinite(lw).all()
    floor_s = err_vs(g["ref32_mc_samples"], g["ref64_mc_samples"])
    floor_w = err_vs(g["ref32_mc_logw"], g["ref64_mc_logw"])
    # max-norm is dominated by a few heavy-tail (Student-t) samples: k = 5; bulk quantiles: k = 3
    for ref in ("ref32", "ref64"):
        assert err_vs(smp, g[ref + "_mc_samples"]) < max(1e-4, 5 * floor_s)
        assert err_vs(lw, g[ref + "_mc_logw"]) < max(1e-4, 5 * floor_w)
    mine = np.abs(lw - g["ref64_mc_logw"])
    ref = np.abs(g["ref32_mc_logw"] - g["ref64_mc_logw"])
    for q in (50, 99):
        assert np.percentile(mine, q) < 3 * np.percentile(ref, q) + 1e-5
    if record:
        record_parity(record, samples_vs_ref64=err_stats(smp, g["ref64_mc_samples"]), logw_vs_ref64=err_stats(lw, g["ref64_mc_logw"]),
                      logw_vs_ref32=err_stats(lw, g["ref32_mc_logw"]), ref32_vs_ref64_logw=err_stats(g["ref32_mc_logw"], g["ref64_mc_logw"]),
                      ref32_vs_ref64_samples_rel=floor_s)
    if props is not None:
        p = props.cpu().numpy()
        assert err_vs(np.transpose(p[:, :, :3], (1, 0, 2)), g["ref64_mc_trans_mode"]) < 1e-4
        ref_lr = g["ref64_mc_rot_cov_tril"]
        rp = np.stack([ref_lr[..., i, j] for i in range(4) for j in range(i + 1)], -1)
        fr = err_vs(g["ref32_mc_rot_cov_tril"], ref_lr)
        assert err_vs(np.transpose(p[:, :, 9:], (1, 0, 2)), rp) < max(1e-3, 3 * fr)


@pytest.mark.parametrize("name", golden_names("mc6"))
def test_golden_amis_from_reference_solution(cuda_device, name):
    """AMIS kernel alone, started from the reference's own LM pose / covariance, identical base noise."""
    g = load_golden(name)
    prob, _ = _problem(g, cuda_device)
    p = _params(g, mc_samples=int(g["mc_samples_total"]), mc_iter=int(g["mc_iters"]))
    pose = torch.from_numpy(g["ref32_lm_pose"]).to(cuda_device)
    cov = torch.from_numpy(g["ref32_lm_cov"]).to(cuda_device)
    samples, logw, props = native.amis(prob, pose, cov, p, noise=_noise(g, cuda_device), want_proposals=True)
    _check_amis(samples, logw, props, g)


@pytest.mark.parametrize("name", golden_names("mc6"))
def test_golden_fused_lm_amis(cuda_device, name):
    """The fused kernel (= monte_carlo_forward with pose_init, force_init_solve=False)."""
    g = load_golden(name)
    prob, pose0 = _problem(g, cuda_device)
    p = _params(g, mc_samples=int(g["mc_samples_total"]), mc_iter=int(g["mc_iters"]))
    out = native.lm_amis_fused(prob, pose0, p, noise=_noise(g, cuda_device), want_cost=True, want_proposals=True)
    floor = err_vs(g["ref32_mc_pose"], g["ref64_mc_pose"])
    assert err_vs(out["pose_opt"].cpu().numpy(), g["ref64_mc_pose"]) < max(1e-4, 3 * floor)
    assert err_vs(out["cost_init"].cpu().numpy(), g["ref64_mc_cost_init"]) < 2e-5
    assert err_vs(out["cost"].cpu().numpy(), g["ref64_mc_cost"]) < 1e-4
    _check_amis(out["pose_samples"], out["logw"], out["proposals"], g, record=f"fused/{name}")
    record_parity(f"fused/{name}", pose_vs_ref64=err_stats(out["pose_opt"].cpu().numpy(), g["ref64_mc_pose"]))
    # fused == LM kernel followed by AMIS kernel, bit for bit
    lm = native.lm_solve(prob, pose0, p, want_cov=True)
    assert torch.equal(lm["pose_opt"], out["pose_opt"]) and torch.equal(lm["pose_cov"], out["pose_cov"])
    s2, w2, _ = native.amis(prob, lm["pose_opt"], lm["pose_cov"], p, noise=_noise(g, cuda_device))
    assert torch.equal(s2, out["pose_samples"]) and torch.equal(w2, out["logw"])


def test_golden_fused_lm_amis_4dof(cuda_device):
    """EProPnP4DoF path: LM + AMIS with the von Mises / uniform yaw proposal, the reference's own yaw draws and
    Student-t base noise injected (golden from the unmodified reference, fp32 run)."""
    g = load_golden("mc4_basic")
    prob, pose0 = _problem(g, cuda_device)
    B, M, I = int(g["B"]), int(g["mc_samples_total"]), int(g["mc_iters"])
    p = _params(g, mc_samples=M, mc_iter=I)
    dev = cuda_device
    noise = (torch.from_numpy(np.transpose(g["noise_normal"], (2, 0, 1, 3)).reshape(B, -1, 3).copy()).to(dev),
             torch.from_numpy(np.transpose(g["noise_chi2"], (2, 0, 1)).reshape(B, -1).copy()).to(dev),
             torch.from_numpy(np.transpose(g["yaw_samples"], (2, 0, 1)).reshape(B, -1).copy()).to(dev))
    out = native.lm_amis_fused(prob, pose0, p, noise=noise, want_cost=True, want_proposals=True)
    floor_w = err_vs(g["ref32_mc_logw"], g["ref64_mc_logw"])
    lw = out["logw"].transpose(0, 1).cpu().numpy()
    smp = out["pose_samples"].transpose(0, 1).cpu().numpy()
    assert smp.shape == (M, B, 4) and np.isfinite(lw).all()
    assert_lm_parity(out["pose_opt"].cpu().numpy(), out["cost"].cpu().numpy(), g["ref32_mc_pose"], g["ref64_mc_cost"],
                     max(1e-4, 3 * err_vs(g["ref32_mc_pose"], g["ref64_mc_pose"])), what="mc4 pose")
    assert err_vs(smp, g["ref32_mc_samples"]) < 1e-4
    assert err_vs(lw, g["ref32_mc_logw"]) < max(1e-4, 5 * floor_w)
    pr = out["proposals"].cpu().numpy()
    assert err_vs(pr[:, :, 9].T, g["ref32_mc_rot_mode"][..., 0]) < 1e-4
    assert err_vs(pr[:, :, 10].T, g["ref32_mc_rot_kappa"][..., 0]) < 2e-3
    # production sampler (Philox + Best-Fisher): deterministic per seed, healthy weights, yaw on the circle
    a = native.lm_amis_fused(prob, pose0, p, seed=3)
    b = native.lm_amis_fused(prob, pose0, p, seed=3)
    assert torch.equal(a["logw"], b["logw"]) and torch.isfinite(a["logw"]).all()
    assert a["pose_samples"][..., 3].abs().max() <= np.pi + 1e-5
    ess = 1.0 / (torch.softmax(a["logw"], 1) ** 2).sum(1)
    assert ess.min() > 8
    ev = lambda r: torch.logsumexp(r["logw"], dim=1) - np.log(M)
    assert (ev(a) - ev(out)).abs().max() < 0.5           # same evidence estimate within Monte-Carlo error


# ------------------------------------------------------------------------------------------------ oracle
def _oracle_run(prob_cpu, noise_cpu, M, I, dtype, lm_iter=10):
    from oracle import pnp_oracle as orc
    t = lambda k: prob_cpu[k].to(dtype)
    cam = orc.Camera(t("cam_mats"), 0.1)
    delta = orc.adaptive_delta(t("x2d"), t("w2d"), 0.5)
    B = prob_cpu["x3d"].shape[0]
    S = M // I
    n3, c2, n4 = noise_cpu
    nz = (n3.reshape(B, I, S, 3).permute(1, 2, 0, 3).to(dtype), c2.reshape(B, I, S).permute(1, 2, 0).to(dtype),
          n4.reshape(B, I, S, 4).permute(1, 2, 0, 3).to(dtype))
    return orc.monte_carlo_forward_6dof(t("x3d"), t("x2d"), t("w2d"), cam, delta, t("pose_init"), nz, M, I,
                                        orc.LMParams(num_iter=lm_iter))


@pytest.mark.parametrize("B,N,M,I", [(48, 512, 512, 4), (7, 100, 128, 2), (5, 1024, 64, 1)])
def test_fused_against_oracle_north_star_shape(cuda_device, B, N, M, I):
    """Seeded synthetic batch at the north-star shape (N=512, M=512), oracle in fp64 and fp32 on CPU."""
    pc = make_problem(B, N, seed=100 + B)
    noise = make_noise(B, M, seed=200 + B)
    r64 = _oracle_run(pc, noise, M, I, torch.float64)
    r32 = _oracle_run(pc, noise, M, I, torch.float32)
    dev = cuda_device
    delta = native.adaptive_delta(pc["x2d"].to(dev), pc["w2d"].to(dev), 0.5)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None, delta)
    p = native.default_params(6, mc_samples=M, mc_iter=I)
    out = native.lm_amis_fused(prob, pc["pose_init"].to(dev), p, noise=tuple(t.to(dev) for t in noise), want_cost=True)
    pose = out["pose_opt"].cpu().numpy()
    lw = out["logw"].transpose(0, 1).cpu().numpy()
    smp = out["pose_samples"].transpose(0, 1).cpu().numpy()
    floor_p = err_vs(r32["pose_opt"], r64["pose_opt"])
    floor_w = err_vs(r32["logw"], r64["logw"])
    floor_s = err_vs(r32["samples"], r64["samples"])
    flips = assert_lm_parity(pose, out["cost"].cpu().numpy(), r64["pose_opt"].numpy(), r64["lm_cost"].numpy(),
                             max(1e-4, 3 * floor_p), max_flip_frac=0.05, what="oracle shape")
    assert flips == 0.0 or N < 512
    assert err_vs(smp, r64["samples"]) < max(1e-4, 5 * floor_s)
    assert err_vs(lw, r64["logw"]) < max(1e-4, 5 * floor_w)
    if N >= 512 and M == 512:
        # the north-star statement itself: <= 1e-4 rel, poses and log-weights, vs the fp32 layer
        assert err_vs(pose, r32["pose_opt"]) < 1e-4
        assert err_vs(lw, r32["logw"]) < 1e-4 + 2 * floor_w
    mine = np.abs(lw - r64["logw"].numpy())
    ref = np.abs(r32["logw"].numpy() - r64["logw"].numpy())
    assert np.median(mine) < 3 * np.median(ref) + 1e-5
    record_parity(f"oracle/B{B}_N{N}_M{M}", pose_vs_f64=err_stats(pose, r64["pose_opt"]), pose_vs_f32=err_stats(pose, r32["pose_opt"]),
                  logw_vs_f64=err_stats(lw, r64["logw"]), logw_vs_f32=err_stats(lw, r32["logw"]), samples_vs_f64=err_stats(smp, r64["samples"]),
                  f32_vs_f64_logw=err_stats(r32["logw"], r64["logw"]), f32_vs_f64_pose_rel=floor_p, lm_flip_rate=flips)


# ------------------------------------------------------------------------------------------------ properties
@pytest.fixture(scope="module")
def big(cuda_device):
    B, N, M = 4096, 512, 512
    pc = make_problem(B, N, seed=7)
    dev = cuda_device
    d = {k: v.to(dev) for k, v in pc.items()}
    d["delta"] = native.adaptive_delta(d["x2d"], d["w2d"], 0.5)
    d["prob"] = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], None, None, d["delta"])
    d["params"] = native.default_params(6, mc_samples=M, mc_iter=4)
    d["out"] = native.lm_amis_fused(d["prob"], d["pose_init"], d["params"], seed=1234, want_cost=True)
    torch.cuda.synchronize()
    return d


def test_full_size_sanity(big):
    out, M = big["out"], 512
    lw = out["logw"]
    assert torch.isfinite(lw).all() and torch.isfinite(out["pose_samples"]).all()
    q = out["pose_samples"][..., 3:]
    assert (q.norm(dim=-1) - 1).abs().max() < 1e-5
    # LM converged close to the generating pose (sign-free quaternion distance)
    dt = (out["pose_opt"][:, :3] - big["pose_gt"][:, :3]).norm(dim=-1)
    dq = 1 - (out["pose_opt"][:, 3:] * big["pose_gt"][:, 3:]).sum(-1).abs()
    assert dt.median() < 0.03 and dq.median() < 1e-4
    # importance weights are healthy: effective sample size per object
    w = torch.softmax(lw, dim=1)
    ess = 1.0 / (w * w).sum(1)
    assert ess.median() > 0.25 * M and ess.min() > 8
    # the weighted sample mean of the translation sits at the mode within a few posterior sigmas
    mean_t = (w[..., None] * out["pose_samples"][..., :3]).sum(1)
    spread = ((w[..., None] * (out["pose_samples"][..., :3] - mean_t[:, None]) ** 2).sum(1)).sum(-1).sqrt()
    assert (((mean_t - out["pose_opt"][:, :3]).norm(dim=-1)) < 3 * spread + 1e-4).float().mean() > 0.99


def test_full_size_deterministic_and_shard_invariant(big):
    """Same seed -> bit-identical; solving two halves with obj_offset reproduces the full batch exactly
    (what the multi-GPU path relies on)."""
    prob, p = big["prob"], big["params"]
    again = native.lm_amis_fused(prob, big["pose_init"], p, seed=1234, want_cost=True)
    for k in ("pose_opt", "pose_cov", "cost", "logw", "pose_samples"):
        assert torch.equal(again[k], big["out"][k]), k
    h = prob.B // 2 + 3           # uneven split
    for sl, off in ((slice(0, h), 0), (slice(h, prob.B), h)):
        sub = native.Problem(big["x3d"][sl], big["x2d"][sl], big["w2d"][sl], big["cam_mats"][sl], None, None, big["delta"][sl])
        part = native.lm_amis_fused(sub, big["pose_init"][sl], p, seed=1234, obj_offset=off, want_cost=True)
        for k in ("pose_opt", "logw", "pose_samples"):
            assert torch.equal(part[k], big["out"][k][sl]), k
    other = native.lm_amis_fused(prob, big["pose_init"], p, seed=99)
    assert not torch.equal(other["logw"], big["out"]["logw"])
    assert torch.equal(other["pose_opt"], big["out"]["pose_opt"])          # the LM part does not see the seed


def test_lm_flip_rate_at_north_star_shape(big):
    """LM poses of 1024 objects (N = 512) against the fp64 oracle: <= 1e-4 for (almost) all, the rest must
    be cost-equivalent accept/reject flips; the flip rate is printed for the record."""
    from oracle import pnp_oracle as orc
    n = min(1024, big["prob"].B)
    d = torch.float64
    cam = orc.Camera(big["cam_mats"][:n].cpu().to(d), 0.1)
    x3d, x2d, w2d = (big[k][:n].cpu().to(d) for k in ("x3d", "x2d", "w2d"))
    delta = orc.adaptive_delta(x2d, w2d, 0.5)
    pose64, _, cost64 = orc.lm_solve(x3d, x2d, w2d, cam, delta, big["pose_init"][:n].cpu().to(d), orc.LMParams())
    flips = assert_lm_parity(big["out"]["pose_opt"][:n].cpu().numpy(), big["out"]["cost"][:n].cpu().numpy(),
                             pose64.numpy(), cost64.numpy(), 1e-4, max_flip_frac=0.01, what="north-star LM")
    print(f"LM flip rate at N=512: {flips:.4%} of {n} objects")


def test_tma_and_plain_loader_agree(big):
    """Misaligned input pointers force the non-TMA loader; the results must not change by a bit."""
    n = min(64, big["prob"].B)
    def shifted(t):
        buf = torch.empty(t[:n].numel() + 1, dtype=t.dtype, device=t.device)
        buf[1:].copy_(t[:n].reshape(-1))
        return buf[1:].view(t[:n].shape)
    sub = native.Problem(big["x3d"][:n], big["x2d"][:n], big["w2d"][:n], big["cam_mats"][:n], None, None, big["delta"][:n])
    base = native.lm_amis_fused(sub, big["pose_init"][:n], big["params"], seed=5)
    sub.x3d, sub.x2d, sub.w2d = shifted(big["x3d"]), shifted(big["x2d"]), shifted(big["w2d"])
    assert sub.x3d.data_ptr() % 16 != 0
    alt = native.lm_amis_fused(sub, big["pose_init"][:n], big["params"], seed=5)
    for k in ("pose_opt", "logw", "pose_samples"):
        assert torch.equal(base[k], alt[k]), k


def test_point_permutation_invariance(big):
    n = min(128, big["prob"].B)
    perm = torch.randperm(big["prob"].N, device=big["x3d"].device, generator=None)
    sub = native.Problem(big["x3d"][:n], big["x2d"][:n], big["w2d"][:n], big["cam_mats"][:n], None, None, big["delta"][:n])
    subp = native.Problem(big["x3d"][:n][:, perm], big["x2d"][:n][:, perm], big["w2d"][:n][:, perm], big["cam_mats"][:n],
                          None, None, big["delta"][:n])
    a = native.lm_solve(sub, big["pose_init"][:n], big["params"], want_cost=True)
    b = native.lm_solve(subp, big["pose_init"][:n], big["params"], want_cost=True)
    assert err_vs(a["pose_opt"].cpu().numpy(), b["pose_opt"].cpu().numpy()) < 1e-4
    assert err_vs(a["cost"].cpu().numpy(), b["cost"].cpu().numpy()) < 1e-4


def test_philox_draws_are_statistically_equivalent(big):
    """Production RNG (in-kernel Philox) vs injected torch noise: same evidence estimate per object
    (log mean weight) within Monte-Carlo error, and matching ESS distribution."""
    n, M = min(256, big["prob"].B), int(big["params"].mc_samples)
    dev = big["x3d"].device
    sub = native.Problem(big["x3d"][:n], big["x2d"][:n], big["w2d"][:n], big["cam_mats"][:n], None, None, big["delta"][:n])
    noise = tuple(t.to(dev) for t in make_noise(n, M, seed=77))
    a = native.lm_amis_fused(sub, big["pose_init"][:n], big["params"], noise=noise)
    b = native.lm_amis_fused(sub, big["pose_init"][:n], big["params"], seed=4321)
    ev = lambda r: torch.logsumexp(r["logw"], dim=1) - np.log(M)
    ess = lambda r: 1.0 / (torch.softmax(r["logw"], 1) ** 2).sum(1)
    # per-object evidence estimates agree to a few percent (MC std ~ 1/sqrt(ESS))
    assert (ev(a) - ev(b)).abs().median() < 0.1
    assert abs(ess(a).median().item() - ess(b).median().item()) < 0.15 * M


def _oracle_amis_from(prob_cpu, noise_cpu, pose, cov, M, I, dtype, z_min, rel_delta):
    """AMIS of the oracle started from a GIVEN LM solution (so that an LM accept / reject flip cannot leak into the
    comparison of the sampling loop)."""
    from oracle import pnp_oracle as orc
    t = lambda k: prob_cpu[k].to(dtype)
    cam = orc.Camera(t("cam_mats"), z_min)
    delta = orc.adaptive_delta(t("x2d"), t("w2d"), rel_delta)
    B, S = prob_cpu["x3d"].shape[0], M // I
    n3, c2, n4 = noise_cpu
    nz = (n3.reshape(B, I, S, 3).permute(1, 2, 0, 3).to(dtype), c2.reshape(B, I, S).permute(1, 2, 0).to(dtype),
          n4.reshape(B, I, S, 4).permute(1, 2, 0, 3).to(dtype))
    return orc.amis_6dof(t("x3d"), t("x2d"), t("w2d"), cam, delta, pose.to(dtype), cov.to(dtype), nz, M, I)


def test_dense_config_against_oracle_and_capacity(cuda_device):
    """BASELINE config #4 (EPro-PnP-6DoF/lib/test.py:148-229): N = 4096 (64 x 64 coordinate map), AdaptiveHuber(0.1), GN fast
    mode + AMIS -- the 8-warps-per-object LM kernel and the 512-thread AMIS kernel (both chosen by N) against the oracle:
    pose / cost of the solve, then samples and log-weights of the sampling loop started from the kernel's own solution."""
    B, N, M, I = 8, 4096, 512, 4
    pc = make_problem(B, N, seed=3, grid2d=True)
    noise = make_noise(B, M, seed=33)
    dev = cuda_device
    delta = native.adaptive_delta(pc["x2d"].to(dev), pc["w2d"].to(dev), 0.1)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None, delta)
    p = native.default_params(6, lm_iter=3, fast_mode=1, z_min=0.01, mc_samples=M, mc_iter=I)
    out = native.lm_amis_fused(prob, pc["pose_init"].to(dev), p, noise=tuple(t.to(dev) for t in noise), want_cost=True)
    from oracle import pnp_oracle as orc
    cam = orc.Camera(pc["cam_mats"].double(), 0.01)
    d64 = orc.adaptive_delta(pc["x2d"].double(), pc["w2d"].double(), 0.1)
    pose64, cov64, cost64 = orc.lm_solve(pc["x3d"].double(), pc["x2d"].double(), pc["w2d"].double(), cam, d64,
                                         pc["pose_init"].double(), orc.LMParams(num_iter=3), fast_mode=True)
    assert err_vs(out["pose_opt"].cpu().numpy(), pose64.numpy()) < 1e-4
    assert err_vs(out["cost"].cpu().numpy(), cost64.numpy()) < 1e-4
    assert err_vs(out["pose_cov"].cpu().numpy(), cov64.numpy()) < 2e-3
    pose_k, cov_k = out["pose_opt"].cpu(), out["pose_cov"].cpu()
    r64 = _oracle_amis_from(pc, noise, pose_k, cov_k, M, I, torch.float64, 0.01, 0.1)
    r32 = _oracle_amis_from(pc, noise, pose_k, cov_k, M, I, torch.float32, 0.01, 0.1)
    lw = out["logw"].transpose(0, 1).cpu().numpy()
    smp = out["pose_samples"].transpose(0, 1).cpu().numpy()
    floor_w, floor_s = err_vs(r32["logw"], r64["logw"]), err_vs(r32["samples"], r64["samples"])
    assert np.isfinite(lw).all()
    assert err_vs(smp, r64["samples"]) < max(1e-4, 5 * floor_s)
    assert err_vs(lw, r64["logw"]) < max(1e-4, 5 * floor_w)
    mine, ref = np.abs(lw - r64["logw"].numpy()), np.abs(r32["logw"].numpy() - r64["logw"].numpy())
    assert np.median(mine) < 3 * np.median(ref) + 1e-5
    record_parity("oracle/dense_B8_N4096_M512", pose_vs_f64=err_stats(out["pose_opt"].cpu().numpy(), pose64.numpy()),
                  logw_vs_f64=err_stats(lw, r64["logw"]), samples_vs_f64=err_stats(smp, r64["samples"]),
                  f32_vs_f64_logw=err_stats(r32["logw"], r64["logw"]))
    too_many = native.capi.lib().epnp_max_points(6, 512, 4) + 4
    big_prob = native.Problem(torch.zeros(1, too_many, 3, device=dev), torch.zeros(1, too_many, 2, device=dev),
                              torch.zeros(1, too_many, 2, device=dev), pc["cam_mats"][:1].to(dev), None, None, 1.0)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.lm_amis_fused(big_prob, pc["pose_init"][:1].to(dev), p)


def test_full_batch_strided_subset_against_oracle(cuda_device):
    """The metric's own shape, B = 4096 / N = 512 / M = 512, with injected noise: every 64th object of the full-size launch
    (first and last CTAs of the grid included) against the fp64 oracle -- pose, samples and log-weights."""
    B, N, M, I, stride = 4096, 512, 512, 4, 64
    pc = make_problem(B, N, seed=17)
    noise = make_noise(B, M, seed=18)
    dev = cuda_device
    delta = native.adaptive_delta(pc["x2d"].to(dev), pc["w2d"].to(dev), 0.5)
    prob = native.Problem(pc["x3d"].to(dev), pc["x2d"].to(dev), pc["w2d"].to(dev), pc["cam_mats"].to(dev), None, None, delta)
    p = native.default_params(6, mc_samples=M, mc_iter=I)
    out = native.lm_amis_fused(prob, pc["pose_init"].to(dev), p, noise=tuple(t.to(dev) for t in noise), want_cost=True)
    idx = torch.cat((torch.arange(0, B, stride), torch.tensor([B - 1])))
    sub = {k: v[idx] for k, v in pc.items()}
    nz = tuple(t[idx] for t in noise)
    r64 = _oracle_run(sub, nz, M, I, torch.float64)
    r32 = _oracle_run(sub, nz, M, I, torch.float32)
    pose = out["pose_opt"][idx.to(dev)].cpu().numpy()
    lw = out["logw"][idx.to(dev)].transpose(0, 1).cpu().numpy()
    smp = out["pose_samples"][idx.to(dev)].transpose(0, 1).cpu().numpy()
    floor_p, floor_w, floor_s = (err_vs(r32[k], r64[k]) for k in ("pose_opt", "logw", "samples"))
    flips = assert_lm_parity(pose, out["cost"][idx.to(dev)].cpu().numpy(), r64["pose_opt"].numpy(), r64["lm_cost"].numpy(),
                             max(1e-4, 3 * floor_p), max_flip_frac=0.05, what="strided subset")
    assert err_vs(smp, r64["samples"]) < max(1e-4, 5 * floor_s)
    assert err_vs(lw, r64["logw"]) < max(1e-4, 5 * floor_w)
    if flips == 0.0:
        assert err_vs(pose, r32["pose_opt"]) < 1e-4 and err_vs(lw, r32["logw"]) < 1e-4 + 2 * floor_w
    record_parity("oracle/full_batch_B4096_every64th", objects=int(idx.numel()), pose_vs_f64=err_stats(pose, r64["pose_opt"]),
                  logw_vs_f64=err_stats(lw, r64["logw"]), logw_vs_f32=err_stats(lw, r32["logw"]), samples_vs_f64=err_stats(smp, r64["samples"]),
                  f32_vs_f64_logw=err_stats(r32["logw"], r64["logw"]), lm_flip_rate=flips)


def test_host_buffer_entry_point(big):
    """C-ABI call with HOST (pinned) buffers == device-resident call (same seed), chunked copies."""
    n = 512
    p = big["params"]
    host = {k: big[k][:n].cpu().contiguous().pin_memory() for k in ("x3d", "x2d", "w2d", "cam_mats", "delta", "pose_init")}
    ws = torch.empty(native.fused_workspace_bytes(n, 512, p), dtype=torch.uint8, device=big["x3d"].device)
    res = native.lm_amis_fused_host(host, p, ws, n_chunks=4, seed=1234)
    torch.cuda.synchronize()
    for k in ("pose_opt", "logw", "pose_samples", "pose_cov", "cost"):
        assert torch.equal(res[k], big["out"][k][:n].cpu()), k
