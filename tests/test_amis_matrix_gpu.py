"""The AMIS loop (amis_loop, pnp_amis.cuh) against the float64 oracle per object and per iteration, across its kernel
forms, clamps and sample counts.

amis_loop runs in three forms: amis_kernel<DOF, 128> for N < 2048 (one thread draws and sweeps one sample; S > 128 takes
a second draw pass), amis_kernel<DOF, 512> from N = 2048 (the sweep of a sample cut into four point ranges at multiples
of four pairs) and amis_split_kernel (the same loop on a thread-block cluster, the ranks' partial costs summed per
iteration).  The form depends on N alone.

Every case injects its noise (no Philox) and starts from a fixed local solution, so no LM decision enters the
comparison: the resident forms run native.amis from the float64 oracle LM pose and covariance rounded to float32; the
split form, which has no AMIS-only entry point, runs the fused call and the oracle starts from the kernel's own pose_opt /
pose_cov.  The oracle's amis_6dof / amis_4dof (oracle/pnp_oracle.py, pinned to the reference by test_oracle_cpu.py) runs
on the same float32 inputs in float64 and in float32.

Each metric of each object is held to max(MIN, K * floor), floor = the same metric of the float32 oracle against the
float64 one on that object.  Per iteration i: the samples' translation max|dt| / max|t64| and quaternion max|dq|
(absolute, in units of what the draw magnifies an error of L_r by; the same noise, so the same sign), 4DoF yaw equal to the injected draws; the proposal's mode (relative; at
i = 0 equal to pose_opt[:3]), L_t and L_r (max|dL| / max|L64|), 4DoF yaw mode (wrapped, absolute) and kappa (relative).
The final log-weights: logsumexp (absolute, over max(1, |lse64|)), the normalised weights (max|dw| / max w64) and the
log-weights themselves (max|dlogw| / max|logw64|).

The bounds clamp, the z_min clamp and the Huber branch are continuous in the cost, so bounds and z_min need no gap.  The
one decision left is the positive-definiteness test of the refit's Cholesky factorisations: every refit of an ordinary
case must have its smallest pivot above PIVOT_MARGIN of its trace in float64 (a census), and the collapse cases put one
object where the weights are one-hot in float32 and float64 alike, so that the fallback is taken on both sides.
"""
import math

import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
import test_lm_matrix_gpu as lmm
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp_b200 import native
from epropnp_b200.synth import make_noise, make_problem

pytestmark = pytest.mark.gpu

f64 = torch.float64
K_FIRST = 5             # iteration 0 and its proposal: max(MIN, K_FIRST * floor) per object and metric
K_LATER = 10            # later iterations and the final log-weights: every refit passes its rounding on
MIN = 1e-4              # every metric
PIVOT_MARGIN = 1e-6     # least smallest-Cholesky-pivot / trace of a refit matrix in an ordinary case (about 17 float32
#                         units of roundoff of the trace: rounding cannot take the factorisation to the fallback)
COLLAPSE_GAP = 800.0    # log-weight gap at every refit of a collapse object: exp(-800) is 0 in float32 and float64
COLLAPSE_SCALE = 300.0  # its w2d factor, applied after the local solution (the cost grows with its square)
MAX_ITER = 8            # MAX_ITER (pnp_math.cuh)
DENSE_N = 2048          # AMIS_DENSE_MIN_N (pnp_amis.cuh)
ORACLE_PAIRS = 1 << 23  # (sample, point) pairs per oracle call and iteration: objects are run in chunks below it


# ------------------------------------------------------------------------------------------------ the cases
# form ("resident" | "split"), dof, N (an int, "max" = max_points(dof, M, I), "split_max" = max_points_split(dof, M, I)),
# M, I, B, bounds (None | "scalar" | "tensor"), zmin (z_min at the 15 % quantile of the depths), outliers (share of
# points moved off the Huber quadratic branch), mixed (object 0's w2d times 1e-3), ctas (split: cluster size, 0 =
# automatic), kappa (4DoF: yaw draws concentrated on the mode, so the refit's kappa is large), collapse (resident:
# object 0's w2d times COLLAPSE_SCALE after its local solution, so its weights are one-hot at every refit), seed.
def _c(form, dof, N, M, I, B, bounds=None, zmin=False, outliers=0.0, mixed=False, ctas=0, kappa=False, collapse=False,
       seed=1):
    tag = "".join([f"{form}_d{dof}_N{N}_M{M}_I{I}_B{B}", f"_{bounds}" if bounds else "", "_zmin" if zmin else "",
                   "_outl" if outliers else "", "_mixed" if mixed else "", f"_C{ctas}" if form == "split" else "",
                   "_kappa" if kappa else "", "_collapse" if collapse else ""])
    return dict(id=tag, form=form, dof=dof, N=N, M=M, I=I, B=B, bounds=bounds, zmin=zmin, outliers=outliers,
                mixed=mixed, ctas=ctas, kappa=kappa, collapse=collapse, seed=seed)


CASES = [
    # resident, T = 128
    _c("resident", 6, 3, 8, 1, 4),                                                  # I = 1: no refit
    _c("resident", 6, 7, 64, 8, 4, bounds="scalar"),                                # I = MAX_ITER
    _c("resident", 6, 127, 508, 4, 4, bounds="tensor"),
    _c("resident", 6, 128, 512, 4, 4, zmin=True),
    _c("resident", 6, 129, 516, 4, 4, outliers=0.1),                                # S = 129: the second draw pass
    _c("resident", 6, 513, 520, 2, 6, zmin=True, mixed=True),                       # S = 260
    _c("resident", 6, 2047, 512, 4, 4, bounds="scalar", outliers=0.1),
    # (M / I = 8 / 2 leaves four samples per refit: their weighted 3 x 3 covariance is singular in float64 for most
    # objects, so the fallback would be decided by rounding; 32 per refit clear the pivot margin)
    _c("resident", 4, 5, 64, 2, 4),
    _c("resident", 4, 128, 512, 4, 4, bounds="tensor", zmin=True),
    _c("resident", 4, 129, 1032, 8, 4, outliers=0.1),                               # I = 8, S = 129
    # resident, T = 512
    _c("resident", 6, 2048, 512, 4, 4, bounds="tensor", zmin=True),
    _c("resident", 6, 2050, 132, 4, 4),                 # 1025 pairs: the four ranges 256 / 256 / 256 / 257
    _c("resident", 6, 4096, 512, 4, 8, outliers=0.1, mixed=True),
    _c("resident", 6, "max", 512, 4, 3, bounds="tensor"),
    _c("resident", 4, 2048, 256, 4, 4, bounds="scalar"),
    _c("resident", 4, 4096, 512, 4, 4, kappa=True),
    # split
    # (seed 1 put one object's iteration-2 quaternion samples at 1.0006 x their bound, and seed 1 at split_max one
    # object's iteration-3 ones at 1.25 x MIN: the ACG proposal is eps-dominated at these N, its L_r's short axes carry
    # rounding into the draws beyond what the float32 oracle's own rounding shows; the emulator build passes seed 1)
    _c("split", 6, 16384, 512, 4, 3, bounds="tensor", outliers=0.1, seed=2),
    _c("split", 6, 4096, 512, 4, 3, zmin=True, ctas=2),
    _c("split", 6, 4096, 512, 4, 3, zmin=True, ctas=8),
    _c("split", 6, "split_max", 512, 4, 2, ctas=8, seed=2),
    _c("split", 6, 16384, 64, 8, 3),
    _c("split", 4, 16384, 512, 4, 3, bounds="scalar", zmin=True),
    # collapse
    _c("resident", 6, 512, 512, 4, 3, collapse=True),
    _c("resident", 4, 512, 512, 4, 3, collapse=True),
]


def resolve_n(case):
    N = case["N"]
    if N == "max":
        return native.max_points(case["dof"], case["M"], case["I"])
    if N == "split_max":
        return native.max_points_split(case["dof"], case["M"], case["I"])
    return N


def _d(t):
    return t.detach().cpu().to(f64)


# ------------------------------------------------------------------------------------------------ building a case
def _yaw_draws(c, case, gen):
    """4DoF injected yaw (B, M): three quarters around the local solution's yaw (spread 3 sigma of its variance, at
    least 0.05 rad; 0.01 rad for a kappa case), a quarter uniform on the circle, as the proposal mixture draws."""
    B, M = case["B"], case["M"]
    mode = _d(c["pose_opt"])[:, 3:4]
    sd = (3 * _d(c["pose_cov"])[:, 3, 3].clamp(min=0).sqrt()).clamp(min=0.05)[:, None]
    if case["kappa"]:
        sd = torch.full_like(sd, 0.01)
    near = mode + sd * torch.randn(B, M, generator=gen, dtype=f64)
    far = torch.rand(B, M, generator=gen, dtype=f64) * (2 * math.pi) - math.pi
    yaw = torch.where(torch.rand(B, M, generator=gen, dtype=f64) < 0.75, near, far)
    return torch.atan2(torch.sin(yaw), torch.cos(yaw)).float()


def _place(c, case):
    """z_min at the 15 % quantile of the depths at pose_init; bounds about 4 % of the projections in on each side."""
    x3d, cam, p0 = _d(c["x3d"]), _d(c["cam_mats"]), _d(c["pose_init"])[:, None]
    if case["zmin"]:
        zh, _ = bm.project(x3d, p0.transpose(0, 1), cam, 0.1)
        c["z_min"] = float(np.float32(float(bm.quantile(zh.reshape(1, -1), 0.15)[0])))
    if case["bounds"]:
        lb, ub, _ = bm.place_bounds(x3d, p0, cam, c["z_min"], case["bounds"] == "tensor")
        dev = c["x3d"].device
        c["lb"], c["ub"] = (lb.to(dev), ub.to(dev)) if torch.is_tensor(lb) else (lb, ub)


def build_case(case, dev):
    dof, B, M, I, N = case["dof"], case["B"], case["M"], case["I"], resolve_n(case)
    pc = make_problem(B, N, seed=case["seed"] + N, dof=dof, outlier_frac=case["outliers"])
    if case["mixed"]:
        pc["w2d"][0] *= 1e-3
    if case["zmin"]:
        # every object at depth 4 (points and translation scaled together: the projections do not change), so one
        # z_min cuts into each of them
        s = 4.0 / pc["pose_gt"][:, 2]
        pc["x3d"] = (pc["x3d"] * s[:, None, None]).contiguous()
        for k in ("pose_gt", "pose_init"):
            pc[k][:, :3] *= s[:, None]
    c = {k: v.to(dev) for k, v in pc.items()}
    c.update(dof=dof, B=B, N=N, M=M, I=I, z_min=0.1, lb=None, ub=None)
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5)
    _place(c, case)
    c["params"] = native.default_params(dof, z_min=c["z_min"], lm_iter=3, fast_mode=1, mc_samples=M, mc_iter=I)
    n3, c2, r = make_noise(B, M, seed=case["seed"] + 7, dof=dof)
    c["noise"] = [n3, c2, r]
    if case["form"] == "resident":
        # the local solution: the float64 oracle's LM, rounded to float32 (both sides start from these values)
        r64 = lmm.Ref(c, f64)
        pose, cov, _ = orc.lm_solve(r64.x3d, r64.x2d, r64.w2d, r64.cam, r64.delta, _d(c["pose_init"]),
                                    orc.LMParams(num_iter=10, eps=1e-5))
        c["pose_opt"], c["pose_cov"] = pose.float().to(dev), cov.float().to(dev)
        if case["collapse"]:
            # after the local solution: proposal 0 is COLLAPSE_SCALE times wider than the object's posterior, so one
            # sample outweighs the rest by more than COLLAPSE_GAP
            c["w2d"][0] *= COLLAPSE_SCALE
            c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5)
    if dof == 4:
        if "pose_opt" not in c:         # split: the yaw draws centre on the kernel's LM, which has the same inputs
            out = native.lm_solve(problem(c), c["pose_init"], c["params"], want_cov=True)
            c["pose_opt"], c["pose_cov"] = out["pose_opt"], out["pose_cov"]
        c["noise"][2] = _yaw_draws(c, case, torch.Generator().manual_seed(case["seed"] + 11))
    c["noise"] = tuple(t.contiguous().to(dev) for t in c["noise"])
    return c


def problem(c, objs=slice(None)):
    cut = lambda b: b[objs] if torch.is_tensor(b) else b
    return native.Problem(c["x3d"][objs], c["x2d"][objs], c["w2d"][objs], c["cam_mats"][objs], cut(c["lb"]),
                          cut(c["ub"]), c["delta"][objs])


def run_kernel(c, case, objs=slice(None)):
    """-> samples (B, M, D), logw (B, M), proposals (B, I, 19), pose_opt, pose_cov the AMIS loop started from."""
    nz = tuple(t[objs] for t in c["noise"])
    if case["form"] == "resident":
        smp, lw, props = native.amis(problem(c, objs), c["pose_opt"][objs], c["pose_cov"][objs], c["params"], noise=nz,
                                     want_proposals=True)
        return dict(samples=smp, logw=lw, proposals=props, pose_opt=c["pose_opt"][objs], pose_cov=c["pose_cov"][objs])
    out = native.lm_amis_fused_split(problem(c, objs), c["pose_init"][objs], c["params"], noise=nz,
                                     want_proposals=True, cluster_ctas=case["ctas"])
    return dict(samples=out["pose_samples"], logw=out["logw"], proposals=out["proposals"], pose_opt=out["pose_opt"],
                pose_cov=out["pose_cov"])


# ------------------------------------------------------------------------------------------------ the oracle
def _cat(parts, key):
    v = [p[key] for p in parts]
    if isinstance(v[0], list):
        return [torch.cat([x[k] for x in v], -1) for k in range(len(v[0]))]
    return torch.cat(v, 2 if key == "cost" else 1)


def oracle(c, pose, cov, dtype):
    """The oracle's AMIS loop on the case's float32 inputs and the float32 start (pose, cov), in `dtype`, objects in
    chunks of at most ORACLE_PAIRS (sample, point) pairs per iteration."""
    B, M, I, N, dof = c["B"], c["M"], c["I"], c["N"], c["dof"]
    S = M // I
    cv = lambda t: t.detach().cpu().to(dtype)
    n3, c2, r = (t.cpu() for t in c["noise"])
    nz = [n3.reshape(B, I, S, 3).permute(1, 2, 0, 3), c2.reshape(B, I, S).permute(1, 2, 0)]
    nz.append(r.reshape(B, I, S, 4).permute(1, 2, 0, 3) if dof == 6 else r.reshape(B, I, S).permute(1, 2, 0))
    step = max(1, ORACLE_PAIRS // (S * N))
    parts = []
    for b0 in range(0, B, step):
        sl = slice(b0, min(B, b0 + step))
        bound = lambda b: cv(b[sl]) if torch.is_tensor(b) else b
        cam = orc.Camera(cv(c["cam_mats"][sl]), c["z_min"], bound(c["lb"]), bound(c["ub"]))
        args = (cv(c["x3d"][sl]), cv(c["x2d"][sl]), cv(c["w2d"][sl]), cam, cv(c["delta"][sl]), cv(pose[sl]),
                cv(cov[sl]), tuple(cv(t[:, :, sl]) for t in nz), M, I)
        parts.append((orc.amis_6dof if dof == 6 else orc.amis_4dof)(*args, return_refit=True))
    return {k: _cat(parts, k) for k in parts[0]}


# ------------------------------------------------------------------------------------------------ metrics (float64)
_TRIL3 = ([0, 1, 1, 2, 2, 2], [0, 0, 1, 0, 1, 2])
_TRIL4 = ([0, 1, 1, 2, 2, 2, 3, 3, 3, 3], [0, 0, 1, 0, 1, 2, 0, 1, 2, 3])


def rel(a, b):
    """(B,): max|a - b| / max|b| per object (leading axis)."""
    return bm.per_object(_d(a), _d(b))


def absd(a, b, units=None):
    """(B,): max|a - b| per object; units (B, S): each sample's difference is divided by its unit first."""
    a, b = _d(a), _d(b)
    d = (a - b).abs()
    if units is not None:
        d = d / units[..., None]
    return d.reshape(a.shape[0], -1).amax(1).numpy()


def draw_units(n4, L):
    """(B, S): how much the ACG draw q = L n4 / |L n4| magnifies an error of L, ||L||_max |n4| / |L n4| (float64 L of
    the iteration's proposal, injected n4 (B, S, 4)).  A sample whose noise points along a short axis of L divides by a
    small |L n4|; the quaternion differences are compared in these units, so that one such sample does not decide the
    metric of its object."""
    n4, L = _d(n4), _d(L)
    g = (L[:, None] @ n4[..., None]).squeeze(-1)
    return L.abs().amax((1, 2))[:, None] * n4.norm(dim=-1) / g.norm(dim=-1)


def wrapped(a, b):
    d = _d(a) - _d(b)
    return torch.atan2(torch.sin(d), torch.cos(d)).abs().reshape(d.shape[0], -1).amax(1).numpy()


def lse_err(a, b):
    la, lb = torch.logsumexp(_d(a), 1), torch.logsumexp(_d(b), 1)
    return ((la - lb).abs() / lb.abs().clamp(min=1.0)).numpy()


def softmax_err(a, b):
    return rel(torch.softmax(_d(a), 1), torch.softmax(_d(b), 1))


def oracle_views(r, dof):
    """The oracle's outputs in the kernel's layouts: samples (B, M, D), logw (B, M), per iteration (B, I, ...)."""
    v = dict(samples=r["samples"].transpose(0, 1), logw=r["logw"].transpose(0, 1),
             mode=r["trans_mode"].transpose(0, 1), lt=r["trans_tril"][..., _TRIL3[0], _TRIL3[1]].transpose(0, 1))
    if dof == 6:
        v["lr"] = r["rot_tril"][..., _TRIL4[0], _TRIL4[1]].transpose(0, 1)
    else:
        v["rot_mode"], v["kappa"] = r["rot_mode"].T, r["rot_kappa"].T
    return v


def compare(c, case, got, r64, r32, stats, skip_lt=()):
    """Every metric of every object against max(MIN, K * floor).  skip_lt: (object, iteration) pairs whose L_t is the
    Cholesky fallback, compared exactly by the caller."""
    what, dof, M, I = case["id"], c["dof"], c["M"], c["I"]
    S = M // I
    a, o, f = dict(samples=got["samples"], logw=got["logw"]), oracle_views(r64, dof), oracle_views(r32, dof)
    props = got["proposals"]
    assert torch.isfinite(got["samples"]).all() and torch.isfinite(got["logw"]).all() and torch.isfinite(props).all()
    for i in range(I):
        k = K_FIRST if i == 0 else K_LATER
        sl = slice(i * S, (i + 1) * S)
        ks, os_, fs = a["samples"][:, sl], o["samples"][:, sl], f["samples"][:, sl]
        lmm.check(stats, what, f"it{i}_sample_t", rel(ks[..., :3], os_[..., :3]), rel(fs[..., :3], os_[..., :3]), k, MIN)
        if dof == 6:
            u = draw_units(c["noise"][2][:, sl], r64["rot_tril"][i])
            lmm.check(stats, what, f"it{i}_sample_q", absd(ks[..., 3:], os_[..., 3:], u),
                      absd(fs[..., 3:], os_[..., 3:], u), k, MIN)
        else:
            assert torch.equal(ks[..., 3].cpu(), c["noise"][2][:, sl].cpu()), (what, i, "yaw draws")
        if i == 0:
            assert torch.equal(props[:, 0, :3], got["pose_opt"][:, :3]), (what, "proposal 0 mode")
        else:
            lmm.check(stats, what, f"it{i}_mode", rel(props[:, i, :3], o["mode"][:, i]),
                      rel(f["mode"][:, i], o["mode"][:, i]), k, MIN)
        keep = np.array([(b, i) not in skip_lt for b in range(c["B"])])
        lmm.check(stats, what, f"it{i}_L_t", rel(props[:, i, 3:9], o["lt"][:, i]), rel(f["lt"][:, i], o["lt"][:, i]),
                  k, MIN, only=keep)
        if dof == 6:
            lmm.check(stats, what, f"it{i}_L_r", rel(props[:, i, 9:19], o["lr"][:, i]),
                      rel(f["lr"][:, i], o["lr"][:, i]), k, MIN)
        else:
            lmm.check(stats, what, f"it{i}_yaw_mode", wrapped(props[:, i, 9:10], o["rot_mode"][:, i:i + 1]),
                      wrapped(f["rot_mode"][:, i:i + 1], o["rot_mode"][:, i:i + 1]), k, MIN)
            lmm.check(stats, what, f"it{i}_kappa", rel(props[:, i, 10:11], o["kappa"][:, i:i + 1]),
                      rel(f["kappa"][:, i:i + 1], o["kappa"][:, i:i + 1]), k, MIN)
    k = K_FIRST if I == 1 else K_LATER
    lmm.check(stats, what, "lse", lse_err(a["logw"], o["logw"]), lse_err(f["logw"], o["logw"]), k, MIN)
    lmm.check(stats, what, "weights", softmax_err(a["logw"], o["logw"]), softmax_err(f["logw"], o["logw"]), k, MIN)
    lmm.check(stats, what, "logw", rel(a["logw"], o["logw"]), rel(f["logw"], o["logw"]), k, MIN)


# ------------------------------------------------------------------------------------------------ census (float64)
def census(c, samples):
    """Shares of the (sample, point) pairs of the float64 run below z_min, clamped by a bound, on the Huber linear
    branch; samples (B, M, D)."""
    x3d, x2d, w2d, cam, delta = (_d(c[k]) for k in ("x3d", "x2d", "w2d", "cam_mats", "delta"))
    B, M, N = samples.shape[0], samples.shape[1], c["N"]
    counts = torch.zeros(3, dtype=f64)
    step = max(1, (1 << 22) // (B * N))
    for p0 in range(0, M, step):
        ps = _d(samples[:, p0:p0 + step]).transpose(0, 1)
        zh, u = bm.project(x3d, ps, cam, c["z_min"])
        counts[0] += float((zh < c["z_min"]).sum())
        if c["lb"] is not None:
            lo = orc._bound(_d(c["lb"]) if torch.is_tensor(c["lb"]) else c["lb"], u)
            hi = orc._bound(_d(c["ub"]) if torch.is_tensor(c["ub"]) else c["ub"], u)
            counts[1] += float(((u < lo) | (u > hi)).any(-1).sum())
            u = torch.minimum(torch.maximum(u, lo), hi)
        counts[2] += float((((u - x2d) * w2d).norm(dim=-1) > delta[:, None]).sum())
    fr = (counts / (B * M * N)).tolist()
    return dict(below_zmin=fr[0], clamped=fr[1], outlier=fr[2])


def pivot_margin(mats):
    """(..., n, n) -> (...): smallest Cholesky pivot (L_jj^2) over the trace; 0 where the factorisation fails."""
    L, info = torch.linalg.cholesky_ex(mats)
    piv = L.diagonal(dim1=-2, dim2=-1).square().amin(-1) / mats.diagonal(dim1=-2, dim2=-1).sum(-1).abs()
    return torch.where(info == 0, piv, torch.zeros_like(piv))


def refit_margins(r64):
    """(B,): the least pivot margin over every refit matrix of each object (inf without a refit)."""
    ms = [pivot_margin(r64[k]) for k in ("refit_trans", "refit_rot") if k in r64 and r64[k].shape[0]]
    if not ms:
        return torch.full((r64["logw"].shape[1],), float("inf"), dtype=f64)
    return torch.cat(ms, 0).amin(0)


def refit_gaps(r64):
    """(B,): the least gap between the largest and the second-largest log-weight over the refits."""
    gaps = [(lambda t: t[0] - t[1])(lw.topk(2, dim=0).values) for lw in r64["refit_logw"]]
    return torch.stack(gaps).amin(0)


def check_conditions(case, c, fr):
    # (a case without zmin may still put the heavy tails of its Student-t draws below the default z_min: recorded only)
    if case["zmin"]:
        assert 0.02 <= fr["below_zmin"] <= 0.9, fr
    if case["bounds"]:
        assert 0.02 <= fr["clamped"] <= 0.9, fr
    else:
        assert fr["clamped"] == 0.0, fr
    if case["outliers"]:
        assert 0.01 <= fr["outlier"] <= 0.99, fr          # both Huber branches
    if case["mixed"]:
        w = c["w2d"].abs().double().mean((1, 2))
        assert float(w[0]) < 1e-2 * float(w[1:].min())


# ------------------------------------------------------------------------------------------------ a case
def run_case(case, dev, record="amis_matrix"):
    c = build_case(case, dev)
    what, dof, I = case["id"], case["dof"], case["I"]
    got = run_kernel(c, case)
    r64 = oracle(c, got["pose_opt"], got["pose_cov"], f64)
    r32 = oracle(c, got["pose_opt"], got["pose_cov"], torch.float32)
    fr = census(c, r64["samples"].transpose(0, 1))
    check_conditions(case, c, fr)
    stats = {}
    margins = refit_margins(r64)
    ordinary = np.ones(c["B"], bool)
    skip_lt = set()
    if case["collapse"]:
        ordinary[0] = False
        gap = float(refit_gaps(r64)[0])
        assert gap > COLLAPSE_GAP, (what, gap)
        stats["collapse_logw_gap"] = gap
        # the weights are one-hot: the translation covariance is exactly zero, and both sides take the fallback
        assert float(r64["refit_trans"][:, 0].abs().max()) == 0.0
        o_lt = oracle_views(r64, dof)["lt"]
        for i in range(1, I):
            assert torch.equal(got["proposals"][0, i, 3:9].cpu(), o_lt[0, i].float()), (what, i, "fallback L_t")
            skip_lt.add((0, i))
    if I > 1:
        m = margins.numpy()[ordinary]
        assert (m > PIVOT_MARGIN).all(), (what, "refit pivot margins", m.tolist())
        stats["refit_pivot_margin_min"] = float(m.min())
    compare(c, case, got, r64, r32, stats, skip_lt)
    record_parity(f"{record}/{what}", B=c["B"], N=c["N"], M=c["M"], I=I, dof=dof, form=case["form"],
                  cluster_ctas=case["ctas"] if case["form"] == "split" else None, z_min=c["z_min"],
                  bounds=case["bounds"] or "none", k_first=K_FIRST, k_later=K_LATER, min=MIN,
                  pivot_margin_bound=PIVOT_MARGIN, **fr, **stats)
    return c, got


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_amis_matrix(cuda_device, case):
    run_case(case, cuda_device)


def test_every_form_is_in_the_matrix():
    """Both sides of the 128 / 512-thread boundary, S on both sides of 128, I = 1 and MAX_ITER, a dense pair count that
    is not a multiple of 4, both DoFs in every form, and every clamp."""
    res = [cs for cs in CASES if cs["form"] == "resident"]
    ns = {(cs["dof"], cs["N"]) for cs in res}
    assert {(6, DENSE_N - 1), (6, DENSE_N), (4, DENSE_N)} <= ns and any(cs["dof"] == 4 and cs["N"] < DENSE_N for cs in res)
    s = {cs["M"] // cs["I"] for cs in res if isinstance(cs["N"], int) and cs["N"] < DENSE_N}
    assert {127, 128, 129} <= s and any(v > 256 for v in s)
    assert {cs["I"] for cs in CASES} >= {1, 2, 4, MAX_ITER}
    assert any(isinstance(n, int) and n >= DENSE_N and ((n + 1) // 2) % 4 for _, n in ns)
    assert {cs["dof"] for cs in CASES if cs["form"] == "split"} == {4, 6}
    assert {cs["ctas"] for cs in CASES if cs["form"] == "split"} >= {0, 2, 8}
    assert {(cs["dof"], cs["collapse"]) for cs in CASES} >= {(6, True), (4, True)}
    for key in ("bounds", "zmin", "outliers", "mixed", "kappa"):
        assert any(cs[key] for cs in CASES)
    assert {cs["bounds"] for cs in CASES} == {None, "scalar", "tensor"}


# ------------------------------------------------------------------------------------------------ per-object independence
@pytest.mark.parametrize("idx", [3, 12])
def test_object_alone_equals_its_row(cuda_device, idx):
    """The kernel's form depends on N alone: an object run by itself gives its row of the batched run bit for bit."""
    case = CASES[idx]
    c = build_case(case, cuda_device)
    full = run_kernel(c, case)
    for b in (0, c["B"] - 1):
        one = run_kernel(c, case, slice(b, b + 1))
        for k in ("samples", "logw", "proposals"):
            assert torch.equal(one[k][0], full[k][b]), (case["id"], b, k)
