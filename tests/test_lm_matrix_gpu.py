"""The LM / GN solve (lm_warp_kernel) against the float64 oracle per object, across its kernel variants, clamps and
outputs.

lm_warp_kernel has three forms, chosen by N alone: <D, true, 1> stages the object's points in one warp's shared memory
(N <= 640, by TMA when N % 4 == 0 and the inputs are 16-byte aligned, else by the plain loader), <D, false, 1> reads them
from global memory with one warp (641 <= N <= 2047) and <D, false, 8> with eight warps whose partial sums meet in shared
memory (N >= 2048).  The matrix puts cases on both sides of each boundary with N = 1, 2, 3 (mod 4), in 6DoF and 4DoF,
unbounded, with scalar and per-object bounds, with depths below z_min, with both Huber branches, and in batches where one
object's weights are 1e-3 of its neighbours' (its cost and gradients 1e-6 of theirs).  The reference is
oracle/pnp_oracle.py in float64 (pinned to the reference implementation by test_oracle_cpu.py).

Every object is compared on its own, against max(MIN, K * floor), floor = the same oracle in float32 against float64 for
that object.  Metrics: translation |dt| / |t64|; rotation the sign-free angle between the quaternions (6DoF) or |dyaw|
(4DoF), in radians, absolute; a Gauss-Newton step or pose_opt_plus by its increment (dt and the rotation increment in
the tangent space of the start quaternion) against the float64 increment, relative to its norm; pose_cov max|a - b| /
max|b| within the object; cost and cost_init relative.

Part A: single evaluations, no accept / reject decision, so no flip clause.  Part B: whole solves; GN (fast mode) has no
decisions either; LM may leave the tight bound only for an object whose float64 trajectory had a decision inside float32
noise, and then must be cost-equivalent (conftest.assert_lm_parity's clause).

The clamps make the solve discontinuous: a projection within float32 rounding of a bound, or a depth within rounding of
z_min, may take the other side in the kernel.  So bounds and z_min are placed in the widest gap of the float64
projections at every float64 iterate (accepted or proposed) and the margin is asserted.
"""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
from conftest import assert_lm_parity, record_parity
from oracle import pnp_oracle as orc
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

f64 = torch.float64
K_A = 5                 # Part A bound: max(MIN, K_A * floor) per object and output
K_B = 10                # Part B: an iterated solve compounds the rounding of every step
REL_MIN = 2e-4          # cost, cost_init, pose_cov, the residual / Jacobian and the increments (relative)
TRANS_MIN = 2e-5        # translation, relative to |t64|
ROT_MIN = 2e-5          # rotation, radians (absolute)
TIE = 1e-5              # a float64 LM decision with |cost - cost_new| or |model_change| below TIE * cost is a tie
MAX_FLIP = 0.5          # share of the objects of a case that may take the flip clause
CONVERGED_STEP = 1e-4   # pose_opt_plus after a whole solve: the increment's scale is at least this times |t64|
COV_COND_MAX = 1e6      # pose_cov is compared where cond(J^T J + eps I) is below this
BOUND_GAP = bm.BOUND_GAP
ZMIN_GAP = bm.ZMIN_GAP
EPS = 1e-5
HUBER_EPS = 1e-10
STAGE_MAX_N = 640       # LM_STAGE_MAX_N (pnp_lm.cuh)
EIGHT_WARP_N = 2048     # lm_warps_per_object (pnp_kernels.cu)


def resolve_n(case):
    N = case["N"]
    if N == "epnp_max":
        return native.max_points(6, 512, 4)
    if N == "split_max":
        return native.max_points_split(6, 0, 0)
    return N


# ------------------------------------------------------------------------------------------------ the cases
# dof, N, B, mode ("lm": Part B is LM with lm_iter = 10, "fast": GN with lm_iter = 3), bounds (None | "scalar" |
# "tensor"), zmin (a share of the depths below z_min), outliers (share of points on the Huber linear branch), mixed
# (object 0's w2d times 1e-3), seed (of the problem; one whose float64 trajectory leaves no gap wide enough for the
# bounds takes another -- seed 3 at N = 16384 left 2.3e-4 px).
def _c(dof, N, B, mode, bounds=None, zmin=False, outliers=0.0, mixed=False, seed=3):
    tag = "".join([f"d{dof}_N{N}_B{B}_{mode}", f"_{bounds}" if bounds else "", "_zmin" if zmin else "",
                   "_outl" if outliers else "", "_mixed" if mixed else ""])
    return dict(id=tag, dof=dof, N=N, B=B, mode=mode, bounds=bounds, zmin=zmin, outliers=outliers, mixed=mixed,
                seed=seed)


CASES = [
    _c(6, 1, 1, "lm"),
    _c(4, 3, 3, "fast"),
    _c(6, 4, 3, "fast", bounds="scalar"),
    _c(6, 7, 5, "lm", outliers=0.2, mixed=True),
    _c(4, 64, 8, "lm", bounds="tensor"),
    _c(6, 511, 4, "lm", zmin=True),
    _c(6, 512, 1, "fast", bounds="tensor", outliers=0.1),
    _c(4, 513, 4, "fast", zmin=True),
    _c(6, 637, 3, "lm", outliers=0.1),
    _c(4, 638, 3, "lm", bounds="scalar"),
    _c(6, 639, 3, "fast", mixed=True),
    _c(6, 640, 4, "lm", bounds="tensor", outliers=0.1),
    _c(4, 640, 4, "fast"),
    _c(6, 641, 4, "fast", bounds="tensor"),
    _c(4, 641, 4, "lm", outliers=0.1, mixed=True),
    _c(6, 642, 3, "lm", zmin=True),
    _c(4, 643, 3, "fast", bounds="scalar"),
    _c(6, 1024, 6, "lm", bounds="scalar", outliers=0.1),
    _c(4, 2045, 3, "lm", bounds="tensor"),
    _c(6, 2046, 3, "fast", outliers=0.1),
    _c(6, 2047, 4, "lm", mixed=True),
    _c(4, 2047, 4, "fast", zmin=True),
    _c(6, 2048, 4, "fast", bounds="tensor", zmin=True),
    _c(4, 2048, 4, "lm", outliers=0.1),
    _c(6, 2049, 4, "lm", bounds="tensor", outliers=0.1),
    _c(4, 2050, 3, "lm", bounds="scalar"),
    _c(6, 2051, 3, "fast", mixed=True),
    _c(6, 4096, 16, "lm", outliers=0.1, mixed=True),
    _c(4, 4096, 8, "fast", bounds="tensor"),
    _c(6, "epnp_max", 8, "fast", outliers=0.1),
    _c(4, 7000, 3, "lm", zmin=True),
    _c(6, 16384, 4, "lm", bounds="tensor", outliers=0.1, seed=5),
    _c(6, "split_max", 2, "lm", outliers=0.1),
]


# ------------------------------------------------------------------------------------------------ float64 references
class Ref:
    """The oracle on one case's float32 inputs, in `dtype`, on the CPU."""

    def __init__(self, c, dtype):
        cv = lambda t: t.detach().cpu().to(dtype)
        self.x3d, self.x2d, self.w2d, self.delta = cv(c["x3d"]), cv(c["x2d"]), cv(c["w2d"]), cv(c["delta"])
        bound = lambda b: cv(b) if torch.is_tensor(b) else b
        self.cam = orc.Camera(cv(c["cam_mats"]), c["z_min"], bound(c["lb"]), bound(c["ub"]))
        self.dtype = dtype

    def eval(self, pose, jac=False, clip=True):
        return orc.evaluate(self.x3d, self.x2d, self.w2d, pose.detach().cpu().to(self.dtype), self.cam, self.delta,
                            want_jac=jac, clip_jac=clip, eps_huber=HUBER_EPS)

    def cost(self, pose):
        return self.eval(pose)["cost"]

    def cov(self, pose, clip=True):
        jtj, _ = orc._normal_eq(self.eval(pose, jac=True, clip=clip))
        return torch.linalg.inv(jtj + EPS * torch.eye(jtj.shape[-1], dtype=self.dtype))

    def gn_plus(self, pose):
        """pose (+) gn_step(pose), in this precision."""
        p = pose.detach().cpu().to(self.dtype)
        return orc.pose_add(p, orc.gn_step(self.x3d, self.x2d, self.w2d, self.cam, self.delta, p, EPS))

    def fast(self, pose_init, iters):
        prm = orc.LMParams(num_iter=iters, eps=EPS)
        return orc.lm_solve(self.x3d, self.x2d, self.w2d, self.cam, self.delta, pose_init.cpu().to(self.dtype), prm,
                            fast_mode=True)

    def lm(self, pose_init, iters):
        return lm_trace(self.x3d, self.x2d, self.w2d, self.cam, self.delta, pose_init.cpu().to(self.dtype),
                        orc.LMParams(num_iter=iters, eps=EPS))


def lm_trace(x3d, x2d, w2d, cam, delta, pose_init, prm):
    """orc.lm_solve (LM mode) restated to also return what the decisions saw: every proposed pose (B, K, D), and per
    iteration (B, K) rho, cost - cost_new and model_change.  -> pose, cov, cost, dict."""
    dof = 4 if pose_init.shape[-1] == 4 else 6
    eye = torch.eye(dof, dtype=x2d.dtype)
    ev = lambda p: orc.evaluate(x3d, x2d, w2d, p, cam, delta, want_jac=True, clip_jac=True, eps_huber=HUBER_EPS)
    pose = pose_init.clone()
    cur = ev(pose)
    jtj, g = orc._normal_eq(cur)
    cost = cur["cost"]
    B = pose.shape[0]
    radius = x2d.new_full((B,), prm.initial_trust_region_radius)
    shrink = x2d.new_full((B,), 2.0)
    tr = dict(proposed=[], rho=[], decrease=[], model_change=[], cost=[])
    for _ in range(prm.num_iter):
        d = torch.diagonal(jtj, dim1=-2, dim2=-1)
        damp = d.clamp(min=prm.min_lm_diagonal, max=prm.max_lm_diagonal) / radius[:, None] + prm.eps
        step = -torch.linalg.solve(jtj + torch.diag_embed(damp), g)
        pose_new = orc.pose_add(pose, step)
        new = ev(pose_new)
        model_change = -(step * ((jtj @ step[..., None]).squeeze(-1) / 2 + g)).sum(-1)
        rho = (cost - new["cost"]) / model_change
        for k, v in (("proposed", pose_new), ("rho", rho), ("decrease", cost - new["cost"]),
                     ("model_change", model_change), ("cost", cost)):
            tr[k].append(v)
        ok = (rho >= prm.min_relative_decrease) & (model_change > 0.0)
        pose = torch.where(ok[:, None], pose_new, pose)
        grow = radius / (1.0 - (2.0 * rho - 1.0) ** 3).clamp(min=1.0 / 3.0)
        radius = torch.where(ok, grow, radius).clamp(max=prm.max_trust_region_radius, min=prm.eps)
        radius = torch.where(ok, radius, radius / shrink)
        shrink = torch.where(ok, torch.full_like(shrink, 2.0), shrink * 2.0)
        jtj_new, g_new = orc._normal_eq(new)
        jtj = torch.where(ok[:, None, None], jtj_new, jtj)
        g = torch.where(ok[:, None], g_new, g)
        cost = torch.where(ok, new["cost"], cost)
    out = {k: torch.stack(v, 1) if v else torch.zeros(B, 0, dtype=x2d.dtype) for k, v in tr.items()}
    return pose, torch.linalg.inv(jtj + prm.eps * eye), cost, out


def tie_margin(tr):
    """Per object: the least |cost - cost_new| / cost and |model_change| / cost over the float64 iterations."""
    c = tr["cost"].abs().clamp(min=1e-300)
    m = torch.minimum(tr["decrease"].abs() / c, tr["model_change"].abs() / c)
    return m.amin(1) if m.shape[1] else torch.full((m.shape[0],), float("inf"), dtype=f64)


# ------------------------------------------------------------------------------------------------ metrics (float64)
def _d(t):
    return t.detach().cpu().to(f64)


def trans_err(p, ref):
    p, ref = _d(p), _d(ref)
    return ((p[:, :3] - ref[:, :3]).norm(dim=1) / ref[:, :3].norm(dim=1).clamp(min=1e-300)).numpy()


def rot_err(p, ref):
    """Radians: the sign-free angle between unit quaternions (|qa - s qb| = 2 sin(theta / 4)), or |dyaw|."""
    p, ref = _d(p), _d(ref)
    if p.shape[1] == 4:
        d = p[:, 3] - ref[:, 3]
        return torch.atan2(torch.sin(d), torch.cos(d)).abs().numpy()
    qa = p[:, 3:] / p[:, 3:].norm(dim=1, keepdim=True)
    qb = ref[:, 3:] / ref[:, 3:].norm(dim=1, keepdim=True)
    s = torch.where((qa * qb).sum(1, keepdim=True) < 0, -1.0, 1.0).to(f64)
    return (4 * torch.asin(((qa - s * qb).norm(dim=1) / 2).clamp(max=1.0))).numpy()


def increment(start, end):
    """(B, dof): dt and the rotation increment d with end ~ start + T(q0) d (T has orthonormal columns orthogonal to
    q0, so d = T^T q1 / (q0 . q1) inverts pose_add exactly), or dyaw."""
    start, end = _d(start), _d(end)
    if start.shape[1] == 4:
        return end - start
    q0, q1 = start[:, 3:], end[:, 3:]
    d = (orc.quat_tangent_map(q0).transpose(-1, -2) @ q1[..., None]).squeeze(-1) / (q0 * q1).sum(1, keepdim=True)
    return torch.cat((end[:, :3] - start[:, :3], d), 1)


def inc_err(start, end, start_ref, end_ref, converged=False):
    """|inc - inc64| / |inc64|.  converged: the step after a finished solve is at the float32 resolution of the pose,
    so it is measured against max(|inc64|, CONVERGED_STEP * |t64|) instead."""
    a, b = increment(start, end), increment(start_ref, end_ref)
    scale = b.norm(dim=1)
    if converged:
        scale = torch.maximum(scale, CONVERGED_STEP * _d(start_ref)[:, :3].norm(dim=1))
    return ((a - b).norm(dim=1) / scale.clamp(min=1e-300)).numpy()


def check_cov(stats, what, name, got, v64, v32, k, allow=None):
    """pose_cov per object, where well_posed."""
    return check(stats, what, name, rel_err(got, v64), rel_err(v32, v64), k, REL_MIN, allow, well_posed(v64))


def rel_err(a, b):
    return bm.per_object(_d(a).reshape(a.shape[0], -1), _d(b).reshape(b.shape[0], -1))


def check(stats, what, name, err, floor, k, floor_min, allow=None, only=None):
    """err, floor (B,) -> asserts err < max(floor_min, k * floor) per object, except where `allow` (B,) is True, over
    the objects where `only` (B,) is True (all when None); records the numbers under `name`.  Returns the objects over
    the bound (B,)."""
    err, floor = np.asarray(err, np.float64), np.asarray(floor, np.float64)
    full = np.zeros(err.shape, bool)
    if only is not None:
        only = np.asarray(only, bool)
        stats[f"{name}_ill_posed_objects"] = int((~only).sum())
        if not only.any():
            return full
        err, floor = err[only], floor[only]
        allow = None if allow is None else np.asarray(allow)[only]
    assert np.isfinite(err).all(), (what, name, err)
    bound = np.maximum(floor_min, k * floor)
    over = err >= bound
    bad = np.nonzero(over & ~(np.zeros_like(over) if allow is None else allow))[0]
    assert bad.size == 0, (what, name, "objects", bad[:8].tolist(), err[bad[:8]].tolist(), bound[bad[:8]].tolist())
    stats[f"{name}_max"] = float(err.max())
    stats[f"{name}_f32_floor_max"] = float(floor.max())
    stats[f"{name}_over_bound_max"] = float((err / bound).max())
    if only is None:
        return over
    full[only] = over
    return full


def well_posed(v64):
    """(B,) bool: cond(J^T J + eps I) < COV_COND_MAX, from the float64 covariance.  Beyond it (a rank-deficient object:
    one point in 6DoF) the float32 J^T J is indefinite by more than eps, and the kernel's Cholesky -- of the
    covariance and of every Gauss-Newton step -- returns NaN; those objects are counted, not compared."""
    finite = torch.isfinite(v64).all(-1).all(-1)        # a start pose the kernel already returned as NaN
    return (finite & (torch.linalg.cond(torch.where(finite[:, None, None], v64, 1.0)) < COV_COND_MAX)).numpy()


# ------------------------------------------------------------------------------------------------ building a case
def _params(dof, z_min, **kw):
    return native.default_params(dof, z_min=float(z_min), eps=EPS, huber_eps=HUBER_EPS, **kw)


def problem(c):
    return native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])


def _iterates(c, mode):
    """Every pose at which the float64 oracle evaluates in this case's Part A and Part B: (B, P, D)."""
    r = Ref(c, f64)
    p0 = _d(c["pose_init"])
    poses = [p0[:, None]]
    fast1, _, _ = r.fast(p0, 1)
    poses.append(fast1[:, None])
    if mode == "fast":
        for k in (2, 3):
            poses.append(r.fast(p0, k)[0][:, None])
    else:
        pose, _, _, tr = r.lm(p0, 10)
        poses.append(tr["proposed"])
        poses.append(pose[:, None])
    return torch.cat(poses, 1)


def _depths(c, poses):
    zh, _ = bm.project(_d(c["x3d"]), poses.transpose(0, 1), _d(c["cam_mats"]), c["z_min"])
    return zh.permute(1, 0, 2).reshape(poses.shape[0], -1)             # (B, P * N)


def _place(c, case, poses):
    if case["zmin"]:
        zh = _depths(c, poses).reshape(1, -1)
        mid, _ = bm.widest_gap_mid(zh, bm.quantile(zh, 0.15), 0.1)
        c["z_min"] = float(np.float32(float(mid[0])))
    if case["bounds"]:
        x3d, cam = _d(c["x3d"]), _d(c["cam_mats"])
        lb, ub, _ = bm.place_bounds(x3d, poses, cam, c["z_min"], case["bounds"] == "tensor")
        dev = c["x3d"].device
        c["lb"], c["ub"] = (lb.to(dev), ub.to(dev)) if torch.is_tensor(lb) else (lb, ub)


def margins(c, case, poses):
    """Least distance of a float64 depth from z_min and of a projection from a bound, over `poses` (B, P, D)."""
    out = {}
    if case["zmin"]:
        out["zmin_margin"] = float((_depths(c, poses) - c["z_min"]).abs().min())
    if case["bounds"]:
        _, u = bm.project(_d(c["x3d"]), poses.transpose(0, 1), _d(c["cam_mats"]), c["z_min"])
        u = u.permute(1, 0, 2, 3).reshape(poses.shape[0], -1, 2)
        lo = _d(c["lb"])[:, None, :] if torch.is_tensor(c["lb"]) else torch.tensor(float(c["lb"]), dtype=f64)
        hi = _d(c["ub"])[:, None, :] if torch.is_tensor(c["ub"]) else torch.tensor(float(c["ub"]), dtype=f64)
        out["bound_margin"] = float(torch.minimum((u - lo).abs().min(), (u - hi).abs().min()))
    return out


def census(c, poses):
    """Shares of (pose, point) pairs below z_min, clamped by a bound, and on the Huber linear branch at `poses`."""
    x3d, x2d, w2d, cam = _d(c["x3d"]), _d(c["x2d"]), _d(c["w2d"]), _d(c["cam_mats"])
    zh, u = bm.project(x3d, poses.transpose(0, 1), cam, c["z_min"])
    fr = dict(below_zmin=float((zh < c["z_min"]).double().mean()), clamped=0.0)
    if c["lb"] is not None:
        lo, hi = orc._bound(_d(c["lb"]) if torch.is_tensor(c["lb"]) else c["lb"], u), \
            orc._bound(_d(c["ub"]) if torch.is_tensor(c["ub"]) else c["ub"], u)
        fr["clamped"] = float(((u < lo) | (u > hi)).any(-1).double().mean())
        u = torch.minimum(torch.maximum(u, lo), hi)
    s = ((u - x2d) * w2d).norm(dim=-1)
    fr["outlier"] = float((s > _d(c["delta"])[:, None]).double().mean())
    return fr


def build_case(case, dev, seed=None):
    dof, B, N = case["dof"], case["B"], resolve_n(case)
    seed = case["seed"] if seed is None else seed
    pc = make_problem(B, N, seed=seed + N, dof=dof, outlier_frac=case["outliers"])
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
    c.update(dof=dof, B=B, N=N, z_min=0.1, lb=None, ub=None)
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5) if N > 1 else torch.full((B,), 4.0, device=dev)
    if case["zmin"] or case["bounds"]:
        poses = _iterates(c, case["mode"])
        for _ in range(3):          # the clamps move the trajectory: place them against the union of its iterates
            _place(c, case, poses)
            new = _iterates(c, case["mode"])
            poses = torch.cat((poses, new), 1)
            m = margins(c, case, new)
            if m.get("zmin_margin", 1.0) > ZMIN_GAP and m.get("bound_margin", 1.0) > BOUND_GAP:
                break
    poses = _iterates(c, case["mode"])
    c["margins"] = margins(c, case, poses)
    c["census"] = census(c, poses)
    return c


def check_conditions(case, c):
    m, fr = c["margins"], c["census"]
    if case["zmin"]:
        assert m["zmin_margin"] > ZMIN_GAP, m
        assert 0.01 <= fr["below_zmin"] <= 0.4, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if case["bounds"]:
        assert m["bound_margin"] > BOUND_GAP, m
        assert 0.03 <= fr["clamped"] <= 0.3, fr
    if case["outliers"]:
        assert 0.01 <= fr["outlier"] <= 0.99, fr          # both Huber branches
    if case["mixed"]:
        w = c["w2d"].abs().double().mean((1, 2))
        assert float(w[0]) < 1e-2 * float(w[1:].min())


# ------------------------------------------------------------------------------------------------ Part A
def part_a_lm(c, stats, what):
    """LM mode, lm_iter = 0, every output: pose_opt is pose_init; cost_init and cost the cost at pose_init; pose_cov
    inv(J^T J + eps I) with the clipped Jacobian; pose_opt_plus pose_init (+) gn_step."""
    prob, p0 = problem(c), c["pose_init"]
    out = native.lm_solve(prob, p0, _params(c["dof"], c["z_min"], lm_iter=0), want_cov=True, want_cost=True,
                          want_plus=True, want_cost_init=True)
    assert torch.equal(out["pose_opt"], p0)
    r64, r32 = Ref(c, f64), Ref(c, torch.float32)
    c64, c32 = r64.cost(p0), r32.cost(p0)
    for name in ("cost_init", "cost"):
        # K_A = 5: five times what float32 rounding moves the same object's cost
        check(stats, what, f"A_lm0_{name}", rel_err(out[name], c64), rel_err(c32, c64), K_A, REL_MIN)
    v64, v32 = r64.cov(p0), r32.cov(p0)
    check_cov(stats, what, "A_lm0_pose_cov", out["pose_cov"], v64, v32, K_A)
    e64, e32 = r64.gn_plus(p0), r32.gn_plus(p0)
    check(stats, what, "A_lm0_plus_increment", inc_err(p0, out["pose_opt_plus"], p0, e64), inc_err(p0, e32, p0, e64),
          K_A, REL_MIN, only=well_posed(v64))
    return out


def part_a_fast(c, stats, what):
    """Fast mode, lm_iter = 1: pose_opt = pose_init (+) one undamped GN step with the UNCLIPPED Jacobian; cost and
    cost_init the cost before it; pose_cov from the J^T J before it; pose_opt_plus = pose_opt (+) gn_step (clipped)."""
    prob, p0 = problem(c), c["pose_init"]
    out = native.lm_solve(prob, p0, _params(c["dof"], c["z_min"], lm_iter=1, fast_mode=1), want_cov=True,
                          want_cost=True, want_plus=True, want_cost_init=True)
    r64, r32 = Ref(c, f64), Ref(c, torch.float32)
    (p64, v64, c64), (p32, v32, c32) = r64.fast(p0, 1), r32.fast(p0, 1)
    check(stats, what, "A_fast1_step_increment", inc_err(p0, out["pose_opt"], p0, p64), inc_err(p0, p32, p0, p64),
          K_A, REL_MIN, only=well_posed(v64))
    for name in ("cost_init", "cost"):
        check(stats, what, f"A_fast1_{name}", rel_err(out[name], c64), rel_err(c32, c64), K_A, REL_MIN)
    check_cov(stats, what, "A_fast1_pose_cov", out["pose_cov"], v64, v32, K_A)
    start = out["pose_opt"]             # the GN step of pose_opt_plus starts where the kernel's solve ended
    e64, e32 = r64.gn_plus(start), r32.gn_plus(start)
    check(stats, what, "A_fast1_plus_increment", inc_err(start, out["pose_opt_plus"], start, e64),
          inc_err(start, e32, start, e64), K_A, REL_MIN, only=well_posed(r64.cov(start)))


def part_a_evaluate(c, stats, what, s_list=(1, 128, 129, 1024)):
    """evaluate_full (residual, Jacobian with the clip on and off, cost) at pose_init; evaluate_cost on S poses around
    it; adaptive_delta."""
    prob, p0, dof = problem(c), c["pose_init"], c["dof"]
    r64, r32 = Ref(c, f64), Ref(c, torch.float32)
    for clip in (True, False):
        res, cost, jac = native.evaluate_full(prob, p0, dof, c["z_min"], HUBER_EPS, clip, True, True, True)
        e64, e32 = r64.eval(p0, jac=True, clip=clip), r32.eval(p0, jac=True, clip=clip)
        tag = "clip" if clip else "noclip"
        check(stats, what, f"A_eval_{tag}_jac", rel_err(jac, e64["jac"]), rel_err(e32["jac"], e64["jac"]), K_A, REL_MIN)
        check(stats, what, f"A_eval_{tag}_residual", rel_err(res, e64["residual"]),
              rel_err(e32["residual"], e64["residual"]), K_A, REL_MIN)
        check(stats, what, f"A_eval_{tag}_cost", rel_err(cost, e64["cost"]), rel_err(e32["cost"], e64["cost"]), K_A,
              REL_MIN)
    cost_fn = native.evaluate_cost if c["N"] <= native.max_points(dof) else native.evaluate_cost_split
    gen = torch.Generator().manual_seed(c["N"])
    for S in s_list:
        poses = _d(p0)[None].repeat(S, 1, 1)
        poses[..., :3] += 0.02 * torch.randn(S, c["B"], 3, generator=gen, dtype=f64)
        if dof == 6:
            q = poses[..., 3:] + 0.02 * torch.randn(S, c["B"], 4, generator=gen, dtype=f64)
            poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
        else:
            poses[..., 3] += 0.03 * torch.randn(S, c["B"], generator=gen, dtype=f64)
        poses = poses.float()
        got = cost_fn(prob, poses.to(p0.device), dof, c["z_min"])
        chunk = max(1, (1 << 22) // (c["B"] * c["N"]))
        c64 = torch.cat([r64.cost(poses[i:i + chunk]) for i in range(0, S, chunk)])
        c32 = torch.cat([r32.cost(poses[i:i + chunk]) for i in range(0, S, chunk)])
        # per object over its S poses
        check(stats, what, f"A_evaluate_cost_S{S}", rel_err(got.T, c64.T), rel_err(c32.T, c64.T), K_A, REL_MIN)
    d = native.adaptive_delta(c["x2d"], c["w2d"], 0.5)
    d64 = orc.adaptive_delta(_d(c["x2d"]), _d(c["w2d"]), 0.5)
    d32 = orc.adaptive_delta(c["x2d"].cpu(), c["w2d"].cpu(), 0.5)
    if c["N"] > 1:
        check(stats, what, "A_adaptive_delta", rel_err(d[:, None], d64[:, None]), rel_err(d32[:, None], d64[:, None]),
              K_A, REL_MIN)


# ------------------------------------------------------------------------------------------------ Part B
def part_b_fast(c, stats, what):
    """GN, lm_iter = 3 (the test-time path): no decisions, every object on the tight bound."""
    prob, p0 = problem(c), c["pose_init"]
    out = native.lm_solve(prob, p0, _params(c["dof"], c["z_min"], lm_iter=3, fast_mode=1), want_cov=True,
                          want_cost=True, want_plus=True, want_cost_init=True)
    r64, r32 = Ref(c, f64), Ref(c, torch.float32)
    (p64, v64, c64), (p32, v32, c32) = r64.fast(p0, 3), r32.fast(p0, 3)
    # K_B = 10: three steps, each of which passes its rounding on to the next
    check(stats, what, "B_fast3_trans", trans_err(out["pose_opt"], p64), trans_err(p32, p64), K_B, TRANS_MIN)
    check(stats, what, "B_fast3_rot", rot_err(out["pose_opt"], p64), rot_err(p32, p64), K_B, ROT_MIN)
    check(stats, what, "B_fast3_cost", rel_err(out["cost"], c64), rel_err(c32, c64), K_B, REL_MIN)
    check_cov(stats, what, "B_fast3_pose_cov", out["pose_cov"], v64, v32, K_B)
    check(stats, what, "B_fast3_cost_init", rel_err(out["cost_init"], r64.cost(p0)),
          rel_err(r32.cost(p0), r64.cost(p0)), K_A, REL_MIN)
    start = out["pose_opt"]
    e64, e32 = r64.gn_plus(start), r32.gn_plus(start)
    check(stats, what, "B_fast3_plus_increment", inc_err(start, out["pose_opt_plus"], start, e64, True),
          inc_err(start, e32, start, e64, True), K_B, REL_MIN, only=well_posed(r64.cov(start)))


def part_b_lm(c, stats, what):
    """LM, lm_iter = 10.  An object may miss the tight bound only where the float64 trajectory had a decision inside
    float32 noise (tie_margin < TIE), and then must be cost-equivalent (assert_lm_parity's clause)."""
    prob, p0 = problem(c), c["pose_init"]
    out = native.lm_solve(prob, p0, _params(c["dof"], c["z_min"], lm_iter=10), want_cov=True, want_cost=True,
                          want_plus=True, want_cost_init=True)
    r64, r32 = Ref(c, f64), Ref(c, torch.float32)
    p64, v64, c64, tr = r64.lm(p0, 10)
    p32, v32, c32, _ = r32.lm(p0, 10)
    tie = (tie_margin(tr) < TIE).numpy()
    # K_B = 10 on the tight bound; objects over it are flips
    flip = check(stats, what, "B_lm10_trans", trans_err(out["pose_opt"], p64), trans_err(p32, p64), K_B, TRANS_MIN, tie)
    flip |= check(stats, what, "B_lm10_rot", rot_err(out["pose_opt"], p64), rot_err(p32, p64), K_B, ROT_MIN, tie)
    flip |= check(stats, what, "B_lm10_cost", rel_err(out["cost"], c64), rel_err(c32, c64), K_B, REL_MIN, tie)
    flip |= check_cov(stats, what, "B_lm10_pose_cov", out["pose_cov"], v64, v32, K_B, tie)
    if flip.any():
        # a flip lands on the same cost (2e-6) with the pose within 50 times the tight bound
        pose_k, pose_r = _d(out["pose_opt"]).numpy(), p64.numpy()
        scale_tol = float(np.maximum(TRANS_MIN, K_B * trans_err(p32, p64)).max())
        frac = assert_lm_parity(pose_k[flip], _d(out["cost"]).numpy()[flip], pose_r[flip], c64.numpy()[flip],
                                scale_tol, max_flip_frac=1.0, what=what)
        assert frac <= 1.0
    stats["B_lm10_flip_rate"] = float(flip.mean())
    stats["B_lm10_tie_objects"] = int(tie.sum())
    assert flip.sum() <= max(1.0, MAX_FLIP * flip.size), (what, flip.mean())      # one object may flip at B = 1
    check(stats, what, "B_lm10_cost_init", rel_err(out["cost_init"], r64.cost(p0)),
          rel_err(r32.cost(p0), r64.cost(p0)), K_A, REL_MIN)
    start = out["pose_opt"]
    e64, e32 = r64.gn_plus(start), r32.gn_plus(start)
    check(stats, what, "B_lm10_plus_increment", inc_err(start, out["pose_opt_plus"], start, e64, True),
          inc_err(start, e32, start, e64, True), K_B, REL_MIN, only=well_posed(r64.cov(start)))


def run_case(case, dev, s_list=(1, 128, 129, 1024), record="lm_matrix"):
    c = build_case(case, dev)
    check_conditions(case, c)
    stats, what = {}, case["id"]
    part_a_lm(c, stats, what)
    part_a_fast(c, stats, what)
    part_a_evaluate(c, stats, what, s_list)
    (part_b_lm if case["mode"] == "lm" else part_b_fast)(c, stats, what)
    record_parity(f"{record}/{case['id']}", B=c["B"], N=c["N"], dof=c["dof"], mode=case["mode"],
                  bounds=case["bounds"] or "none", z_min=c["z_min"], k_part_a=K_A, k_part_b=K_B, rel_min=REL_MIN,
                  trans_min=TRANS_MIN, rot_min_rad=ROT_MIN, **c["census"], **c["margins"], **stats)


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_lm_matrix(cuda_device, case):
    run_case(case, cuda_device)


def test_every_boundary_is_in_the_matrix():
    """Each N of the axis list, every kernel boundary with N = 1, 2, 3 (mod 4) on both sides, in both DoFs."""
    ns = {(cs["dof"], cs["N"]) for cs in CASES}
    allN = {n for _, n in ns}
    assert allN >= {1, 3, 4, 7, 64, 511, 512, 513, 640, 641, 1024, 2047, 2048, 2049, 4096, "epnp_max", 7000, 16384,
                    "split_max"}
    for lo, hi in ((STAGE_MAX_N, STAGE_MAX_N + 1), (EIGHT_WARP_N - 1, EIGHT_WARP_N)):
        for dof in (4, 6):
            assert (dof, lo) in ns and (dof, hi) in ns, (dof, lo, hi)
        below = {n % 4 for n in allN if isinstance(n, int) and lo - 4 <= n <= lo}
        above = {n % 4 for n in allN if isinstance(n, int) and hi <= n <= hi + 4}
        assert below >= {1, 2, 3} and above >= {1, 2, 3}, (lo, below, above)
    for key in ("bounds", "zmin", "outliers", "mixed"):
        assert any(cs[key] for cs in CASES) and not all(cs[key] for cs in CASES)
    assert {cs["bounds"] for cs in CASES} == {None, "scalar", "tensor"}
    assert {cs["mode"] for cs in CASES} == {"lm", "fast"} and any(cs["B"] == 1 for cs in CASES)


# ------------------------------------------------------------------------------------------------ exact properties
def _slice(c, b):
    one = dict(c)
    for k in ("x3d", "x2d", "w2d", "cam_mats", "delta", "pose_init"):
        one[k] = c[k][b:b + 1].clone()
    if torch.is_tensor(c["lb"]):
        one["lb"], one["ub"] = c["lb"][b:b + 1].clone(), c["ub"][b:b + 1].clone()
    return one


def _misaligned(t):
    """A copy of t whose data starts 4 bytes past a 16-byte boundary (the plain loader)."""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    out = buf[1:1 + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 != 0
    return out


def check_exact_properties(dev, N, B=5, dof=6):
    """One output alone equals the all-outputs call; object b alone equals row b of the batch; at a staged N, a
    misaligned copy of the inputs (plain loader) equals the TMA path.  All bit for bit, LM and fast mode."""
    case = _c(dof, N, B, "lm", bounds="tensor", outliers=0.1)
    c = build_case(case, dev, seed=11)
    for mode in (dict(lm_iter=10), dict(lm_iter=3, fast_mode=1)):
        prm = _params(dof, c["z_min"], **mode)
        full = native.lm_solve(problem(c), c["pose_init"], prm, want_cov=True, want_cost=True, want_plus=True,
                               want_cost_init=True)
        only_ci = native.lm_solve(problem(c), c["pose_init"], prm, want_cost_init=True)
        assert torch.equal(only_ci["cost_init"], full["cost_init"]) and torch.equal(only_ci["pose_opt"], full["pose_opt"])
        only_plus = native.lm_solve(problem(c), c["pose_init"], prm, want_plus=True)
        assert torch.equal(only_plus["pose_opt_plus"], full["pose_opt_plus"])
        for b in (0, 2, B - 1):
            one = native.lm_solve(problem(_slice(c, b)), c["pose_init"][b:b + 1], prm, want_cov=True, want_cost=True,
                                  want_plus=True, want_cost_init=True)
            for k, v in one.items():
                assert torch.equal(v[0], full[k][b]), (mode, b, k)
        if N <= STAGE_MAX_N and N % 4 == 0:
            mis = dict(c, **{k: _misaligned(c[k]) for k in ("x3d", "x2d", "w2d")})
            got = native.lm_solve(problem(mis), c["pose_init"], prm, want_cov=True, want_cost=True, want_plus=True,
                                  want_cost_init=True)
            for k, v in got.items():
                assert torch.equal(v, full[k]), (mode, "misaligned", k)


@pytest.mark.parametrize("N", [512, 641, 2049])
def test_lm_exact_properties(cuda_device, N):
    check_exact_properties(cuda_device, N)


def _fused_lm_half(dev, N, B, split):
    case = _c(6, N, B, "lm", outliers=0.1)
    c = build_case(case, dev, seed=13)
    prm = _params(6, c["z_min"], lm_iter=10, mc_samples=64, mc_iter=4)
    solo = native.lm_solve(problem(c), c["pose_init"], prm, want_cov=True)
    fused = (native.lm_amis_fused_split if split else native.lm_amis_fused)(problem(c), c["pose_init"], prm, seed=5)
    assert torch.equal(fused["pose_opt"], solo["pose_opt"]) and torch.equal(fused["pose_cov"], solo["pose_cov"])


def test_lm_solve_equals_fused_lm_half(cuda_device):
    """lm_solve's pose_opt and pose_cov equal the LM half of lm_amis_fused at N = 2048 (8 warps) and of
    lm_amis_fused_split at N = 16384, bit for bit."""
    _fused_lm_half(cuda_device, 2048, 3, split=False)
    _fused_lm_half(cuda_device, 16384, 2, split=True)


def test_lm_kernel_variant_by_n(cuda_device):
    """The kernel each boundary N runs: <D, true, 1> up to 640, <D, false, 1> for 641 - 2047, <D, false, 8> from 2048."""
    from torch.profiler import ProfilerActivity, profile
    want = {640: "true, 1>", 641: "false, 1>", 2047: "false, 1>", 2048: "false, 8>"}
    for dof in (6, 4):
        for N, tail in want.items():
            pc = {k: v.to(cuda_device) for k, v in make_problem(2, N, seed=N, dof=dof).items()}
            prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, 4.0)
            native.lm_solve(prob, pc["pose_init"], _params(dof, 0.1, lm_iter=2))
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                native.lm_solve(prob, pc["pose_init"], _params(dof, 0.1, lm_iter=2))
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if "lm_warp_kernel" in e.name]
            assert names and all(f"lm_warp_kernel<{dof}, {tail}" in n for n in names), (dof, N, names)
