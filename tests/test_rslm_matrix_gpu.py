"""The random-sample LM initialiser against the float64 oracle per hypothesis, across its resident and cluster kernels,
subset sizes, clamps and iteration counts.

The initialiser runs in two forms: rslm_kernel (native.rslm: one CTA per object, thread <-> hypothesis, P > 128 takes
further passes of the thread loop, the mini-problem's points read out of the object's resident pair records) and, for
objects beyond one SM, rslm_refine_kernel -> cost_split_kernel -> rslm_select_kernel (native.rslm_split: one thread per
(hypothesis, object) over a grid of P B threads reading the object's global rows, the scoring on a thread-block cluster,
one thread per object keeping the cheapest).  Each case draws its subsets and starting poses with the production draw
(native.rslm_draw), and the kernel and orc.rslm_solve (oracle/pnp_oracle.py, pinned to the reference by
test_oracle_rslm_cpu.py) get the same inds / start, so no random draw enters the comparison.  The oracle runs on the same
float32 inputs in float64.

Per hypothesis (pose_all): translation |dt| / |t64|, rotation the sign-free quaternion angle or |dyaw|, each held to
max(POSE_MIN, K_POSE * floor).  The floor is an ensemble floor: the largest error against float64 of the float32 oracle
run on R_ORDERS orderings of the hypothesis' subset (identity, reversed, two seeded shuffles) -- a permutation changes
only the float32 summation order, and one float32 run can land on the float64 result by chance.

LM mode makes accept / reject decisions.  A float64 decision with |cost - cost_new|, |model_change| or |cost - cost_new
- min_relative_decrease model_change| below TIE * cost is tied: float32 rounding may take it either way.  Every tied
decision is replayed reversed (lm_trace with a `force` mask); with at most MAX_TIED_DECISIONS tied decisions in the
whole decision tree of a hypothesis (at most four branches) the kernel must match one branch within the bound above.  A
hypothesis with more is tangled, and at most MAX_TANGLED of a case with lm_iter <= 3 may be.  With lm_iter = 10 the
n = 16 mini-problems converge by the fourth iteration, and every later decision weighs a decrease of about 1e-7 of the
cost against a model change of the same size (rho near 1 in float64, float32 noise in the kernel): most hypotheses are
tangled there, and their share is recorded.  A tangled hypothesis is held to the float64 pose within the bound above
plus the summed size of its tied float64 steps (translation and rotation apart): taking or refusing one of them moves
the pose by that step.

The clamps make the mini-problem discontinuous (LM mode clips the Jacobian of a clamped point).  z_min and the bounds are
placed against the union of every hypothesis' float64 iterates; a hypothesis with a subset depth within ZMIN_GAP of z_min
or a projection within BOUND_GAP of a bound at one of its float64 iterates is counted and left out of the pose clause.

Full-set cost (cost_all) against the float64 cost at the kernel's own pose_all, for every hypothesis (tied, tangled and
clamp-excluded ones too): max(COST_MIN, K_COST * floor), floor per object = the float32 oracle's largest cost error at
that object's P poses.  Selection, exactly: pose / cost are bit copies of the pose_all / cost_all row that torch.min's
order picks (NaN first, then the smaller cost, then the earlier hypothesis); the float64 cost of that winner is within
the cost bound of the float64 minimum over the kernel's P poses; the winner is the float64 oracle's unless their float64
costs are within the cost bound or the oracle's winner is tied, tangled or clamp-excluded.

The draw's centre-based translation guess (t_out) is held to orc.center_based_init in float64 the same way, at N up to
the largest the draw accepts.
"""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
import test_lm_matrix_gpu as lmm
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

f64 = torch.float64
K_POSE = 10             # pose_all: max(POSE_MIN, K_POSE * ensemble floor) per hypothesis; an iterated solve compounds
POSE_MIN = 2e-5         # translation relative to |t64|, rotation in radians (absolute)
K_COST = 5              # cost_all: max(COST_MIN, K_COST * floor) with the floor per object
COST_MIN = 2e-6
R_ORDERS = 4            # subset orderings of the float32 ensemble
TIE = 1e-5              # a float64 decision within TIE * cost of either side is tied
MAX_TIED_DECISIONS = 2  # tied decisions in one hypothesis' decision tree beyond which it is tangled
MAX_TANGLED = 0.05      # share of the hypotheses of an LM case that may be tangled ...
MAX_TANGLED_ITERS = 3   # ... with lm_iter up to this (beyond it the mini-problems have converged: share recorded)
MAX_EXCLUDED = 0.1      # share of the hypotheses of a case that a clamp margin may leave out of the pose clause
COND_ILL = 1e6          # cond(J^T J + eps I) census threshold
EPS = 1e-5
HUBER_EPS = 1e-10
NT = 128                # threads per CTA of rslm_kernel and rslm_refine_kernel
SMEM_LIMIT = 227 * 1024  # pnp_device.cuh
ORACLE_PAIRS = 1 << 22  # (hypothesis, point) pairs per full-set oracle call: objects are run in chunks below it
BOUND_GAP = bm.BOUND_GAP
ZMIN_GAP = bm.ZMIN_GAP


# ------------------------------------------------------------------------------------------------ the cases
# form ("resident" | "split"), dof, N (an int, "max" = max_points(dof), "split_max" = max_points_split(dof)), P, n, B,
# mode ("lm" | "fast"), iters (lm_iter), bounds (None | "scalar" | "tensor"), zmin (z_min among the subset depths of
# the float64 iterates), outliers (share of points moved onto the Huber linear branch), mixed (object 0's w2d times
# 1e-3), ctas (split: cluster size, 0 = automatic), seed.
def _c(form, dof, N, P, n, B, mode, iters, bounds=None, zmin=False, outliers=0.0, mixed=False, ctas=0, seed=1):
    tag = "".join([f"{form}_d{dof}_N{N}_P{P}_n{n}_B{B}_{mode}{iters}", f"_{bounds}" if bounds else "",
                   "_zmin" if zmin else "", "_outl" if outliers else "", "_mixed" if mixed else "",
                   f"_C{ctas}" if form == "split" else ""])
    return dict(id=tag, form=form, dof=dof, N=N, P=P, n=n, B=B, mode=mode, iters=iters, bounds=bounds, zmin=zmin,
                outliers=outliers, mixed=mixed, ctas=ctas, seed=seed)


CASES = [
    # resident
    # (B = 3 put one of 387 minimal-subset hypotheses at 1.007 x its bound on the emulator build)
    _c("resident", 6, 33, 129, 3, 2, "fast", 3),
    _c("resident", 6, 33, 64, 8, 4, "lm", 3, outliers=0.1, mixed=True),
    _c("resident", 4, 33, 127, 3, 3, "fast", 1, bounds="scalar"),
    _c("resident", 4, 8, 64, 8, 3, "lm", 1),                                        # n = N = 8: the whole object
    _c("resident", 6, 256, 128, 16, 3, "lm", 10, outliers=0.1),                     # the one LM case at lm_iter = 10
    _c("resident", 4, 256, 129, 9, 3, "lm", 3, zmin=True),
    _c("resident", 6, 2047, 300, 7, 2, "fast", 10, bounds="tensor"),                # three passes of the thread loop
    _c("resident", 4, 2047, 1, 16, 4, "lm", 0),
    _c("resident", 6, "max", 64, 16, 2, "lm", 3, bounds="tensor", outliers=0.1),
    _c("resident", 4, "max", 64, 8, 2, "fast", 0),
    _c("resident", 6, 256, 257, 16, 2, "fast", 3, zmin=True),
    # split
    _c("split", 6, 16384, 64, 16, 3, "lm", 3, bounds="tensor", outliers=0.1),
    _c("split", 6, 2047, 129, 8, 3, "fast", 3, zmin=True, ctas=2),                 # P B = 387: a partial refine CTA
    _c("split", 4, 16384, 128, 16, 2, "fast", 10, bounds="scalar", ctas=8),
    _c("split", 4, "split_max", 64, 8, 2, "lm", 1, outliers=0.1),
    _c("split", 6, "split_max", 1, 3, 2, "fast", 1, ctas=8),
    _c("split", 6, 33, 257, 9, 2, "lm", 3, mixed=True, ctas=8),
    _c("split", 4, 256, 64, 3, 3, "fast", 0, ctas=2),
    _c("split", 6, 256, 129, 16, 2, "lm", 0, ctas=2),
]


def resolve_n(case):
    N = case["N"]
    if N == "max":
        return native.max_points(case["dof"])
    if N == "split_max":
        return native.max_points_split(case["dof"])
    return N


def _d(t):
    return t.detach().cpu().to(f64)


# ------------------------------------------------------------------------------------------------ the mini-problems
class Sub:
    """The P B gathered n-point mini-problems of a case in float64 (rows h B + b), as the oracle builds them."""

    def __init__(self, c, dtype=f64):
        P, B, n = c["inds"].shape
        idx = c["inds"].detach().cpu().long()[..., None]
        gather = lambda t: torch.gather(_d(t)[None].expand(P, *t.shape), 2,
                                        idx.expand(P, B, n, t.shape[-1])).reshape(P * B, n, -1).to(dtype)
        rep = lambda t: _d(t)[None].expand(P, *t.shape).reshape(P * B, *t.shape[1:]).to(dtype)
        self.x3d, self.x2d, self.w2d = gather(c["x3d"]), gather(c["x2d"]), gather(c["w2d"])
        self.cam_mats, self.delta = rep(c["cam_mats"]), rep(c["delta"])
        bound = lambda b: rep(b) if torch.is_tensor(b) else b
        self.lb, self.ub, self.z_min = bound(c["lb"]), bound(c["ub"]), c["z_min"]
        self.start = _d(c["start"]).reshape(P * B, -1).to(dtype)

    def args(self, rows=slice(None)):
        cut = lambda b: b[rows] if torch.is_tensor(b) else b
        cam = orc.Camera(self.cam_mats[rows], self.z_min, cut(self.lb), cut(self.ub))
        return self.x3d[rows], self.x2d[rows], self.w2d[rows], cam, self.delta[rows]


def lm_trace_forced(x3d, x2d, w2d, cam, delta, pose_init, prm, force=None):
    """lmm.lm_trace with the accept / reject decision of iteration k reversed where force[:, k] is True."""
    ev = lambda p: orc.evaluate(x3d, x2d, w2d, p, cam, delta, want_jac=True, clip_jac=True, eps_huber=HUBER_EPS)
    pose = pose_init.clone()
    cur = ev(pose)
    jtj, g = orc._normal_eq(cur)
    cost = cur["cost"]
    B = pose.shape[0]
    radius = x2d.new_full((B,), prm.initial_trust_region_radius)
    shrink = x2d.new_full((B,), 2.0)
    tr = dict(current=[], proposed=[], rho=[], decrease=[], model_change=[], cost=[])
    for k in range(prm.num_iter):
        d = torch.diagonal(jtj, dim1=-2, dim2=-1)
        damp = d.clamp(min=prm.min_lm_diagonal, max=prm.max_lm_diagonal) / radius[:, None] + prm.eps
        step = -torch.linalg.solve(jtj + torch.diag_embed(damp), g)
        pose_new = orc.pose_add(pose, step)
        new = ev(pose_new)
        model_change = -(step * ((jtj @ step[..., None]).squeeze(-1) / 2 + g)).sum(-1)
        rho = (cost - new["cost"]) / model_change
        for key, v in (("current", pose), ("proposed", pose_new), ("rho", rho), ("decrease", cost - new["cost"]),
                       ("model_change", model_change), ("cost", cost)):
            tr[key].append(v)
        ok = (rho >= prm.min_relative_decrease) & (model_change > 0.0)
        if force is not None:
            ok = ok ^ force[:, k]
        pose = torch.where(ok[:, None], pose_new, pose)
        grow = radius / (1.0 - (2.0 * rho - 1.0) ** 3).clamp(min=1.0 / 3.0)
        radius = torch.where(ok, grow, radius).clamp(max=prm.max_trust_region_radius, min=prm.eps)
        radius = torch.where(ok, radius, radius / shrink)
        shrink = torch.where(ok, torch.full_like(shrink, 2.0), shrink * 2.0)
        jtj_new, g_new = orc._normal_eq(new)
        jtj = torch.where(ok[:, None, None], jtj_new, jtj)
        g = torch.where(ok[:, None], g_new, g)
        cost = torch.where(ok, new["cost"], cost)
    out = {key: torch.stack(v, 1) if v else torch.zeros(B, 0, dtype=x2d.dtype) for key, v in tr.items()}
    if not tr["proposed"]:
        out["current"] = out["proposed"] = pose.new_zeros(B, 0, pose.shape[-1])
    return pose, out


def tied_decisions(tr, prm):
    """(H, K) bool: the float64 decisions within TIE * cost of going the other way (lmm.tie_margin's two criteria per
    iteration, and rho against min_relative_decrease) about a step that is not negligible.  A step shorter than
    POSE_MIN / lm_iter (translation relative to |t|, rotation in radians) is taken or not within the pose bound even if
    every later decision goes the other way too: a converged solve makes such decisions on rounding at every iteration,
    and they move nothing."""
    H, K = tr["cost"].shape
    if K == 0:
        return torch.zeros((H, 0), dtype=torch.bool)
    per_it = torch.stack([lmm.tie_margin({k: v[:, i:i + 1] for k, v in tr.items()}) for i in range(K)], 1)
    c = tr["cost"].abs().clamp(min=1e-300)
    thr = (tr["decrease"] - prm.min_relative_decrease * tr["model_change"]).abs() / c
    size = np.maximum(*step_sizes(tr))
    return (torch.minimum(per_it, thr) < TIE) & torch.from_numpy(size >= POSE_MIN / K)


def step_sizes(tr):
    """(H, K) each: every proposed float64 step's translation (relative to |t|) and rotation (radians)."""
    H, K = tr["cost"].shape
    cur, new = tr["current"].reshape(H * K, -1), tr["proposed"].reshape(H * K, -1)
    return lmm.trans_err(new, cur).reshape(H, K), lmm.rot_err(new, cur).reshape(H, K)


def lm_branches(sub, prm, base_pose, base_tr):
    """The float64 decision tree of every tied hypothesis.  -> candidate poses (H, 4, D) (NaN where a hypothesis has
    fewer branches), tied (H,), tangled (H,) bool."""
    H, D = base_pose.shape
    tied_at = tied_decisions(base_tr, prm)
    tied = tied_at.any(1)
    cands = torch.full((H, 1 << MAX_TIED_DECISIONS, D), float("nan"), dtype=f64)
    cands[:, 0] = base_pose
    count = torch.ones(H, dtype=torch.long)
    seen = {int(h): set(torch.nonzero(tied_at[h])[:, 0].tolist()) for h in torch.nonzero(tied)[:, 0]}
    tangled = {h for h, s in seen.items() if len(s) > MAX_TIED_DECISIONS}
    frontier = sorted({(h, (t,)) for h, s in seen.items() if h not in tangled for t in s})
    while frontier:
        rows = torch.tensor([h for h, _ in frontier])
        force = torch.zeros(len(frontier), prm.num_iter, dtype=torch.bool)
        for i, (_, F) in enumerate(frontier):
            force[i, list(F)] = True
        pose, tr = lm_trace_forced(*sub.args(rows), sub.start[rows], prm, force)
        t_at = tied_decisions(tr, prm)
        nxt = set()
        for i, (h, F) in enumerate(frontier):
            if h in tangled:
                continue
            cands[h, count[h]] = pose[i]
            count[h] += 1
            new = [t for t in torch.nonzero(t_at[i])[:, 0].tolist() if t > max(F)]
            seen[h] |= set(new)
            if len(seen[h]) > MAX_TIED_DECISIONS:
                tangled.add(h)
                continue
            nxt |= {(h, tuple(sorted(F + (t,)))) for t in new}
        frontier = sorted(nxt)
    tg = torch.zeros(H, dtype=torch.bool)
    tg[list(tangled)] = True
    return cands, tied, tg


def trajectories(sub, c):
    """Every pose at which the float64 mini-problems evaluate, (H, K, D), the final float64 pose (H, D) and, in LM
    mode, the trace."""
    prm = orc.LMParams(num_iter=c["iters"], eps=EPS)
    p0 = sub.start
    if c["mode"] == "lm":
        pose, tr = lm_trace_forced(*sub.args(), p0, prm)
        return torch.cat((p0[:, None], tr["proposed"], pose[:, None]), 1), pose, tr
    poses, pose = [p0], p0
    for _ in range(c["iters"]):         # one GN step at a time: the same arithmetic as lm_solve's loop
        pose, _, _ = orc.lm_solve(*sub.args(), pose, orc.LMParams(num_iter=1, eps=EPS), fast_mode=True)
        poses.append(pose)
    return torch.stack(poses, 1), pose, None


# ------------------------------------------------------------------------------------------------ the oracle
def oracle(c, inds, dtype):
    """orc.rslm_solve on the case's float32 inputs in `dtype`, objects in chunks of at most ORACLE_PAIRS (hypothesis,
    point) pairs.  lm_iter = 0 leaves every start pose as it is in both modes (the oracle's fast mode needs a step)."""
    P, B, N = c["P"], c["B"], c["N"]
    cv = lambda t: t.detach().cpu().to(dtype)
    prm = orc.LMParams(num_iter=c["iters"], eps=EPS)
    fast = c["mode"] == "fast" and c["iters"] > 0
    step = max(1, ORACLE_PAIRS // (P * N))
    parts = []
    for b0 in range(0, B, step):
        sl = slice(b0, min(B, b0 + step))
        bound = lambda b: cv(b[sl]) if torch.is_tensor(b) else b
        cam = orc.Camera(cv(c["cam_mats"][sl]), c["z_min"], bound(c["lb"]), bound(c["ub"]))
        parts.append(orc.rslm_solve(cv(c["x3d"][sl]), cv(c["x2d"][sl]), cv(c["w2d"][sl]), cam, cv(c["delta"][sl]),
                                    inds[:, sl].cpu(), cv(c["start"][:, sl]), prm, fast_mode=fast))
    return dict(hyp_pose=torch.cat([p["hyp_pose"] for p in parts], 1),
                hyp_cost=torch.cat([p["hyp_cost"] for p in parts], 1),
                winner=torch.cat([p["winner"] for p in parts], 0))


def full_cost(c, poses, dtype):
    """The oracle's full-set cost of poses (P, B, D) in `dtype`, objects in chunks."""
    P, B, N = poses.shape[0], c["B"], c["N"]
    cv = lambda t: t.detach().cpu().to(dtype)
    step = max(1, ORACLE_PAIRS // (P * N))
    out = []
    for b0 in range(0, B, step):
        sl = slice(b0, min(B, b0 + step))
        bound = lambda b: cv(b[sl]) if torch.is_tensor(b) else b
        cam = orc.Camera(cv(c["cam_mats"][sl]), c["z_min"], bound(c["lb"]), bound(c["ub"]))
        out.append(orc.evaluate(cv(c["x3d"][sl]), cv(c["x2d"][sl]), cv(c["w2d"][sl]), cv(poses[:, sl]), cam,
                                cv(c["delta"][sl]), eps_huber=HUBER_EPS)["cost"])
    return torch.cat(out, 1)


def orderings(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.arange(n), torch.arange(n).flip(0)] + [torch.randperm(n, generator=g) for _ in range(R_ORDERS - 2)]


# ------------------------------------------------------------------------------------------------ building a case
def _place(c, case, sub, iterates):
    """z_min at the widest gap near the 15 % quantile of the subset depths at every float64 iterate; bounds by
    bm.place_bounds against every iterate of every hypothesis on the object's full set."""
    P, B = c["P"], c["B"]
    if case["zmin"]:
        zh, _ = bm.project(sub.x3d, iterates.transpose(0, 1), sub.cam_mats, c["z_min"])
        zh = zh.reshape(1, -1)
        mid, _ = bm.widest_gap_mid(zh, bm.quantile(zh, 0.15), 0.1)
        c["z_min"] = float(np.float32(float(mid[0])))
    if case["bounds"]:
        K, D = iterates.shape[1], iterates.shape[2]
        per_obj = iterates.reshape(P, B, K, D).permute(1, 0, 2, 3).reshape(B, P * K, D)
        lb, ub, _ = bm.place_bounds(_d(c["x3d"]), per_obj, _d(c["cam_mats"]), c["z_min"], case["bounds"] == "tensor")
        dev = c["x3d"].device
        c["lb"], c["ub"] = (lb.to(dev), ub.to(dev)) if torch.is_tensor(lb) else (lb, ub)


def clamp_exposure(c, case, sub, iterates):
    """-> (H,) bool: a subset depth within ZMIN_GAP of z_min or a projection within BOUND_GAP of a bound at one of the
    hypothesis' float64 iterates, and the census (shares of (iterate, subset point) pairs below z_min, clamped, on the
    Huber linear branch)."""
    zh, u = bm.project(sub.x3d, iterates.transpose(0, 1), sub.cam_mats, c["z_min"])   # (K, H, n), (K, H, n, 2)
    near = ((zh - c["z_min"]).abs() < ZMIN_GAP).any(2).any(0)
    fr = dict(below_zmin=float((zh < c["z_min"]).double().mean()), clamped=0.0)
    if sub.lb is not None:
        lo, hi = orc._bound(sub.lb, u), orc._bound(sub.ub, u)
        near |= (((u - lo).abs() < BOUND_GAP) | ((u - hi).abs() < BOUND_GAP)).any(-1).any(2).any(0)
        fr["clamped"] = float(((u < lo) | (u > hi)).any(-1).double().mean())
        u = torch.minimum(torch.maximum(u, lo), hi)
    s = ((u - sub.x2d) * sub.w2d).norm(dim=-1)
    fr["outlier"] = float((s > sub.delta[:, None]).double().mean())
    return near.numpy(), fr


def build_case(case, dev):
    dof, B, P, n, N = case["dof"], case["B"], case["P"], case["n"], resolve_n(case)
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
    c.update(dof=dof, B=B, N=N, P=P, n=n, mode=case["mode"], iters=case["iters"], z_min=0.1, lb=None, ub=None)
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5)
    c["inds"], c["start"] = native.rslm_draw(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], P, n, dof,
                                             seed=case["seed"] + 101)
    if case["zmin"] or case["bounds"]:
        iterates, _, _ = trajectories(Sub(c), c)
        _place(c, case, Sub(c), iterates)
    return c


def check_conditions(case, c, fr):
    # (a case without zmin may still send a wild LM proposal below the default z_min: recorded only)
    if case["zmin"]:
        assert 0.01 <= fr["below_zmin"] <= 0.4, fr
    if case["bounds"]:
        assert 0.02 <= fr["clamped"] <= 0.4, fr
    if case["outliers"]:
        assert 0.01 <= fr["outlier"] <= 0.99, fr          # both Huber branches
    if case["mixed"]:
        w = c["w2d"].abs().double().mean((1, 2))
        assert float(w[0]) < 1e-2 * float(w[1:].min())


def problem(c, objs=slice(None)):
    cut = lambda b: b[objs] if torch.is_tensor(b) else b
    return native.Problem(c["x3d"][objs], c["x2d"][objs], c["w2d"][objs], c["cam_mats"][objs], cut(c["lb"]),
                          cut(c["ub"]), c["delta"][objs])


def params(c):
    return native.default_params(c["dof"], z_min=float(c["z_min"]), lm_iter=c["iters"],
                                 fast_mode=int(c["mode"] == "fast"), eps=EPS, huber_eps=HUBER_EPS)


def run_kernel(c, case, objs=slice(None), inds=None, start=None):
    inds = (c["inds"] if inds is None else inds)[:, objs].contiguous()
    start = (c["start"] if start is None else start)[:, objs].contiguous()
    if case["form"] == "resident":
        return native.rslm(problem(c, objs), inds, start, params(c), want_all=True)
    return native.rslm_split(problem(c, objs), inds, start, params(c), want_all=True, cluster_ctas=case["ctas"])


# ------------------------------------------------------------------------------------------------ the checks
def winner_of(cost_all):
    """torch.min's choice over the hypotheses (dim 0) of a (P, B) float32 array: the first NaN, else the first
    smallest."""
    nan = np.isnan(cost_all)
    first_nan = nan.argmax(0)
    return np.where(nan.any(0), first_nan, np.where(nan, np.inf, cost_all).argmin(0))


def conditioning(sub, pose, fast):
    """cond(J^T J + eps I) of every mini-problem at `pose` (H, D)."""
    x3d, x2d, w2d, cam, delta = sub.args()
    e = orc.evaluate(x3d, x2d, w2d, pose, cam, delta, want_jac=True, clip_jac=not fast, eps_huber=HUBER_EPS)
    jtj, _ = orc._normal_eq(e)
    return torch.linalg.cond(jtj + EPS * torch.eye(jtj.shape[-1], dtype=f64)).numpy()


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def run_case(case, dev, record="rslm_matrix"):
    c = build_case(case, dev)
    what, P, B, dof = case["id"], c["P"], c["B"], c["dof"]
    H = P * B
    stats = {}
    sub = Sub(c)
    iterates, pose64_sub, tr = trajectories(sub, c)
    exposed, fr = clamp_exposure(c, case, sub, iterates)
    check_conditions(case, c, fr)
    out = run_kernel(c, case)
    pose_all, cost_all = out["pose_all"].cpu(), out["cost_all"].cpu()
    assert torch.isfinite(pose_all).all() and torch.isfinite(cost_all).all(), what

    # ---- per-hypothesis pose
    r64 = oracle(c, c["inds"], f64)
    p64 = r64["hyp_pose"].reshape(H, -1)
    # the trace restates the oracle's solve
    assert (lmm.trans_err(pose64_sub, p64) < 1e-12).all() and (lmm.rot_err(pose64_sub, p64) < 1e-12).all(), what
    lm = c["mode"] == "lm" and c["iters"] > 0
    if lm:
        prm = orc.LMParams(num_iter=c["iters"], eps=EPS)
        cands, tied, tangled = lm_branches(sub, prm, p64, tr)
        tied_at = tied_decisions(tr, prm).numpy()
        st, sr = (s * tied_at for s in step_sizes(tr))
        st, sr = st.sum(1), sr.sum(1)                                                   # (H,)
    else:
        cands, tied, tangled = p64[:, None], torch.zeros(H, dtype=torch.bool), torch.zeros(H, dtype=torch.bool)
    tied, tangled = tied.numpy(), tangled.numpy()
    nb = cands.shape[1]
    present = torch.isfinite(cands).all(-1).numpy()                                   # (H, nb)
    err_to = lambda p, fn: np.stack([np.where(present[:, k], fn(p, torch.nan_to_num(cands[:, k])), np.inf)
                                     for k in range(nb)], 1)
    ft, fr_ = np.zeros(H), np.zeros(H)
    for r, perm in enumerate(orderings(c["n"], case["seed"])):
        p32 = oracle(c, c["inds"][..., perm], torch.float32)["hyp_pose"].reshape(H, -1)
        # against the nearest branch: a float32 run may take the other side of a tied decision
        ft = np.maximum(ft, err_to(p32, lmm.trans_err).min(1))
        fr_ = np.maximum(fr_, err_to(p32, lmm.rot_err).min(1))
    kp = pose_all.reshape(H, -1)
    et, er = err_to(kp, lmm.trans_err), err_to(kp, lmm.rot_err)
    bt, br = np.maximum(POSE_MIN, K_POSE * ft), np.maximum(POSE_MIN, K_POSE * fr_)
    best = np.argmin(np.maximum(et / bt[:, None], er / br[:, None]), 1)
    rows = np.arange(H)
    held = ~exposed & ~tangled
    lmm.check(stats, what, "pose_trans", et[rows, best], ft, K_POSE, POSE_MIN, only=held)
    lmm.check(stats, what, "pose_rot", er[rows, best], fr_, K_POSE, POSE_MIN, only=held)
    loose = tangled & ~exposed
    if loose.any():
        # against the float64 pose: the bound above plus the summed size of the hypothesis' tied steps
        ratio = np.maximum(et[:, 0] / (bt + st), er[:, 0] / (br + sr))[loose]
        assert np.isfinite(ratio).all() and (ratio < 1.0).all(), \
            (what, "tangled", np.nonzero(loose)[0][ratio >= 1.0][:8].tolist(), ratio[ratio >= 1.0][:8].tolist())
        stats.update(tangled_pose_over_bound_max=float(ratio.max()),
                     tangled_tied_steps_trans_median=float(np.median(st[loose])),
                     tangled_tied_steps_rot_median=float(np.median(sr[loose])))
    stats.update(pose_held_hypotheses=int(held.sum()), tangled_held_hypotheses=int(loose.sum()),
                 tied_share=float(tied.mean()), tangled_share=float(tangled.mean()),
                 clamp_excluded_share=float(exposed.mean()), other_branch_matched=int((best > 0)[held].sum()),
                 pose_floor_trans_median=float(np.median(ft)), pose_floor_rot_median=float(np.median(fr_)))
    if c["mode"] == "lm" and c["iters"] <= MAX_TANGLED_ITERS:
        assert tangled.mean() <= MAX_TANGLED, (what, "tangled", float(tangled.mean()))
    assert exposed.mean() <= MAX_EXCLUDED, (what, "clamp-excluded", float(exposed.mean()))
    cond = conditioning(sub, p64, c["mode"] == "fast")
    stats.update(cond_median=float(np.median(cond)), cond_max=float(cond.max()),
                 cond_ill_share=float((cond > COND_ILL).mean()))

    # ---- full-set cost at the kernel's own poses
    c64 = full_cost(c, pose_all, f64)
    c32 = full_cost(c, pose_all, torch.float32)
    rel_c = lambda a, b: ((_d(a) - b).abs() / b.abs()).numpy()
    cerr = rel_c(cost_all, c64)                                                       # (P, B)
    cfloor = rel_c(c32, c64).max(0)                                                   # per object
    lmm.check(stats, what, "cost", cerr.reshape(-1), np.broadcast_to(cfloor, (P, B)).reshape(-1), K_COST, COST_MIN)
    cbound = np.maximum(COST_MIN, K_COST * cfloor)

    # ---- selection
    ca = cost_all.numpy()
    win = torch.from_numpy(winner_of(ca))
    objs = torch.arange(B)
    assert torch.equal(bits(out["pose"]), bits(pose_all[win, objs])), what
    assert torch.equal(bits(out["cost"]), bits(cost_all[win, objs])), what
    c64n = c64.numpy()
    lo64 = c64n.min(0)
    assert ((c64n[win, objs] - lo64) / lo64 < cbound).all(), (what, "winner's float64 cost")
    win, objs = win.numpy(), objs.numpy()
    w64 = r64["winner"].numpy()
    h64 = r64["hyp_cost"].numpy()
    agree = win == w64
    near = np.abs(h64[win, objs] - h64[w64, objs]) / np.abs(h64[w64, objs]) < cbound
    # the oracle's winner may have had a decision go the other way in float32, or a clamp within rounding
    unsure = (tied | tangled | exposed).reshape(P, B)
    excused = near | unsure[w64, objs]
    assert (agree | excused).all(), (what, "winners", win.tolist(), w64.tolist())
    stats["winner_agreement"] = float(agree.mean())
    record_parity(f"{record}/{what}", form=case["form"], dof=dof, N=c["N"], P=P, n=c["n"], B=B, mode=c["mode"],
                  lm_iter=c["iters"], cluster_ctas=case["ctas"] if case["form"] == "split" else None,
                  bounds=case["bounds"] or "none", z_min=c["z_min"], k_pose=K_POSE, pose_min=POSE_MIN, k_cost=K_COST,
                  cost_min=COST_MIN, r_orders=R_ORDERS, tie=TIE, **fr, **stats)
    return stats


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_rslm_matrix(cuda_device, case):
    run_case(case, cuda_device)


def test_every_boundary_is_in_the_matrix():
    """Both forms in both DoFs, split cluster sizes 0 / 2 / 8, P on both sides of every thread-loop pass, minimal / odd /
    whole-object subsets, the N axis, a refine grid that does not fill its last CTA, lm_iter 0 / 1 / 3 / 10 in both
    modes, every clamp."""
    for form in ("resident", "split"):
        assert {cs["dof"] for cs in CASES if cs["form"] == form} == {4, 6}, form
    assert {cs["ctas"] for cs in CASES if cs["form"] == "split"} >= {0, 2, 8}
    ps = {cs["P"] for cs in CASES}
    assert {1, 64, 127, 128, 129} <= ps and any(p > 2 * NT for p in ps)
    for form in ("resident", "split"):
        assert any(cs["P"] > NT for cs in CASES if cs["form"] == form)
    ns = {cs["n"] for cs in CASES}
    assert {3, 8, 16} <= ns and any(n % 2 for n in ns if n > 3)
    assert all(cs["mode"] == "fast" for cs in CASES if cs["n"] == 3 and cs["dof"] == 6)
    assert any(cs["n"] == cs["N"] for cs in CASES)
    Ns = {(cs["form"], cs["N"]) for cs in CASES}
    assert {("resident", N) for N in (33, 256, 2047, "max")} <= Ns
    assert {("split", N) for N in (16384, "split_max")} <= Ns
    assert any(isinstance(cs["N"], int) and cs["N"] % 2 for cs in CASES if cs["form"] == "split")
    assert any(cs["P"] * cs["B"] % NT for cs in CASES if cs["form"] == "split")
    for mode in ("lm", "fast"):
        assert {cs["iters"] for cs in CASES if cs["mode"] == mode} >= {0, 1, 3, 10}, mode
    lm_long = [cs for cs in CASES if cs["mode"] == "lm" and cs["iters"] > 3]
    assert all(cs["n"] >= 6 for cs in CASES if cs["mode"] == "lm") and len(lm_long) == 1 and lm_long[0]["n"] == 16
    assert {cs["bounds"] for cs in CASES} == {None, "scalar", "tensor"}
    for key in ("zmin", "outliers", "mixed"):
        assert any(cs[key] for cs in CASES) and not all(cs[key] for cs in CASES)


# ------------------------------------------------------------------------------------------------ exact properties
def check_exact_properties(case, dev):
    """An object alone equals its row of the batch, bit for bit; with each object's winner swapped into hypothesis 0,
    hypothesis 0 is refined to the same bits and wins."""
    c = build_case(case, dev)
    full = run_kernel(c, case)
    B, P = c["B"], c["P"]
    for b in (0, B - 1):
        one = run_kernel(c, case, slice(b, b + 1))
        for k in ("pose_all", "cost_all"):
            assert torch.equal(bits(one[k][:, 0]), bits(full[k][:, b])), (case["id"], b, k)
        for k in ("pose", "cost"):
            assert torch.equal(bits(one[k][0]), bits(full[k][b])), (case["id"], b, k)
    win = torch.from_numpy(winner_of(full["cost_all"].cpu().numpy()))
    inds, start = c["inds"].clone(), c["start"].clone()
    for b in range(B):
        for h, src in ((0, int(win[b])), (int(win[b]), 0)):
            inds[h, b], start[h, b] = c["inds"][src, b], c["start"][src, b]
    dup = run_kernel(c, case, inds=inds, start=start)
    objs = torch.arange(B)
    assert torch.equal(bits(dup["pose_all"][0]), bits(full["pose_all"][win, objs]))
    assert (winner_of(dup["cost_all"].cpu().numpy()) == 0).all(), case["id"]
    assert torch.equal(bits(dup["pose"]), bits(dup["pose_all"][0])) and torch.equal(bits(dup["cost"]),
                                                                                     bits(dup["cost_all"][0]))


@pytest.mark.parametrize("idx", [1, 16])
def test_object_alone_equals_its_row(cuda_device, idx):
    check_exact_properties(CASES[idx], cuda_device)


# ------------------------------------------------------------------------------------------------ the translation guess
def draw_max_n(n):
    """The largest N rslm_draw accepts with n-point subsets: its weights (N rounded up to 4 floats) and n keys and
    indices per thread, plus 2 KB of static shared memory, within SMEM_LIMIT."""
    return (SMEM_LIMIT - 2048 - n * NT * 8) // 16 * 4


def center_guess(x2d, x3d, cam_mats, dof, dtype, perm=None):
    """orc.center_based_init in `dtype`, the points taken in the order `perm`."""
    cv = lambda t: t.detach().cpu().to(dtype)
    x2d, x3d = cv(x2d), cv(x3d)
    if perm is not None:
        x2d, x3d = x2d[:, perm], x3d[:, perm]
    return orc.center_based_init(x2d, x3d, orc.Camera(cv(cam_mats)), dof)


def check_translation_guess(dev, dof, sizes, n=16, B=3, record="rslm_matrix"):
    """t_out against the float64 centre-based guess, max(POSE_MIN, K_POSE * floor) per object, floor the float32 oracle
    on R_ORDERS orderings of the points.  Object 1's 2D points lie near a horizontal line (their y spread 1e-2 of the
    others': a small ray spread in y, what the 4DoF depth divides by); object 2's are shrunk to 1e-2 of their spread
    about their mean in both directions (a small ray spread in x and y, what the 6DoF depth divides by)."""
    for N in sizes:
        pc = make_problem(B, N, seed=N + dof, dof=dof)
        x2d = pc["x2d"]
        x2d[1, :, 1] = x2d[1, :, 1].mean() + 1e-2 * (x2d[1, :, 1] - x2d[1, :, 1].mean())
        x2d[2] = x2d[2].mean(0) + 1e-2 * (x2d[2] - x2d[2].mean(0))
        d = {k: v.to(dev) for k, v in pc.items()}
        _, _, t = native.rslm_draw(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], 4, n, dof, seed=N, want_t=True)
        t64 = center_guess(d["x2d"], d["x3d"], d["cam_mats"], dof, f64)
        g = torch.Generator().manual_seed(N)
        perms = [None, torch.arange(N).flip(0)] + [torch.randperm(N, generator=g) for _ in range(R_ORDERS - 2)]
        floor = np.max([lmm.trans_err(center_guess(d["x2d"], d["x3d"], d["cam_mats"], dof, torch.float32, pm), t64)
                        for pm in perms], 0)
        stats = {}
        lmm.check(stats, f"t_out d{dof} N{N}", "t_out", lmm.trans_err(t, t64), floor, K_POSE, POSE_MIN)
        record_parity(f"{record}/t_out/d{dof}_N{N}", k=K_POSE, min=POSE_MIN, **stats)


@pytest.mark.parametrize("dof", [6, 4])
def test_translation_guess_at_production_sizes(cuda_device, dof):
    n = 16
    n_max = draw_max_n(n)
    check_translation_guess(cuda_device, dof, (256, 7000, 16384, n_max), n)
    # one point more is refused
    B, dev = 2, cuda_device
    z = lambda k: torch.ones(B, n_max + 1, k, device=dev)
    with pytest.raises(native.NativeError):
        native.rslm_draw(z(3), z(2), z(2), torch.eye(3, device=dev).expand(B, 3, 3).contiguous(), 4, n, dof)
