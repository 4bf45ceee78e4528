"""The second-order and forward-mode kernels against float64 across their tiles, launch paths, Hessian blocks and clamps.

Three entry points, five kernels:
  cost_hvp      cost_hvp_point_kernel (thread <-> point, poses staged in tiles of HVP_POSE_TILE = 128) for the point,
                delta and camera rows; cost_hvp_pose_kernel (thread <-> pose, B x ceil(P / NT) CTAs, a serial sum over the
                points) for the pose rows and d cost_p . v.
  gn_plus_hvp   gn_plus_hvp_kernel (one CTA per object, thread <-> point).
  evaluate_jvp  evaluate_jvp_kernel (one CTA per (pose, object), thread <-> point); evaluate_jvp_cost_kernel (thread <->
                pose, a serial sum over the points) when only the cost is asked for and S >= JVP_POSE_MAJOR_MIN_S = 64.

The matrix puts N on both sides of the thread loop (NT = 128) and at the largest N the calls take, P on both sides of
one and two pose tiles and at the Monte-Carlo loss's 513 poses, and S on both sides of the pose-major switch, in both
DoFs, unbounded, with scalar and with per-object bounds, with depths below z_min, and with both Huber branches mixed and
alone.  The reference is the oracle's float64 double backward (test_cost_hvp_gpu.oracle_hvp,
test_gn_plus_hvp_gpu.oracle_hvp) or forward-mode derivative (test_evaluate_jvp_gpu.oracle_jvp), run in chunks of
(object, pose) pairs at the large sizes: H v is linear in the upstream gradient, so the point, delta and camera rows sum
over pose chunks and the pose rows are per pose.

Bound, per object and output (per pose and object for the pose rows and the JVP's residual and Jacobian):
max|a - b| / max|b| < max(REL_MIN, K_FLOOR * floor), floor = the largest error of the same oracle in float32 over ORDERS
orders of the points (the kernels' serial sums over thousands of points against torch's pairwise sums).  Rows that
float64 gives as exactly zero must come back within ZERO_REL of the output's largest entry under the full tangent.
Objects whose Gauss-Newton system has cond(H + eps I) > COND_MAX are left out of the gn_plus_hvp comparison, as in
test_gn_plus_hvp_gpu.py.  Each case asserts the clamps and Huber branches it claims and its margins from them, and
records what it measured through record_parity.  Some cases also run every tangent part alone (block by block), so
that a small wrong block is not hidden in the sum of the others."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
import test_cost_hvp_gpu as hv
import test_evaluate_jvp_gpu as jv
import test_gn_plus_hvp_gpu as gp
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp_b200 import native

pytestmark = pytest.mark.gpu

NT = 128                    # threads per CTA (pnp_device.cuh)
HVP_POSE_TILE = 128         # poses per shared-memory tile of cost_hvp_point_kernel (pnp_kernels.cu)
JVP_POSE_MAJOR_MIN_S = 64   # least S at which a cost-only evaluate_jvp runs evaluate_jvp_cost_kernel (pnp_kernels.cu)
REL_MIN, K_FLOOR = hv.REL_MIN, hv.K_FLOOR
ORDERS = gp.ORDERS
CHUNK = bm.CHUNK            # (pose, point) pairs per oracle call
ZERO_REL = 1e-6             # |a| of a row float64 gives as zero, relative to the output's largest entry
POINTS = ("x3d", "x2d", "w2d")
JVP_WANT = dict(residual=(True, False, False), jac=(False, True, False), cost=(False, False, True),
                all=(True, True, True))


def resolve_n(case):
    return native.max_points_split(case["dof"]) if case["N"] == "max" else case["N"]


def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def case_id(cs):
    poses = {"cost": "P", "jvp": "S", "gn": ""}[cs["entry"]]
    parts = [cs["entry"], f"d{cs['dof']}", f"N{cs['N']}"] + ([f"{poses}{cs['P']}"] if poses else []) + [f"B{cs['B']}"]
    parts += [cs[k] for k in ("bounds",) if cs.get(k)] + [k for k in ("zmin",) if cs.get(k)]
    parts += [cs["branch"]] if cs.get("branch", "mixed") != "mixed" else []
    if cs["entry"] == "jvp":
        parts += [cs["want"]] + ([] if cs.get("clip", True) else ["noclip"])
    return "_".join(str(p) for p in parts + (["blocks"] if cs.get("blocks") else []))


def kernels_of(cs):
    """The kernels a case launches."""
    if cs["entry"] == "cost":
        return {"cost_hvp_point_kernel"} | ({"cost_hvp_pose_kernel"} if cs["P"] > 0 else set())
    if cs["entry"] == "gn":
        return {"gn_plus_hvp_kernel"}
    if cs["P"] == 0:
        return set()
    pose_major = cs["want"] == "cost" and cs["P"] >= JVP_POSE_MAJOR_MIN_S
    return {"evaluate_jvp_cost_kernel" if pose_major else "evaluate_jvp_kernel"}


# ------------------------------------------------------------------------------------------------ cases
def _c(entry, dof, N, P, B, bounds=None, zmin=False, branch="mixed", blocks=False, want="all", clip=True):
    cs = dict(entry=entry, dof=dof, N=N, P=P, B=B, bounds=bounds, zmin=zmin, branch=branch, blocks=blocks, want=want,
              clip=clip)
    cs["id"] = case_id(cs)
    return cs


COST_CASES = [
    # the point-major axes: N against the thread loop and the largest N, P against the pose tiles
    _c("cost", 6, 1, 513, 3, "tensor", branch="inlier"),
    _c("cost", 6, 127, 128, 3, "scalar"),
    _c("cost", 6, 128, 129, 3, "tensor", zmin=True),
    _c("cost", 6, 129, 127, 3),
    _c("cost", 6, 129, 0, 3),
    _c("cost", 6, 128, 1, 4, branch="outlier"),
    _c("cost", 6, 2048, 256, 2, "tensor"),
    _c("cost", 6, 16384, 3, 2, "scalar", zmin=True),
    _c("cost", 6, "max", 1, 2, "tensor", zmin=True),
    # the pose-major kernel's serial sums at the large N
    _c("cost", 6, 16384, 257, 2),
    _c("cost", 6, 16384, 513, 2),                   # the Monte-Carlo loss: 512 samples and cost_init
    _c("cost", 6, "max", 129, 2),
    _c("cost", 4, 1, 257, 3, branch="outlier"),
    _c("cost", 4, 127, 129, 3, "tensor"),
    _c("cost", 4, 128, 127, 3, zmin=True),
    _c("cost", 4, 129, 128, 3, "scalar"),
    _c("cost", 4, 128, 0, 2),
    _c("cost", 4, 129, 1, 4, branch="inlier"),
    _c("cost", 4, 2048, 256, 2, "scalar"),
    _c("cost", 4, 16384, 3, 2, "tensor"),
    _c("cost", 4, "max", 1, 2, "scalar", zmin=True),
    _c("cost", 4, 16384, 513, 2),
    _c("cost", 4, 2048, 513, 2),
    _c("cost", 4, "max", 128, 2),
    # every tangent part alone
    _c("cost", 6, 129, 3, 3, blocks=True),
    _c("cost", 6, 128, 5, 3, "scalar", blocks=True),
    _c("cost", 6, 127, 4, 3, "tensor", zmin=True, blocks=True),
    _c("cost", 4, 129, 3, 3, blocks=True),
    _c("cost", 4, 128, 5, 3, "scalar", blocks=True),
    _c("cost", 4, 127, 4, 3, "tensor", zmin=True, blocks=True),
]

GN_CASES = [
    _c("gn", 6, 5, 1, 4),
    _c("gn", 6, 127, 1, 4, "scalar"),
    _c("gn", 6, 128, 1, 4, "tensor", zmin=True),
    _c("gn", 6, 129, 1, 4, branch="inlier"),
    _c("gn", 6, 129, 1, 4, "tensor", branch="outlier"),
    _c("gn", 6, 2048, 1, 3, "tensor"),
    _c("gn", 6, 16384, 1, 2, "scalar"),
    _c("gn", 6, "max", 1, 2, zmin=True),
    _c("gn", 4, 5, 1, 4, "tensor"),
    _c("gn", 4, 127, 1, 4),
    _c("gn", 4, 128, 1, 4, "scalar", zmin=True),
    _c("gn", 4, 129, 1, 4, "tensor", branch="inlier"),
    _c("gn", 4, 129, 1, 4, branch="outlier"),
    _c("gn", 4, 2048, 1, 3, zmin=True),
    _c("gn", 4, 16384, 1, 2, "tensor"),
    _c("gn", 4, "max", 1, 2, "scalar"),
    _c("gn", 6, 128, 1, 3, blocks=True),
    _c("gn", 6, 129, 1, 3, "scalar", blocks=True),
    _c("gn", 6, 127, 1, 3, "tensor", zmin=True, blocks=True),
    _c("gn", 4, 128, 1, 3, blocks=True),
    _c("gn", 4, 129, 1, 3, "scalar", blocks=True),
    _c("gn", 4, 127, 1, 3, "tensor", zmin=True, blocks=True),
]

JVP_CASES = [
    _c("jvp", 6, 129, 0, 3, want="all"),
    _c("jvp", 6, 1, 1, 4, branch="outlier", want="all"),
    _c("jvp", 6, 300, 63, 3, "scalar", want="cost"),            # the last S of the point-major kernel ...
    _c("jvp", 6, 300, 64, 3, "scalar", want="cost"),            # ... and the first of the pose-major one
    _c("jvp", 6, 128, 127, 2, "tensor", zmin=True, want="residual"),
    _c("jvp", 6, 127, 128, 2, zmin=True, want="jac", clip=False),
    _c("jvp", 6, 129, 129, 2, "tensor", zmin=True, want="cost"),
    _c("jvp", 6, 129, 513, 2, branch="inlier", want="all"),
    _c("jvp", 6, 16384, 513, 2, want="cost"),                   # the layer's forward mode of the Monte-Carlo loss
    _c("jvp", 6, 2048, 64, 2, "tensor", want="cost"),
    _c("jvp", 4, 129, 0, 2, want="cost"),
    _c("jvp", 4, 1, 1, 4, branch="inlier", want="all", clip=False),
    _c("jvp", 4, 257, 63, 3, want="cost"),
    _c("jvp", 4, 257, 64, 3, want="cost"),
    _c("jvp", 4, 127, 127, 2, "scalar", want="jac"),
    _c("jvp", 4, 128, 128, 2, "tensor", zmin=True, want="all", clip=False),
    _c("jvp", 4, 129, 129, 2, branch="outlier", want="residual"),
    _c("jvp", 4, 129, 513, 2, "scalar", zmin=True, want="cost"),
    _c("jvp", 4, 16384, 513, 2, want="cost"),
    _c("jvp", 6, 128, 3, 3, blocks=True, want="all"),
    _c("jvp", 6, 129, 2, 3, "scalar", blocks=True, want="all", clip=False),
    _c("jvp", 6, 127, 3, 3, "tensor", zmin=True, blocks=True, want="all"),
    _c("jvp", 4, 128, 3, 3, blocks=True, want="all"),
    _c("jvp", 4, 129, 2, 3, "scalar", blocks=True, want="all"),
    _c("jvp", 4, 127, 3, 3, "tensor", zmin=True, blocks=True, want="all", clip=False),
]

CASES = COST_CASES + GN_CASES + JVP_CASES


# ------------------------------------------------------------------------------------------------ building a case
def census(c, poses_pb):
    """float64 shares and margins of every (pose, point) pair, poses (P, B, D), and the residual norms (P, B, N)."""
    d = torch.float64
    zh, u = bm.project(c["x3d"].to(d), poses_pb.to(d), c["cam_mats"].to(d), c["z_min"])
    if zh.numel() == 0:
        return {}, zh
    fr = dict(below_zmin=float((zh < c["z_min"]).double().mean()), zmin_margin=float((zh - c["z_min"]).abs().min()),
              clamped=0.0)
    if c["lb"] is not None:
        lo, hi = orc._bound(c["lb"].to(d), u), orc._bound(c["ub"].to(d), u)
        fr["bound_margin"] = min(float((u - lo).abs().min()), float((u - hi).abs().min()))
        uc = torch.minimum(torch.maximum(u, lo), hi)
        fr["clamped"] = float((uc != u).any(-1).double().mean())
        u = uc
    return fr, ((u - c["x2d"].to(d)) * c["w2d"].to(d)).norm(dim=-1)


def set_delta(c, s, branch):
    """mixed: the middle of the widest gap between the object's residual norms within 25 % of their 90 % quantile (with
    millions of pairs a fixed delta would have some norm within float32 rounding of it); inlier: twice the object's
    largest norm; outlier: half its smallest."""
    if branch == "mixed":
        sb = s.transpose(0, 1).reshape(s.shape[1], -1)
        target = bm.quantile(sb, 0.9)
        c["delta"] = torch.cat([bm.widest_gap_mid(sb[b:b + 1], target[b:b + 1], 0.25 * float(target[b]))[0]
                                for b in range(sb.shape[0])]).float()
    elif branch == "inlier":
        c["delta"] = (2.0 * s.amax((0, 2))).float()
    else:
        c["delta"] = (0.5 * s.amin((0, 2))).float()


def huber_census(fr, s, delta):
    dl = delta.double()[None, :, None]
    fr.update(outlier=float((s > dl).double().mean()), huber_gap=float(((s - dl).abs() / dl).min()))


def place_bounds(c, poses_bp, kind, gen):
    B = c["x3d"].shape[0]
    dev = c["x3d"].device
    lb, ub, _ = bm.place_bounds(c["x3d"], poses_bp, c["cam_mats"], c["z_min"], kind == "tensor")
    full = lambda b: b.to(dev) if torch.is_tensor(b) else torch.full((B, 2), float(b), device=dev)
    c["lb"], c["ub"] = full(lb), full(ub)
    c["t"]["lb"], c["t"]["ub"] = (torch.randn(B, 2, generator=gen).to(dev) for _ in range(2))


def build(cs, dev, seed=5):
    """-> the case's inputs (the builders of test_cost_hvp_gpu / test_gn_plus_hvp_gpu / test_evaluate_jvp_gpu) and its
    census."""
    N, dof, B, P = resolve_n(cs), cs["dof"], cs["B"], cs["P"]
    outliers = 0.2 if cs["branch"] == "mixed" else 0.0
    gen = torch.Generator().manual_seed(seed + 7)
    if cs["entry"] == "gn":
        c = gp.build_case(dof, N, B, dev, zmin=cs["zmin"], seed=seed, outliers=outliers)
        poses_bp = c["pose"][:, None]
    else:
        c = hv.build_case(dof, N, P, B, dev, zmin=cs["zmin"], seed=seed, outliers=outliers)
        poses_bp = c["poses"]
    if cs["bounds"]:
        place_bounds(c, poses_bp, cs["bounds"], gen)
    fr, s = census(c, poses_bp.transpose(0, 1))
    if s.numel():
        set_delta(c, s, cs["branch"])
        huber_census(fr, s, c["delta"])
    else:                                           # no pose: no pair
        c["delta"] = orc.adaptive_delta(c["x2d"], c["w2d"], 0.1)
    if cs["entry"] == "jvp":
        c["poses"] = c["poses"].transpose(0, 1).contiguous()
        c["t"]["pose"] = c["t"]["pose"].transpose(0, 1).contiguous()
        c["S"], c["clip"] = P, cs["clip"]
    return c, fr


def check_census(cs, fr):
    """The clamps and branches the case claims happen, and every pair keeps its margin from them."""
    if "outlier" not in fr:
        return
    assert fr["huber_gap"] > hv.HUBER_GAP, fr
    if cs["zmin"]:
        assert fr["below_zmin"] > 0.01 and fr["zmin_margin"] > bm.ZMIN_GAP, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if cs["bounds"]:
        assert fr["clamped"] > 0.01 and fr["bound_margin"] > bm.BOUND_GAP, fr
    if cs["branch"] == "mixed":
        assert 0.01 < fr["outlier"] < 0.99, fr
    else:
        assert fr["outlier"] == (1.0 if cs["branch"] == "outlier" else 0.0), fr


# ------------------------------------------------------------------------------------------------ chunked oracles
def pair_chunks(B, P, N):
    ob = max(1, min(B, CHUNK // max(1, N * P)))
    pp = max(1, min(P, CHUNK // (N * ob)))
    for b0 in range(0, B, ob):
        for p0 in range(0, P, pp):
            yield slice(b0, min(B, b0 + ob)), slice(p0, min(P, p0 + pp))


def _objects(c, sb):
    out = dict(c)
    for k in ("x3d", "x2d", "w2d", "cam_mats", "delta", "lb", "ub"):
        if c[k] is not None:
            out[k] = c[k][sb]
    return out


def _permuted(c, t, perm):
    if perm is None:
        return c, t
    c = dict(c, **{k: c[k][:, perm] for k in POINTS})
    return c, {k: (v[:, perm] if k in POINTS else v) for k, v in t.items()}


def cost_oracle(c, dtype, t, perm=None):
    """hv.oracle_hvp over (object, pose) chunks, the points in the order `perm` (outputs in the original order)."""
    c, t = _permuted(c, t, perm)
    B, P, N = c["up"].shape[0], c["up"].shape[1], c["x3d"].shape[1]
    out = {}
    for sb, sp in pair_chunks(B, P, N):
        sub = dict(_objects(c, sb), poses=c["poses"][sb, sp], up=c["up"][sb, sp])
        r = hv.oracle_hvp(sub, dtype, t={k: (v[sb, sp] if k == "pose" else v[sb]) for k, v in t.items()})
        for k, v in r.items():
            per_pose = k in ("pose", "grad")
            if k not in out:
                out[k] = torch.zeros(((B, P) if per_pose else (B,)) + tuple(v.shape[2 if per_pose else 1:]),
                                     dtype=dtype, device=v.device)
            if per_pose:
                out[k][sb, sp] = v
            else:
                out[k][sb] += v
    return _unpermute(out, perm, lambda k: k in POINTS)


def _unpermute(out, perm, is_point):
    if perm is None:
        return out
    inv = torch.argsort(perm)
    return {k: (v[:, inv.to(v.device)] if is_point(k) else v) for k, v in out.items()}


def jvp_oracle(c, dtype, t, want, perm=None):
    """jv.oracle_jvp over (pose, object) chunks; only the outputs in `want` are kept."""
    c, t = _permuted(c, t, perm)
    S, B, N = c["poses"].shape[0], c["x3d"].shape[0], c["x3d"].shape[1]
    keep = [k for k, w in zip(jv.OUTPUTS, want) if w]
    out = {}
    for sb, sp in pair_chunks(B, S, N):
        sub = dict(_objects(c, sb), poses=c["poses"][sp, sb])
        r = jv.oracle_jvp(sub, dtype, t={k: (v[sp, sb] if k == "pose" else v[sb]) for k, v in t.items()})
        for k in keep:
            if k not in out:
                out[k] = torch.zeros((S, B) + tuple(r[k].shape[2:]), dtype=dtype, device=r[k].device)
            out[k][sp, sb] = r[k]
    if perm is None:
        return out
    inv = torch.argsort(perm)
    for k in ("residual", "jac"):
        if k in out:
            v = out[k]
            v = v.reshape(S, B, N, 2, *v.shape[3:])[:, :, inv.to(v.device)]
            out[k] = v.reshape(S, B, 2 * N, *v.shape[4:])
    return out


def floors(oracle, ref64, lead, N):
    """Per output: the largest relative error of the float32 oracle over ORDERS orders of the points (first the
    identity), row by row."""
    out = {}
    for s in range(ORDERS):
        perm = None if s == 0 else torch.randperm(N, generator=torch.Generator().manual_seed(s))
        r = oracle(torch.float32, perm)
        for k, b in ref64.items():
            e = hv.rel_rows(r[k], b, lead(k))
            out[k] = e if k not in out else np.maximum(out[k], e)
    return out


# ------------------------------------------------------------------------------------------------ comparing
def row_max(x, lead):
    x = x.detach().double().abs().cpu()
    return x.reshape(x.shape[:lead] + (-1,)).amax(-1).numpy() if x.numel() else np.zeros(x.shape[:lead])


def compare(got, ref64, floor, lead, what, scale=None, ok=None):
    """Every row of every output within max(REL_MIN, K_FLOOR * floor); rows float64 gives as zero within ZERO_REL of
    the output's largest entry under the full tangent (`scale`, by default ref64 itself).  ok: objects compared.
    Returns the largest share of the bound used per output."""
    ratios = {}
    for k, b in ref64.items():
        a = got.get(k)
        if a is None or b.numel() == 0:
            continue
        assert torch.isfinite(a).all(), (what, k)
        L = lead(k)
        err, bmax = hv.rel_rows(a, b, L), row_max(b, L)
        bound = np.maximum(REL_MIN, K_FLOOR * floor[k])
        keep = np.ones(err.shape, bool) if ok is None else np.broadcast_to(ok.reshape((-1,) + (1,) * (L - 1)),
                                                                             err.shape)
        zero = bmax == 0
        top = float((ref64 if scale is None else scale)[k].abs().max())
        loud = row_max(a, L)[zero & keep]
        assert (loud <= ZERO_REL * top).all(), (what, k, "zero rows", loud.max(), top)
        live = keep & ~zero
        bad = np.argwhere(live & (err >= bound))
        assert bad.size == 0, (what, k, bad[:4].tolist(), err[live].max(), floor[k][live].max())
        if live.any():
            ratios[k] = float((err / bound)[live].max())
    return ratios


def cost_lead(k):
    return 2 if k == "pose" else 1


def jvp_lead(k):
    return 1 if k == "cost" else 2


def gn_lead(k):
    return 1


def parts(c):
    return list(c["t"].items())


# ------------------------------------------------------------------------------------------------ the three entries
def check_cost(cs, c, what):
    N = c["x3d"].shape[1]
    got = hv.run_hvp(c)
    if c["P"] == 0:                     # no pose: the point, delta and camera rows are exact zeros
        for k, v in got.items():
            if v is not None:
                assert v.numel() == 0 or torch.equal(v, torch.zeros_like(v)), (what, k)
        return got, {}
    ref64 = cost_oracle(c, torch.float64, c["t"])
    fl = floors(lambda dt, perm: cost_oracle(c, dt, c["t"], perm), ref64, cost_lead, N)
    ratios = compare(got, ref64, fl, cost_lead, what)
    if cs["blocks"]:
        for name, v in parts(c):
            t = {name: v}
            r64 = cost_oracle(c, torch.float64, t)
            f = floors(lambda dt, perm: cost_oracle(c, dt, t, perm), r64, cost_lead, N)
            r = compare(hv.run_hvp(c, t=t), r64, f, cost_lead, (what, name), scale=ref64)
            ratios.update({f"{k}_by_{name}": x for k, x in r.items()})
    return got, ratios


def check_gn(cs, c, what):
    got = gp.run_hvp(c)
    ref64 = gp.oracle_hvp(c, torch.float64, census=True)
    cond = ref64.pop("census")["cond"]
    ok = cond <= gp.COND_MAX
    assert ok.any(), (what, cond)
    ratios = compare(got, ref64, gp.floors(c, ref64), gn_lead, what, ok=ok)
    if cs["blocks"]:
        for name, v in parts(c):
            t = {k: (w if k == name else torch.zeros_like(w)) for k, w in c["t"].items()}
            cc = dict(c, t=t)
            r64 = gp.oracle_hvp(cc, torch.float64)
            r = compare(gp.run_hvp(c, t={name: v}), r64, gp.floors(cc, r64), gn_lead, (what, name), scale=ref64, ok=ok)
            ratios.update({f"{k}_by_{name}": x for k, x in r.items()})
    ratios["ill_conditioned"] = int((~ok).sum())
    return got, ratios


def check_jvp(cs, c, what):
    want = JVP_WANT[cs["want"]]
    N, S = c["x3d"].shape[1], c["S"]
    got = jv.run_jvp(c, want=want)
    if S == 0:
        for k, w, shape in zip(jv.OUTPUTS, want, ((0, c["B"], 2 * N), (0, c["B"], 2 * N, c["dof"]), (0, c["B"]))):
            assert (got[k] is None) != w and (not w or tuple(got[k].shape) == shape), (what, k)
        return got, {}
    ref64 = jvp_oracle(c, torch.float64, c["t"], want)
    fl = floors(lambda dt, perm: jvp_oracle(c, dt, c["t"], want, perm), ref64, jvp_lead, N)
    ratios = compare(got, ref64, fl, jvp_lead, what)
    if want[2] and any(want[:2]) and S >= JVP_POSE_MAJOR_MIN_S:
        # the cost alone switches to the pose-major kernel: pinned to float64 on its own
        alone = jv.run_jvp(c, want=JVP_WANT["cost"])
        r = compare(alone, {"cost": ref64["cost"]}, fl, jvp_lead, (what, "cost alone"))
        ratios["cost_alone_pose_major"] = r.get("cost", 0.0)
    if cs["blocks"]:
        for name, v in parts(c):
            t = {name: v}
            r64 = jvp_oracle(c, torch.float64, t, want)
            f = floors(lambda dt, perm: jvp_oracle(c, dt, t, want, perm), r64, jvp_lead, N)
            r = compare(jv.run_jvp(c, want=want, t=t), r64, f, jvp_lead, (what, name), scale=ref64)
            ratios.update({f"{k}_by_{name}": x for k, x in r.items()})
    return got, ratios


CHECK = dict(cost=check_cost, gn=check_gn, jvp=check_jvp)


def rerun(cs, c, want=None):
    if cs["entry"] == "cost":
        return hv.run_hvp(c, want=want)
    if cs["entry"] == "gn":
        return gp.run_hvp(c, want=want)
    return jv.run_jvp(c, want=want or JVP_WANT[cs["want"]])


def check_subsets(cs, c, got):
    """Each output asked for alone: the same bits as in the full call (not the JVP cost at S >= 64, which changes
    kernel when asked alone)."""
    names = {"cost": hv.OUTPUTS, "gn": gp.OUTPUTS, "jvp": jv.OUTPUTS}[cs["entry"]]
    for i, k in enumerate(names):
        if got[k] is None or (cs["entry"] == "jvp" and k == "cost" and c["S"] >= JVP_POSE_MAJOR_MIN_S):
            continue
        one = rerun(cs, c, want=tuple(j == i for j in range(len(names))))
        assert all(one[o] is None for o in names if o != k), (cs["id"], k)
        assert torch.equal(one[k], got[k]), (cs["id"], k)


def run_case(cs, dev, record=True):
    c, fr = build(cs, dev)
    check_census(cs, fr)
    got, ratios = CHECK[cs["entry"]](cs, c, cs["id"])
    again = rerun(cs, c)
    for k, v in got.items():                        # run to run: the same bits
        if v is not None:
            assert torch.equal(v, again[k]), (cs["id"], k)
    check_subsets(cs, c, got)
    if record:
        record_parity(f"derivative/{cs['id']}", kernels=sorted(kernels_of(cs)), N=c["N"], B=c["B"], dof=cs["dof"],
                      bounds=cs["bounds"] or "none", bound_k=K_FLOOR, rel_min=REL_MIN, **fr,
                      **{f"{k}_over_bound_max": v for k, v in ratios.items()})
    return ratios


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_derivative_matrix(cuda_device, case):
    run_case(case, cuda_device)


def test_every_boundary_is_in_the_matrix():
    """Every N, P and S of the axes in both DoFs; both kernels of cost_hvp and evaluate_jvp, the pose-major ones at the
    large N; every bound kind, z_min and both one-branch cases for each entry point; blocks per (entry, DoF, bounds)."""
    for dof in (4, 6):
        on = lambda entry, key: {cs[key] for cs in CASES if cs["entry"] == entry and cs["dof"] == dof}
        assert on("cost", "N") >= {1, NT - 1, NT, NT + 1, 2048, 16384, "max"}, dof
        assert on("cost", "P") >= {0, 1, HVP_POSE_TILE - 1, HVP_POSE_TILE, HVP_POSE_TILE + 1, 2 * HVP_POSE_TILE,
                                   2 * HVP_POSE_TILE + 1, 4 * HVP_POSE_TILE + 1}, dof
        pose_major = {(cs["N"], cs["P"]) for cs in CASES if cs["entry"] == "cost" and cs["dof"] == dof}
        big = {p for n, p in pose_major if n in (16384, "max")}
        assert big & {NT - 1, NT, NT + 1} and 4 * NT + 1 in big, dof
        assert on("gn", "N") >= {5, NT - 1, NT, NT + 1, 2048, 16384, "max"}, dof
        m = JVP_POSE_MAJOR_MIN_S
        assert on("jvp", "P") >= {0, 1, m - 1, m, NT - 1, NT, NT + 1, 4 * NT + 1}, dof
        assert on("jvp", "want") == set(JVP_WANT), dof
        assert on("jvp", "clip") == {True, False}, dof
        cost_only = {(cs["N"], cs["P"]) for cs in CASES if cs["entry"] == "jvp" and cs["dof"] == dof
                     and cs["want"] == "cost"}
        assert any((n, m - 1) in cost_only and (n, m) in cost_only for n, _ in cost_only), dof
        for entry in ("cost", "gn", "jvp"):
            assert on(entry, "bounds") == {None, "scalar", "tensor"}, (entry, dof)
            assert on(entry, "zmin") == {True, False}, (entry, dof)
            assert on(entry, "branch") == {"mixed", "inlier", "outlier"}, (entry, dof)
            blocks = {cs["bounds"] for cs in CASES if cs["entry"] == entry and cs["dof"] == dof and cs["blocks"]}
            assert blocks == {None, "scalar", "tensor"}, (entry, dof)
            assert all(resolve_n(cs) <= 2048 for cs in CASES if cs["entry"] == entry and cs["blocks"])
    assert ("jvp", 6, 16384, 513, "cost") in {(cs["entry"], cs["dof"], cs["N"], cs["P"], cs["want"]) for cs in CASES}
    assert ("cost", 6, 16384, 513) in {(cs["entry"], cs["dof"], cs["N"], cs["P"]) for cs in CASES}
    kernels = set().union(*(kernels_of(cs) for cs in CASES))
    assert kernels == {"cost_hvp_point_kernel", "cost_hvp_pose_kernel", "gn_plus_hvp_kernel", "evaluate_jvp_kernel",
                       "evaluate_jvp_cost_kernel"}


# ------------------------------------------------------------------------------------------------ exact properties
def _alone(c, b, pose_axis):
    """Object b of a case as a batch of one."""
    B = c["B"]
    one = {k: (v[b:b + 1] if torch.is_tensor(v) and v.dim() and v.shape[0] == B else v) for k, v in c.items()}
    if pose_axis == 0:
        one["poses"] = c["poses"][:, b:b + 1]
    one["t"] = {k: (v[:, b:b + 1] if k == "pose" and pose_axis == 0 else v[b:b + 1]) for k, v in c["t"].items()}
    one["B"] = 1
    return one


def check_object_independence(dev, grid):
    """B = 2 x SMs + 3: objects 0, B / 2 and B - 1 alone equal their rows, bit for bit, for both cost_hvp kernels
    (P = 129: two pose CTAs per object) and both evaluate_jvp kernels (S = 65: all outputs, then the cost alone)."""
    B = 2 * grid + 3
    c, _ = build(_c("cost", 6, 40, 129, B, "tensor"), dev, seed=9)
    full = hv.run_hvp(c)
    for b in (0, B // 2, B - 1):
        alone = hv.run_hvp(_alone(c, b, 1))
        for k in hv.OUTPUTS:
            assert torch.equal(alone[k], full[k][b:b + 1]), ("cost_hvp", b, k)
    c, _ = build(_c("jvp", 6, 40, JVP_POSE_MAJOR_MIN_S + 1, B, "tensor"), dev, seed=9)
    for want in (JVP_WANT["all"], JVP_WANT["cost"]):
        full = jv.run_jvp(c, want=want)
        for b in (0, B // 2, B - 1):
            alone = jv.run_jvp(_alone(c, b, 0), want=want)
            for k, w in zip(jv.OUTPUTS, want):
                if w:
                    assert torch.equal(alone[k], full[k][:, b:b + 1]), ("evaluate_jvp", want, b, k)


def test_objects_are_independent(cuda_device):
    check_object_independence(cuda_device, sms(cuda_device))


def check_largest_n(dev):
    """max_points_split(dof) points are taken by cost_hvp and gn_plus_hvp; one more is refused."""
    for dof in (6, 4):
        n = native.max_points_split(dof)
        c = hv.build_case(dof, n, 1, 1, dev, seed=3)
        got = hv.run_hvp(c)
        assert all(torch.isfinite(v).all() for v in got.values() if v is not None)
        g = gp.build_case(dof, n, 1, dev, seed=3)
        assert all(torch.isfinite(v).all() for v in gp.run_hvp(g).values() if v is not None)
        pad = lambda x: torch.cat((x, x[:, :1]), 1)
        for k in POINTS:
            c[k], c["t"][k], g[k], g["t"][k] = pad(c[k]), pad(c["t"][k]), pad(g[k]), pad(g["t"][k])
        with pytest.raises(native.NativeError, match="epnp_cost_hvp_f32"):
            hv.run_hvp(c)
        with pytest.raises(native.NativeError, match="epnp_gn_plus_hvp_f32"):
            gp.run_hvp(g)


def test_largest_point_count(cuda_device):
    check_largest_n(cuda_device)
