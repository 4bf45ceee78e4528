"""The training backward against float64 autograd across its tiles, clamps and batch sizes.

cost_backward (epnp_cost_backward_f32) runs one CTA per object over a grid of min(B, 4 * SMs) CTAs, walks the points in
tiles of NT * BW_PPT = 512 and stages the poses in shared memory in tiles of BW_POSE_TILE = 1024.  The matrix below puts
a case on each side of every one of those boundaries, in 6DoF and 4DoF, unbounded, with scalar and with per-object
bounds, with depths below z_min and with both Huber branches, and compares every object of the batch with the oracle's
float64 autograd (pinned to the reference's own autograd by test_oracle_cost_grad_cpu.py).  gn_plus_backward (the
resident form) is compared with the float64 composite; the training step of bench.py's `train` shape with a float64
reference built from the kernel's own samples and log-weights.

The bound is per object and per output: max|a - b| / max|b| within the object, against max(2e-4, K_FLOOR * floor),
floor = the same autograd in float32 against float64 for that object.  A batch-wide scale would let an object whose
gradients are orders of magnitude smaller than its neighbours' be entirely wrong.

The clamps make the gradient discontinuous: a (pose, point) pair whose projection lies within float32 rounding of a
bound, or whose depth lies within rounding of z_min, may take the other side in the kernel.  So the cases place every
bound and every object's depth offset in the widest gap between the float64 projections near a target, and assert the
margin they got.
"""
import numpy as np
import pytest
import torch

from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp_b200 import native
from epropnp_b200.synth import make_noise, make_problem

pytestmark = pytest.mark.gpu

K_FLOOR = 5                 # bound: max(REL_MIN, K_FLOOR * floor) per object and output
REL_MIN = 2e-4
POINT_TILE = 512            # NT * BW_PPT in cost_backward_kernel
POSE_TILE = 1024            # BW_POSE_TILE
CHUNK = 1 << 23             # (pose, point) pairs per float64 autograd chunk: a few GB at most
BOUND_GAP = 3e-4            # least distance (px) of a float64 projection from a bound it is compared with
ZMIN_GAP = 5e-6             # least distance of a float64 depth from z_min
OUTPUTS = ("x3d", "x2d", "w2d", "delta")


def resident_grid(dev):
    """CTAs in cost_backward's grid when B is large: 4 per SM."""
    return 4 * torch.cuda.get_device_properties(dev).multi_processor_count


# ------------------------------------------------------------------------------------------------ references
def _camera(cam_mats, z_min, lb, ub, sl, dtype):
    cast = lambda b: b[sl].to(dtype) if torch.is_tensor(b) else b
    return orc.Camera(cam_mats[sl].to(dtype), z_min, cast(lb), cast(ub))


def project(x3d, pose, cam_mats, z_min):
    """(depth zh, projection with the z clamp, before the bounds) of every (pose, point); pose (P, B, D)."""
    R = orc.pose_rotmat(pose)
    xh = x3d @ (cam_mats @ R).transpose(-1, -2) + (cam_mats @ pose[..., :3, None]).squeeze(-1).unsqueeze(-2)
    zh = xh[..., 2]
    return zh, xh[..., :2] / zh.clamp(min=z_min)[..., None]


def cost_grads(x3d, x2d, w2d, cam_mats, lb, ub, delta, poses, up, z_min, dtype, census=False):
    """dL/d(x3d, x2d, w2d, delta) of L = sum_{b, p} up[b, p] * cost_b(poses[b, p]) by the oracle's autograd in `dtype`,
    in chunks of objects and poses (the gradient is linear in `up`).  poses (B, P, D), up (B, P).  census: also the
    fractions of (pose, point) pairs below z_min, clamped by a bound, and on the Huber outlier branch."""
    B, P = up.shape
    N = x3d.shape[1]
    ob = max(1, min(B, CHUNK // (N * P) if N * P < CHUNK else 1))
    pp = max(1, min(P, CHUNK // (N * ob)))
    out = [torch.zeros(x.shape, dtype=dtype, device=x.device) for x in (x3d, x2d, w2d, delta)]
    counts = torch.zeros(3, dtype=torch.float64)
    for b0 in range(0, B, ob):
        sl = slice(b0, min(B, b0 + ob))
        leaves = [x[sl].detach().to(dtype).clone().requires_grad_(True) for x in (x3d, x2d, w2d, delta)]
        cam = _camera(cam_mats, z_min, lb, ub, sl, dtype)
        for p0 in range(0, P, pp):
            ps = poses[sl, p0:p0 + pp].transpose(0, 1).to(dtype)
            cost = orc.evaluate(*leaves[:3], ps, cam, leaves[3])["cost"]
            (cost * up[sl, p0:p0 + pp].T.to(dtype)).sum().backward()
            if census:
                with torch.no_grad():
                    zh, u = project(leaves[0], ps, cam.cam_mats, z_min)
                    counts[0] += float((zh < z_min).sum())
                    if cam.lb is not None:
                        lo, hi = orc._bound(cam.lb, u), orc._bound(cam.ub, u)
                        counts[1] += float(((u < lo) | (u > hi)).any(-1).sum())
                        u = torch.minimum(torch.maximum(u, lo), hi)
                    s = ((u - leaves[1]) * leaves[2]).norm(dim=-1)
                    counts[2] += float((s > leaves[3][:, None]).sum())
        for o, l in zip(out, leaves):
            o[sl] = l.grad
    fr = (counts / (B * P * N)).tolist()
    return out, dict(below_zmin=fr[0], clamped=fr[1], outlier=fr[2])


def per_object(a, b):
    """max|a - b| / max|b| of every object (leading axis); 0 where both are zero."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    return ((a - b).abs().amax(1) / b.abs().amax(1).clamp(min=1e-300)).numpy()


def assert_per_object(got, g64, g32, what, objs=None, k=None):
    """got / g64 / g32: lists over OUTPUTS (None = not compared); k: {output: K} where it is not K_FLOOR.  Returns the
    recorded numbers."""
    stats = {}
    for name, a, b, c in zip(OUTPUTS, got, g64, g32):
        if a is None:
            continue
        if objs is not None:
            a = a[objs]
        a = a.reshape(a.shape[0], -1)
        assert torch.isfinite(a).all(), (what, name)
        err, floor = per_object(a, b), per_object(c, b)
        bound = np.maximum(REL_MIN, (k or {}).get(name, K_FLOOR) * floor)
        bad = np.nonzero(err >= bound)[0]
        assert bad.size == 0, (what, name, "objects", bad[:8].tolist(), err[bad[:8]].tolist(), floor[bad[:8]].tolist())
        stats[f"grad_{name}_rel_max_per_object"] = float(err.max())
        stats[f"f32_oracle_floor_{name}_max"] = float(floor.max())
        stats[f"grad_{name}_over_bound_max"] = float((err / bound).max())
    return stats


# ------------------------------------------------------------------------------------------------ placing the clamps
def widest_gap_mid(values, target, window):
    """values (R, K), target (R,) -> (mid, half_gap) (R,): the middle of the widest gap between consecutive values within
    target +- window (the window's ends count as values)."""
    ends = torch.stack((target - window, target + window), 1)
    v = torch.cat((values, ends), 1).sort(1).values
    mid, gap = (v[:, 1:] + v[:, :-1]) / 2, v[:, 1:] - v[:, :-1]
    gap = torch.where((mid - target[:, None]).abs() <= window, gap, torch.full_like(gap, -1.0))
    i = gap.argmax(1, keepdim=True)
    return mid.gather(1, i)[:, 0], gap.gather(1, i)[:, 0] / 2


def quantile(v, q):
    """Lower q-quantile along dim 1 (torch.quantile refuses more than 2^24 values)."""
    return v.kthvalue(max(1, min(v.shape[1], int(round(q * v.shape[1])))), dim=1).values


def _each_object_chunk(B, K):
    ob = max(1, (1 << 24) // max(K, 1))
    for b0 in range(0, B, ob):
        yield slice(b0, min(B, b0 + ob))


def place_depths(x3d, poses, cam_mats, z_min):
    """Shift every object's pose depths by one offset so that z_min sits in the widest gap of that object's depths near
    the 15 % quantile; returns the shifted poses (float32) and the least margin."""
    poses = poses.clone()
    d = torch.float64
    B = poses.shape[0]
    for sl in _each_object_chunk(B, poses.shape[1] * x3d.shape[1]):
        ps = poses[sl].transpose(0, 1).to(d)
        zh, _ = project(x3d[sl].to(d), ps, cam_mats[sl].to(d), z_min)
        zh = zh.permute(1, 0, 2).reshape(ps.shape[1], -1)
        target = quantile(zh, 0.15)
        mid, _ = widest_gap_mid(zh, target, 0.05)
        poses[sl, :, 2] += (z_min - mid).to(poses.dtype)[:, None]
    return poses, min_gap_depth(x3d, poses, cam_mats, z_min)


def min_gap_depth(x3d, poses, cam_mats, z_min):
    d, m = torch.float64, float("inf")
    for sl in _each_object_chunk(poses.shape[0], poses.shape[1] * x3d.shape[1]):
        zh, _ = project(x3d[sl].to(d), poses[sl].transpose(0, 1).to(d), cam_mats[sl].to(d), z_min)
        m = min(m, float((zh - z_min).abs().min()))
    return m


def place_bounds(x3d, poses, cam_mats, z_min, per_object, q=0.04):
    """Bounds that clamp about a share q of the projections on each side, placed where no projection is near them: per
    object and coordinate (tensor bounds, (B, 2)) or one value for both coordinates of every object (scalar bounds).
    Each starts at its quantile of the float64 projections and moves into their widest gap within 2 px of it.  Returns
    (lb, ub) and the least margin of any projection from a bound."""
    d = torch.float64
    B = poses.shape[0]
    placed, us, margin = [], [], float("inf")
    for sl in _each_object_chunk(B, poses.shape[1] * x3d.shape[1]):
        _, u = project(x3d[sl].to(d), poses[sl].transpose(0, 1).to(d), cam_mats[sl].to(d), z_min)
        u = u.permute(1, 0, 2, 3).reshape(u.shape[1], -1, 2)                  # (objects, pairs, 2)
        if not per_object:
            us.append(u.reshape(-1, 2))
            continue
        lu = [torch.stack([widest_gap_mid(u[..., c], quantile(u[..., c], qq), 2.0)[0] for c in range(2)], 1).float()
              for qq in (q, 1 - q)]
        for b in lu:
            margin = min(margin, float((u - b.double()[:, None, :]).abs().min()))
        placed.append(lu)
    if per_object:
        return (torch.cat([p[0] for p in placed]).contiguous(), torch.cat([p[1] for p in placed]).contiguous(), margin)
    flat = torch.cat(us).reshape(1, -1)
    out = []
    for qq in (q, 1 - q):
        mid, _ = widest_gap_mid(flat, quantile(flat, qq), 2.0)
        out.append(float(np.float32(float(mid[0]))))
    return out[0], out[1], min(float((flat - v).abs().min()) for v in out)


# ------------------------------------------------------------------------------------------------ the cost_backward matrix
# B = mult * G + add with G = 4 * SMs (the grid); bounds: None | "scalar" | "tensor"; zmin: a share of the pairs below
# z_min; P = PA + PB.
CASES = [
    dict(id="d6_N1_P01_B1", dof=6, bounds=None, N=1, PA=0, PB=1, B=(0, 1)),
    dict(id="d6_scalar_N7_P10_Gm1", dof=6, bounds="scalar", N=7, PA=1, PB=0, B=(1, -1)),
    dict(id="d4_tensor_N128_P512_G", dof=4, bounds="tensor", N=128, PA=512, PB=1, B=(1, 0), outliers=0.1),
    dict(id="d6_N511_P1023_Gp1", dof=6, bounds=None, N=511, PA=1023, PB=1, B=(1, 1), outliers=0.1, beyond_grid=True),
    dict(id="d6_tensor_N512_P1024_B1", dof=6, bounds="tensor", N=512, PA=1024, PB=0, B=(0, 1)),
    dict(id="d6_tensor_N513_P1025_2Gp3", dof=6, bounds="tensor", N=513, PA=1024, PB=1, B=(2, 3), outliers=0.1,
         many_pose_tiles=True, beyond_grid=True),
    dict(id="d4_scalar_N256_P2049_B1", dof=4, bounds="scalar", N=256, PA=2048, PB=1, B=(0, 1), outliers=0.1,
         many_pose_tiles=True),
    dict(id="d6_zmin_N1000_P65_Gp1", dof=6, bounds=None, N=1000, PA=64, PB=1, B=(1, 1), zmin=True, outliers=0.1,
         beyond_grid=True),
    dict(id="d4_zmin_tensor_N513_P01_Gm1", dof=4, bounds="tensor", N=513, PA=0, PB=1, B=(1, -1), zmin=True),
    dict(id="d6_N4096_P513_B3", dof=6, bounds=None, N=4096, PA=512, PB=1, B=(0, 3), outliers=0.1),
    dict(id="d6_scalar_Nmax_P1_B2", dof=6, bounds="scalar", N="max", PA=1, PB=0, B=(0, 2)),
    dict(id="d4_Nmax_P10_2Gp3", dof=4, bounds=None, N="max", PA=1, PB=0, B=(2, 3), outliers=0.1, beyond_grid=True),
    dict(id="d6_tensor_N16384_P33_B3", dof=6, bounds="tensor", N=16384, PA=32, PB=1, B=(0, 3), outliers=0.1),
]


def case_shape(case, dev):
    G = resident_grid(dev)
    B = case["B"][0] * G + case["B"][1]
    N = native.max_points(case["dof"]) if case["N"] == "max" else case["N"]
    return B, N, G


def softmax_like(B, PA, PB, gen):
    """Upstream gradients the way the Monte-Carlo loss hands them down: on the PA sample poses, minus softmax weights
    spanning about 1e-30 .. 1 (half the poses near 1e-27, the others within a few decades of the largest), a random
    sign and about 10 % exact zeros; on the PB poses +1, the cost_init term; all times a per-object scale of 1 .. 1e-12."""
    logits = 4.0 * torch.randn(B, PA, generator=gen, dtype=torch.float64)
    logits -= 60.0 * (torch.rand(B, PA, generator=gen) < 0.5)
    w = -torch.softmax(logits, dim=1)
    sign = torch.where(torch.rand(B, PA, generator=gen) < 0.3, -1.0, 1.0).double()
    zero = torch.rand(B, PA, generator=gen) < 0.1
    w = (w * sign).masked_fill(zero, 0.0)
    scale = 10.0 ** (-12.0 * torch.rand(B, 1, generator=gen, dtype=torch.float64))
    return (torch.cat((w, torch.ones(B, PB, dtype=torch.float64)), 1) * scale).float()


def build_case(case, dev, seed=7):
    """-> dict of the inputs of one cost_backward case (on `dev`) and the checks that its condition holds."""
    B, N, G = case_shape(case, dev)
    dof, P = case["dof"], case["PA"] + case["PB"]
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=case.get("outliers", 0.0))
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, P, 1)
    poses[..., :3] += 0.03 * torch.randn(B, P, 3, generator=gen)
    if dof == 6:
        q = poses[..., 3:] + 0.02 * torch.randn(B, P, 4, generator=gen)
        poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.05 * torch.randn(B, P, generator=gen)
    up = softmax_like(B, case["PA"], case["PB"], gen)
    c = {k: v.to(dev) for k, v in pc.items()}
    c.update(B=B, N=N, P=P, G=G, dof=dof, poses=poses.to(dev), up=up.to(dev), z_min=0.1, lb=None, ub=None)
    margins = {}
    if case.get("zmin"):
        c["z_min"] = 4.0
        c["poses"], margins["zmin_margin"] = place_depths(c["x3d"], c["poses"], c["cam_mats"], c["z_min"])
        assert margins["zmin_margin"] > ZMIN_GAP, margins
    if case["bounds"]:
        c["lb"], c["ub"], margins["bound_margin"] = place_bounds(c["x3d"], c["poses"], c["cam_mats"], c["z_min"],
                                                                 case["bounds"] == "tensor")
        assert margins["bound_margin"] > BOUND_GAP, margins
    # (one point has no spread to scale delta by)
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5) if N > 1 else torch.full((B,), 4.0, device=dev)
    c["margins"] = margins
    return c


def split_poses(c, case):
    PA = case["PA"]
    pa, ga = c["poses"][:, :PA].contiguous(), c["up"][:, :PA].contiguous()
    pb = gb = None
    if case["PB"]:
        pb, gb = c["poses"][:, PA:].contiguous(), c["up"][:, PA:].contiguous()
    return pa, ga, pb, gb


def run_kernel(c, case, want=(True, True, True, True), **over):
    x = dict(c, **over)
    prob = native.Problem(x["x3d"], x["x2d"], x["w2d"], x["cam_mats"], x["lb"], x["ub"], x["delta"])
    pa, ga, pb, gb = split_poses(x, case)
    return native.cost_backward(prob, x["dof"], x["z_min"], pa, ga, pb, gb, want=want)


def reference(c, dtype, census=False):
    return cost_grads(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"], c["poses"], c["up"],
                      c["z_min"], dtype, census)


def check_conditions(case, c, fr):
    """What each case exists for must really happen."""
    if case["bounds"]:
        assert 0.05 <= fr["clamped"] <= 0.2, fr
    if case.get("zmin"):
        assert 0.05 <= fr["below_zmin"] <= 0.3, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if case.get("outliers"):
        assert 0.01 <= fr["outlier"] <= 0.99, fr          # both Huber branches
    if case.get("many_pose_tiles"):
        assert c["P"] > POSE_TILE
    if case.get("beyond_grid"):
        assert c["B"] > c["G"]            # some CTA handles more than one object


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_cost_backward_matrix(cuda_device, case):
    c = build_case(case, cuda_device)
    got = run_kernel(c, case)
    g64, fr = reference(c, torch.float64, census=True)
    g32, _ = reference(c, torch.float32)
    check_conditions(case, c, fr)
    # K_FLOOR = 5: five times what float32 rounding alone moves the same object's gradient
    stats = assert_per_object(list(got), g64, g32, case["id"])
    record_parity(f"backward/cost/{case['id']}", B=c["B"], N=c["N"], P=c["P"], grid=min(c["B"], c["G"]), dof=c["dof"],
                  bounds=case["bounds"] or "none", bound_k=K_FLOOR, rel_min=REL_MIN, **fr, **c["margins"], **stats)


def test_risky_pairs_are_in_the_matrix(cuda_device):
    """P > 1024 with bounds on; N > 512 with B > grid; 4DoF at N > 512."""
    shapes = [(case, *case_shape(case, cuda_device)) for case in CASES]
    assert any(cs["bounds"] and cs["PA"] + cs["PB"] > POSE_TILE for cs, *_ in shapes)
    assert any(N > POINT_TILE and B > G for cs, B, N, G in shapes)
    assert any(cs["dof"] == 4 and N > POINT_TILE for cs, B, N, G in shapes)
    assert {N for _, _, N, _ in shapes} >= {1, 7, 128, 511, 512, 513, 1000, 4096, 16384,
                                             native.max_points(6), native.max_points(4)}


# ------------------------------------------------------------------------------------------------ exact properties
PROP_CASE = dict(id="props", dof=6, bounds="tensor", N=513, PA=1024, PB=1, B=(2, 3), outliers=0.1)


def test_cost_backward_exact_properties(cuda_device):
    """Same bits twice; object b solved alone equals row b (b = 0, G, 2G run on the same CTA one after another);
    leaving out an output leaves the others unchanged; a NaN in object 0 does not reach the objects the same CTA
    handles later."""
    case = PROP_CASE
    c = build_case(case, cuda_device, seed=11)
    G = c["G"]
    full = run_kernel(c, case)
    for a, b in zip(full, run_kernel(c, case)):
        assert torch.equal(a, b)
    for b in (0, G, 2 * G, c["B"] - 1):
        s = slice(b, b + 1)
        one = {k: (v[s] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == c["B"] else v) for k, v in c.items()}
        for x, y in zip(run_kernel(one, case), full):
            assert torch.equal(x[0], y[b]), b
    for i in range(4):
        want = tuple(j != i for j in range(4))
        part = run_kernel(c, case, want=want)
        assert part[i] is None
        for j in range(4):
            if j != i:
                assert torch.equal(part[j], full[j]), (i, j)
    x2d = c["x2d"].clone()
    x2d[0, 5, 0] = float("nan")
    poisoned = run_kernel(c, case, x2d=x2d)
    assert not torch.isfinite(poisoned[3][0])
    for x, y in zip(poisoned, full):
        assert torch.equal(x[1:], y[1:])


# ------------------------------------------------------------------------------------------------ gn_plus_backward, resident
EPS, HUBER_EPS = 1e-5, 1e-10
GN_CASES = [
    dict(id="d6_N5_outlier", dof=6, N=5, bounds=False, outliers=0.2),
    dict(id="d6_N129_bounded_outliers", dof=6, N=129, bounds=True, outliers=0.1),
    dict(id="d4_N129_zmin", dof=4, N=129, bounds=False, zmin=True),
    dict(id="d6_N512_zmin_bounded", dof=6, N=512, bounds=True, zmin=True, outliers=0.1),
    dict(id="d4_N1000_bounded_outliers", dof=4, N=1000, bounds=True, outliers=0.1),
    dict(id="d6_N4096", dof=6, N=4096, bounds=False, outliers=0.1),
    dict(id="d4_N4096_zmin", dof=4, N=4096, bounds=False, zmin=True),
    dict(id="d6_Nmax_bounded", dof=6, N="max", bounds=True, outliers=0.1),
    dict(id="d4_Nmax_zmin_bounded", dof=4, N="max", bounds=True, zmin=True, outliers=0.1),
]


def composite(c, gp, dtype):
    import test_gn_plus_split_gpu as gs
    return gs.composite_grads(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"], c["pose"], gp,
                              c["dof"], c["z_min"], dtype)


def build_gn_case(case, dev, B=3, seed=5):
    dof = case["dof"]
    N = native.max_points(dof) if case["N"] == "max" else case["N"]
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, dof=dof,
                                                outlier_frac=case.get("outliers", 0.0)).items()}
    c = dict(pc, dof=dof, N=N, z_min=0.01, lb=None, ub=None, pose=pc["pose_init"][:, None].clone(), margins={})
    if case.get("zmin"):
        c["z_min"] = 4.0
        c["pose"], c["margins"]["zmin_margin"] = place_depths(c["x3d"], c["pose"], c["cam_mats"], c["z_min"])
        assert c["margins"]["zmin_margin"] > ZMIN_GAP
    if case["bounds"]:
        c["lb"], c["ub"], c["margins"]["bound_margin"] = place_bounds(c["x3d"], c["pose"], c["cam_mats"], c["z_min"],
                                                                      True)
        assert c["margins"]["bound_margin"] > BOUND_GAP
    c["pose"] = c["pose"][:, 0].contiguous()
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.1)
    gp = torch.randn(B, 7 if dof == 6 else 4, generator=torch.Generator().manual_seed(seed)).to(dev)
    return c, gp


@pytest.mark.parametrize("case", GN_CASES, ids=[c["id"] for c in GN_CASES])
def test_gn_plus_backward_matrix(cuda_device, case):
    c, gp = build_gn_case(case, cuda_device)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    full = native.gn_plus_backward(prob, c["pose"], gp, c["dof"], c["z_min"], EPS, HUBER_EPS)
    c64, c32 = composite(c, gp, torch.float64), composite(c, gp, torch.float32)
    # the share of points the clip mask zeroes, and the outliers
    with torch.no_grad():
        zh, u = project(c["x3d"].double(), c["pose"][None].double(), c["cam_mats"].double(), c["z_min"])
        below = float((zh < c["z_min"]).double().mean())
        clamped = 0.0
        if case["bounds"]:
            clamped = float(((u < c["lb"].double()[None, :, None]) | (u > c["ub"].double()[None, :, None]))
                            .any(-1).double().mean())
    if case.get("zmin"):
        assert 0.05 <= below <= 0.3, below
    if case["bounds"]:
        assert 0.01 <= clamped <= 0.3, clamped
    # K_FLOOR = 5 against the float64 composite, per object; grad_delta K = 10: one number per object, a sum of
    # outlier terms of both signs through the solve, whose rounding noise the float32 composite samples only once (on
    # the H100 a 4DoF object measured 5.4 times its float32 floor, at 1.2e-3 of a value 19 times below its neighbour's)
    stats = assert_per_object(list(full), c64, c32, case["id"], k={"delta": 10})
    for i in range(4):                      # an omitted output leaves the others' bits unchanged
        part = native.gn_plus_backward(prob, c["pose"], gp, c["dof"], c["z_min"], EPS, HUBER_EPS,
                                       want=tuple(j != i for j in range(4)))
        assert part[i] is None and all(torch.equal(part[j], full[j]) for j in range(4) if j != i)
    record_parity(f"backward/gn_plus/{case['id']}", N=c["N"], dof=c["dof"], bound_k=K_FLOOR, rel_min=REL_MIN,
                  below_zmin=below, clamped=clamped, **c["margins"], **stats)


# ------------------------------------------------------------------------------------------------ the training step
def mc_reference(x3d, x2d, w2d, cam_mats, delta_fn, pose_init, samples, logw, scale, objs, z_min, dtype):
    """dL/d(x3d, x2d, w2d) of L = scale * sum_b [cost_b(pose_init_b) - sum_m softmax(logw_b)_m cost_b(sample_bm)] with
    delta = delta_fn(w2d) (AdaptiveHuberPnPCost.set_param(x2d.detach(), w2d)), for the objects `objs`, in `dtype`."""
    s = lambda t: t[objs].detach().to(dtype)
    x3d, x2d, w2d, pose_init, samples = s(x3d), s(x2d), s(w2d), s(pose_init), s(samples)
    w = torch.softmax(logw[objs].detach().double(), dim=1).to(dtype)
    w2d_leaf = w2d.clone().requires_grad_(True)
    delta = delta_fn(x2d, w2d_leaf)
    poses = torch.cat((pose_init[:, None], samples), 1)
    up = scale * torch.cat((torch.ones_like(w[:, :1]), -w), 1)
    (g3, g2, gw, gd), _ = cost_grads(x3d, x2d, w2d, cam_mats[objs], None, None, delta.detach(), poses, up, z_min, dtype)
    gw = gw + torch.autograd.grad(delta, w2d_leaf, gd)[0]
    return [g3, g2, gw]


def train_step(dev, monkeypatch, dof, B, N, M, I, epilogue, seed=3):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP4DoF, EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    monkeypatch.setenv("EPNP_NATIVE_MC_EPILOGUE", str(epilogue))
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, dof=dof).items()}
    layer = (EProPnP6DoF if dof == 6 else EProPnP4DoF)(mc_samples=M, num_iter=I, solver=LMSolver(dof=dof, num_iter=10))
    loss_fn = MonteCarloPoseLoss().to(dev)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.1)
    x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(x2d.detach(), w2d)
    kw = dict(amis_noise=tuple(t.to(dev) for t in make_noise(B, M, seed=seed + 1))) if dof == 6 else dict(amis_seed=9)
    _, _, _, samples, logw, cost_tgt = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=pc["pose_gt"],
                                                                 force_init_solve=False, **kw)
    loss = loss_fn(logw, cost_tgt, 1.0)
    loss.backward()
    nf = float(loss_fn.norm_factor)
    return pc, [x3d.grad, x2d.grad, w2d.grad], samples.detach().transpose(0, 1), logw.detach().T, nf


def check_train_step(dev, monkeypatch, dof, B, N, M, I, record):
    objs = torch.cat((torch.arange(0, B, 64), torch.tensor([B - 1]))).unique().to(dev)
    runs = [train_step(dev, monkeypatch, dof, B, N, M, I, e) for e in (0, 1)]
    pc, _, samples, logw, nf = runs[1]
    delta_fn = lambda x2d, w2d: orc.adaptive_delta(x2d, w2d, 0.5)
    ref = [mc_reference(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], delta_fn, pc["pose_gt"], samples, logw,
                        1.0 / (B * nf), objs, 0.1, dt) for dt in (torch.float64, torch.float32)]
    stats = {}
    for e, (_, grads, s_e, l_e, _) in zip((0, 1), runs):
        assert torch.equal(s_e, samples) and torch.equal(l_e, logw)      # same forward either way
        # K_FLOOR = 5 per object against float64 built from the kernel's own samples and log-weights
        st = assert_per_object(grads + [None], ref[0] + [None], ref[1] + [None], f"{record} epilogue={e}", objs)
        stats.update({f"epilogue{e}_{k}": v for k, v in st.items()})
    for name, a, b, g64, g32 in zip(OUTPUTS, runs[0][1], runs[1][1], ref[0], ref[1]):
        floor = per_object(g32, g64)
        err = per_object(a[objs], b[objs])
        assert (err < np.maximum(REL_MIN, K_FLOOR * floor)).all(), (name, err.max())
        stats[f"epilogue0_vs_1_{name}_rel_max_per_object"] = float(err.max())
    record_parity(record, B=B, N=N, M=M, I=I, dof=dof, objects_compared=int(objs.numel()), bound_k=K_FLOOR,
                  rel_min=REL_MIN, **stats)


def test_training_step_bench_shape(cuda_device, monkeypatch):
    """bench.py --config train: B = 4096, N = 512, M = 512, I = 4, pose_init = pose_gt, MonteCarloPoseLoss."""
    check_train_step(cuda_device, monkeypatch, 6, 4096, 512, 512, 4, "backward/train/6dof_B4096_N512_M512")


def test_training_step_4dof(cuda_device, monkeypatch):
    check_train_step(cuda_device, monkeypatch, 4, 512, 512, 512, 4, "backward/train/4dof_B512_N512_M512")


def test_training_step_with_pose_opt_plus(cuda_device, monkeypatch):
    """The 6DoF objective of lib/train.py with loss_t / loss_r on pose_opt_plus, at N = 512: the native step
    (EPNP_NATIVE_GN_STEP=1) against the torch composite (=0) and against float64 (Monte-Carlo part from the kernel's
    samples and log-weights + the float64 composite of the Gauss-Newton step)."""
    check_pose_opt_plus(cuda_device, monkeypatch, 64, 512, 512, 4)


def check_pose_opt_plus(dev, monkeypatch, B, N, M, I):
    import test_gn_plus_split_gpu as gs
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=23).items()}
    layer = EProPnP6DoF(mc_samples=M, num_iter=I, solver=LMSolver(dof=6, num_iter=10))
    mc_loss = MonteCarloPoseLoss().to(dev)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.1)
    pose_gt = pc["pose_gt"]

    def run(native_step):
        monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1" if native_step else "0")
        x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(pc["x2d"], pc["w2d"])
        cost_fun.delta = cost_fun.delta.detach().clone().requires_grad_(True)
        pose_opt, _, plus, samples, logw, cost_tgt = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=pose_gt, force_init_solve=False, with_pose_opt_plus=True,
            amis_noise=tuple(t.to(dev) for t in make_noise(B, M, seed=24)))
        loss_mc = mc_loss(logw, cost_tgt, torch.tensor(1.0, device=dev))
        loss_t = (plus[:, :3] - pose_gt[:, :3]).norm(dim=-1)
        beta = 0.05
        loss_t = torch.where(loss_t < beta, 0.5 * loss_t.square() / beta, loss_t - 0.5 * beta).mean()
        dot_quat = (plus[:, None, 3:] @ pose_gt[:, 3:, None]).squeeze(-1).squeeze(-1)
        loss_r = ((1 - dot_quat.square()) * 2).mean()
        loss = loss_mc + loss_t + loss_r
        ups = torch.autograd.grad(loss, [logw, cost_tgt, plus], retain_graph=True)
        loss.backward()
        return ([t.grad for t in (x3d, x2d, w2d, cost_fun.delta)], ups, pose_opt.detach(), samples.detach(),
                cost_fun.delta.detach())

    grads, (g_logw, g_cost, g_plus), pose_opt, samples, delta = run(True)
    comp, *_ = run(False)
    poses = torch.cat((pc["pose_gt"][:, None], samples.transpose(0, 1)), 1)
    up = torch.cat((g_cost.reshape(B, 1), -g_logw.T), 1)
    refs = []
    for dt in (torch.float64, torch.float32):
        mc, _ = cost_grads(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta, poses, up, 0.1, dt)
        gn = gs.composite_grads(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta, pose_opt, g_plus, 6,
                                0.1, dt)
        refs.append([a + b for a, b in zip(mc, gn)])
    # K_FLOOR = 5 per object: the native step and the composite step against float64
    stats = assert_per_object(grads, refs[0], refs[1], "native GN step")
    cstats = assert_per_object(comp, refs[0], refs[1], "composite GN step")
    record_parity(f"backward/train/6dof_pose_opt_plus_B{B}_N{N}", **stats,
                  **{f"composite_{k}": v for k, v in cstats.items()}, bound_k=K_FLOOR, rel_min=REL_MIN)
