"""Gradients through evaluate_pnp's residual, Jacobian and cost (epnp_evaluate_backward_f32) against float64 autograd,
per object, in the manner of test_backward_matrix_gpu.py (whose clamp placement and per-object measure this file uses).

The reference is the oracle's autograd of L = <g_res, residual> + <g_jac, jacobian> + <g_cost, cost> through
oracle.evaluate(want_jac=True) (pinned to the reference's own autograd by test_oracle_evaluate_grad_cpu.py).  The bound
is max|a - b| / max|b| within one object's gradient of one input under max(2e-4, 5 * floor), floor = the same autograd
in float32 for that object.  The matrix spans N from 1 to 65 536 (above the split limit: the kernel streams the points),
S = 1, 3 and 64, both DOF, clip_jac on and off, no / scalar / per-object / one shared (2,) bound, depths clamped at z_min,
both Huber branches, and each upstream gradient alone and all three together.  Then exact properties, a CUDA-graph
replay, and LMSolver.gn_step under autograd against _PosePlus (the validated gn_plus_backward kernels)."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import HuberPnPCost
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

INPUTS = ("x3d", "x2d", "w2d", "delta", "pose", "cam", "lb", "ub")
HUBER_EPS = 1e-10
UPS = ("res", "jac", "cost")


def build_case(dof, N, S, B=3, bounds=None, zmin=False, outliers=0.0, clip=True, ups=UPS, dev="cpu", seed=17):
    """bounds: None | "scalar" | "tensor" (per object) | "shared" (one (2,) tensor).  -> dict of inputs on `dev`."""
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outliers)
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, S, 1)                       # object-major while placing the clamps
    poses[..., :3] += 0.03 * torch.randn(B, S, 3, generator=gen)
    if dof == 6:
        q = poses[..., 3:] + 0.02 * torch.randn(B, S, 4, generator=gen)
        poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.05 * torch.randn(B, S, generator=gen)
    c = {k: v.to(dev) for k, v in pc.items()}
    c.update(B=B, N=N, S=S, dof=dof, z_min=0.1, lb=None, ub=None, clip=clip, margins={})
    poses = poses.to(dev)
    if zmin:
        c["z_min"] = 4.0
        poses, c["margins"]["zmin_margin"] = bm.place_depths(c["x3d"], poses, c["cam_mats"], c["z_min"])
        assert c["margins"]["zmin_margin"] > bm.ZMIN_GAP, c["margins"]
    if bounds:
        lb, ub, margin = bm.place_bounds(c["x3d"], poses, c["cam_mats"], c["z_min"], bounds == "tensor")
        if bounds == "shared":
            lb, ub = torch.tensor([lb, lb], device=dev), torch.tensor([ub, ub], device=dev)
        c["lb"], c["ub"], c["margins"]["bound_margin"] = lb, ub, margin
        assert margin > bm.BOUND_GAP, margin
    c["poses"] = poses.transpose(0, 1).contiguous()                         # (S, B, D)
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5) if N > 1 else torch.full((B,), 4.0, device=dev)
    D = 7 if dof == 6 else 4
    up = dict(res=torch.randn(S, B, 2 * N, generator=gen), jac=torch.randn(S, B, 2 * N, dof, generator=gen),
              cost=torch.randn(S, B, generator=gen))
    scale = 10.0 ** (-3.0 * torch.rand(1, B, generator=gen))                # objects of different scales
    c["ups"] = {k: (v * scale.reshape((1, B) + (1,) * (v.dim() - 2))).to(dev) if k in ups else None
                for k, v in up.items()}
    c["D"] = D
    return c


def tensor_bounds(c, B):
    """(B, 2) tensors of the case's bounds (None when it has none): what the kernel receives."""
    if c["lb"] is None:
        return None, None
    one = lambda b: (b.expand(B, 2) if torch.is_tensor(b) else torch.full((B, 2), float(b), device=c["x3d"].device))
    return one(c["lb"]), one(c["ub"])


def run_kernel(c, want=(True,) * 8, **over):
    x = dict(c, **over)
    prob = native.Problem(x["x3d"], x["x2d"], x["w2d"], x["cam_mats"], x["lb"], x["ub"], x["delta"])
    want = tuple(w and (i < 6 or prob.lb is not None) for i, w in enumerate(want))
    u = x["ups"]
    return native.evaluate_backward(prob, x["poses"], x["dof"], x["z_min"], HUBER_EPS, x["clip"], u["res"], u["jac"],
                                    u["cost"], want=want)


def reference(c, dtype, census=False):
    """The eight gradients (x3d, x2d, w2d, delta (B), pose (S, B, D), cam (B, 3, 3), lb, ub (B, 2) | None) by the
    oracle's autograd in `dtype`, object by object (an object's gradients depend on its own inputs only)."""
    B = c["B"]
    lbt, ubt = tensor_bounds(c, B)
    out = [None] * 8
    counts = torch.zeros(3, dtype=torch.float64)
    ob = max(1, min(B, (1 << 21) // (c["S"] * c["N"])))
    for b0 in range(0, B, ob):
        sl = slice(b0, min(B, b0 + ob))
        leaves = [c[k][sl].detach().to(dtype).clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d", "delta")]
        leaves.append(c["poses"][:, sl].detach().to(dtype).clone().requires_grad_(True))
        leaves.append(c["cam_mats"][sl].detach().to(dtype).clone().requires_grad_(True))
        lb, ub = c["lb"], c["ub"]
        if torch.is_tensor(lb):
            leaves += [t[sl].detach().to(dtype).clone().requires_grad_(True) for t in (lbt, ubt)]
            lb, ub = leaves[6], leaves[7]
        cam = orc.Camera(leaves[5], c["z_min"], lb, ub)
        e = orc.evaluate(*leaves[:3], leaves[4], cam, leaves[3], want_jac=True, clip_jac=c["clip"], eps_huber=HUBER_EPS)
        loss = 0.0
        for k, name in (("res", "residual"), ("jac", "jac"), ("cost", "cost")):
            if c["ups"][k] is not None:
                loss = loss + (e[name] * c["ups"][k][:, sl].to(dtype)).sum()
        loss.backward()
        if census:
            with torch.no_grad():
                zh, u = bm.project(leaves[0], leaves[4], leaves[5], c["z_min"])
                counts[0] += float((zh < c["z_min"]).sum())
                if c["lb"] is not None:
                    lo, hi = orc._bound(lb, u), orc._bound(ub, u)
                    counts[1] += float(((u < lo) | (u > hi)).any(-1).sum())
                    u = torch.minimum(torch.maximum(u, lo), hi)
                counts[2] += float((((u - leaves[1]) * leaves[2]).norm(dim=-1) > leaves[3][:, None]).sum())
        for i, l in enumerate(leaves):
            if out[i] is None:
                shape = (c["S"], B) + tuple(l.shape[2:]) if i == 4 else (B,) + tuple(l.shape[1:])
                out[i] = torch.zeros(shape, dtype=dtype, device=l.device)
            if i == 4:
                out[i][:, sl] = l.grad
            else:
                out[i][sl] = l.grad
    fr = (counts / (B * c["S"] * c["N"])).tolist()
    return out, dict(below_zmin=fr[0], clamped=fr[1], outlier=fr[2])


def _objects_first(name, t):
    return t.transpose(0, 1) if name == "pose" else t


def assert_per_object(got, g64, g32, what):
    """bm.assert_per_object over the eight inputs; a pose gradient (S, B, D) is judged over all S poses of an object."""
    stats = {}
    for name, a, b, c in zip(INPUTS, got, g64, g32):
        if a is None or b is None:
            continue
        a, b, c = (_objects_first(name, t) for t in (a, b, c))
        assert torch.isfinite(a).all(), (what, name)
        err, floor = bm.per_object(a, b), bm.per_object(c, b)
        bound = np.maximum(bm.REL_MIN, bm.K_FLOOR * floor)
        bad = np.nonzero(err >= bound)[0]
        assert bad.size == 0, (what, name, bad[:8].tolist(), err[bad[:8]].tolist(), floor[bad[:8]].tolist())
        stats[f"grad_{name}_rel_max_per_object"] = float(err.max())
        stats[f"f32_oracle_floor_{name}_max"] = float(floor.max())
        stats[f"grad_{name}_over_bound_max"] = float((err / bound).max())
    return stats


# (id, dof, N, S, bounds, zmin, outliers, clip, upstreams)
CASES = [
    ("d6_N1_S1", 6, 1, 1, None, False, 0.0, True, UPS),
    ("d4_N7_S3_scalar", 4, 7, 3, "scalar", False, 0.0, True, UPS),
    ("d6_N512_S64_tensor_out", 6, 512, 64, "tensor", False, 0.1, True, UPS),
    ("d4_N512_S3_zmin_noclip", 4, 512, 3, None, True, 0.1, False, UPS),
    ("d6_N4096_S3_shared_res", 6, 4096, 3, "shared", False, 0.1, True, ("res",)),
    ("d6_N4096_S1_zmin_tensor_jac", 6, 4096, 1, "tensor", True, 0.0, True, ("jac",)),
    ("d4_N4096_S64_out_cost", 4, 4096, 64, None, False, 0.1, True, ("cost",)),
    ("d6_N16384_S3_zmin_scalar_noclip", 6, 16384, 3, "scalar", True, 0.1, False, UPS),
    ("d4_N16384_S1_tensor", 4, 16384, 1, "tensor", False, 0.1, True, UPS),
    ("d6_N65536_S1_tensor_out", 6, 65536, 1, "tensor", False, 0.1, True, UPS),
    ("d4_N65536_S3_zmin", 4, 65536, 3, None, True, 0.1, True, ("res", "jac")),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_evaluate_gradient_matrix(cuda_device, case):
    cid, dof, N, S, bounds, zmin, outliers, clip, ups = case
    c = build_case(dof, N, S, bounds=bounds, zmin=zmin, outliers=outliers, clip=clip, ups=ups, dev=cuda_device)
    got = run_kernel(c)
    g64, fr = reference(c, torch.float64, census=True)
    g32, _ = reference(c, torch.float32)
    if bounds:
        assert 0.03 <= fr["clamped"] <= 0.25, fr
    if zmin:
        assert 0.05 <= fr["below_zmin"] <= 0.3, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if outliers:
        assert 0.01 <= fr["outlier"] <= 0.99, fr            # both Huber branches
    stats = assert_per_object(got, g64, g32, cid)
    record_parity(f"evaluate_grad/{cid}", B=c["B"], N=N, S=S, dof=dof, bounds=bounds or "none", clip=clip,
                  upstreams="+".join(ups), bound_k=bm.K_FLOOR, rel_min=bm.REL_MIN, **fr, **c["margins"], **stats)


def test_matrix_spans_its_conditions(cuda_device):
    assert max(c[2] for c in CASES) > native.max_points_split(6)
    assert {c[2] for c in CASES} >= {1, 7, 512, 4096, 16384, 65536} and {c[3] for c in CASES} == {1, 3, 64}
    assert {c[4] for c in CASES} == {None, "scalar", "tensor", "shared"} and {c[1] for c in CASES} == {4, 6}
    assert {c[7] for c in CASES} == {True, False}
    assert {c[8] for c in CASES} >= {("res",), ("jac",), ("cost",), UPS}


def _row(c, b):
    one = {k: (v[b:b + 1].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v)
           for k, v in c.items()}
    one["poses"] = c["poses"][:, b:b + 1].contiguous()
    one["ups"] = {k: None if v is None else v[:, b:b + 1].contiguous() for k, v in c["ups"].items()}
    return dict(one, B=1)


def exact_properties(c):
    """An object alone equals its row of the batch; asking for one gradient equals asking for all; a zero upstream gives
    zero; two runs give the same bits."""
    full = run_kernel(c)
    for a, b in zip(full, run_kernel(c)):
        assert a is None or torch.equal(a, b)
    for b in (0, c["B"] - 1):
        for i, (x, y) in enumerate(zip(run_kernel(_row(c, b)), full)):
            if x is not None:
                assert torch.equal(x, y[:, b:b + 1] if i == 4 else y[b:b + 1]), (b, INPUTS[i])
    for i in range(8):
        if full[i] is None:
            continue
        part = run_kernel(c, want=tuple(j == i for j in range(8)))
        assert torch.equal(part[i], full[i]) and all(p is None for j, p in enumerate(part) if j != i), INPUTS[i]
    zero = run_kernel(c, ups={k: None if v is None else torch.zeros_like(v) for k, v in c["ups"].items()})
    assert all(z is None or not z.abs().any() for z in zero)
    return full


def test_exact_properties(cuda_device):
    for dof, N, S, bounds in ((6, 513, 3, "tensor"), (4, 4100, 2, "tensor")):
        exact_properties(build_case(dof, N, S, B=4, bounds=bounds, outliers=0.1, dev=cuda_device))


def _layer_inputs(c, requires=True):
    leaf = lambda t: t.clone().requires_grad_(requires) if torch.is_tensor(t) else t
    camera = PerspectiveCamera(cam_mats=leaf(c["cam_mats"]), z_min=c["z_min"], lb=leaf(c["lb"]), ub=leaf(c["ub"]))
    return ([leaf(c[k]) for k in ("x3d", "x2d", "w2d")], leaf(c["poses"]), camera,
            HuberPnPCost(delta=leaf(c["delta"]), eps=HUBER_EPS))


def test_evaluate_pnp_forward_equals_no_grad_and_routes_to_the_kernel(cuda_device):
    """Under autograd, evaluate_pnp's values are the no-grad call's bits, stacked or not, and its gradients are the
    kernel's, reduced to the inputs' shapes."""
    c = build_case(6, 300, 3, B=3, bounds="tensor", outliers=0.1, dev=cuda_device)
    (x3d, x2d, w2d), poses, camera, cost_fun = _layer_inputs(c)
    for pose in (poses, poses[0]):
        kw = dict(out_residual=True, out_jacobian=True, out_cost=True)
        with torch.no_grad():
            plain = evaluate_pnp(x3d, x2d, w2d, pose, camera, cost_fun, **kw)
        live = evaluate_pnp(x3d, x2d, w2d, pose, camera, cost_fun, **kw)
        assert all(t.grad_fn is not None for t in live)
        for a, b in zip(live, plain):
            assert torch.equal(a.detach(), b)
    r, cost, j = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_residual=True, out_jacobian=True,
                              out_cost=True)
    u = c["ups"]
    ((r * u["res"]).sum() + (j * u["jac"]).sum() + (cost * u["cost"]).sum()).backward()
    direct = run_kernel(c)
    got = [x3d.grad, x2d.grad, w2d.grad, cost_fun.delta.grad, poses.grad, camera.cam_mats.grad, camera.lb.grad,
           camera.ub.grad]
    for i, (a, b) in enumerate(zip(got, direct)):
        assert torch.equal(a, b), INPUTS[i]
    with pytest.raises(RuntimeError):                   # first order only
        r2 = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_residual=True)[0]
        g = torch.autograd.grad(r2.sum(), x3d, create_graph=True)[0]
        g.sum().backward()


def test_graph_replay_equals_eager(cuda_device):
    c = build_case(6, 512, 3, B=4, bounds="tensor", outliers=0.1, dev=cuda_device)
    (x3d, x2d, w2d), poses, camera, cost_fun = _layer_inputs(c)

    def step():
        r, cost, j = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_residual=True, out_jacobian=True,
                                  out_cost=True)
        loss = (r * c["ups"]["res"]).sum() + (j * c["ups"]["jac"]).sum() + (cost * c["ups"]["cost"]).sum()
        return torch.autograd.grad(loss, [x3d, x2d, w2d, poses, camera.cam_mats, camera.lb, cost_fun.delta])
    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream(cuda_device)
    side.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(cuda_device).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize(cuda_device)
    for a, b in zip(captured, eager):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dof,N,bounds", [(6, 513, True), (4, 4096, True), (6, 16384, False)])
def test_gn_step_under_autograd_agrees_with_pose_plus(cuda_device, dof, N, bounds):
    """pose (+) LMSolver.gn_step(pose) under autograd runs the new kernel; _PosePlus runs the validated gn_plus_backward
    kernels: the same gradients within the matrix's bound (the float32 floor: the float64 composite against float32)."""
    case = dict(dof=dof, N=N, bounds=bounds, outliers=0.1)
    c, gp = bm.build_gn_case(case, cuda_device)
    solver = LMSolver(dof=dof, eps=bm.EPS)

    def grads(native_step, dtype=torch.float32):
        leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
        x3d, x2d, w2d, delta = (leaf(c[k]) for k in ("x3d", "x2d", "w2d", "delta"))
        K = leaf(c["cam_mats"])
        lb, ub = (leaf(c[k]) if torch.is_tensor(c[k]) else c[k] for k in ("lb", "ub"))
        camera = PerspectiveCamera(cam_mats=K, z_min=c["z_min"], lb=lb, ub=ub)
        cost_fun = HuberPnPCost(delta=delta, eps=HUBER_EPS)
        pose = c["pose"].detach().to(dtype)
        if native_step == "gn_step":
            plus = solver.pose_add(pose, solver.gn_step(x3d, x2d, w2d, pose, camera, cost_fun), camera)
        elif native_step == "pose_plus":
            params = solver.native_params(camera, cost_fun, False)
            params.lm_iter = 0
            plus = ag._PosePlus.apply(x3d, x2d, w2d, delta, K, lb, ub, pose, params, HUBER_EPS)
        else:
            plus = solver.pose_add(pose, ag.gn_step_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun), camera)
        (plus * gp.to(dtype)).sum().backward()
        return [t.grad for t in (x3d, x2d, w2d, delta)] + [K.grad] + [t.grad if torch.is_tensor(t) else None
                                                                     for t in (lb, ub)]
    new, old = grads("gn_step"), grads("pose_plus")
    c64, c32 = grads("composite", torch.float64), grads("composite", torch.float32)
    names = ("x3d", "x2d", "w2d", "delta", "cam", "lb", "ub")
    stats = {}
    for name, a, b, r64, r32 in zip(names, new, old, c64, c32):
        if a is None:
            continue
        assert torch.isfinite(a).all(), name
        floor = bm.per_object(r32, r64)
        bound = np.maximum(bm.REL_MIN, bm.K_FLOOR * floor) * (10 if name == "delta" else 1)
        err = bm.per_object(a, b)
        assert (err < bound).all(), (name, err.tolist(), floor.tolist())
        stats[f"{name}_rel_max_vs_pose_plus"] = float(err.max())
    record_parity(f"evaluate_grad/gn_step/d{dof}_N{N}", bound_k=bm.K_FLOOR, rel_min=bm.REL_MIN, **stats)
