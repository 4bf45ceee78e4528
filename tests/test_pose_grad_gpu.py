"""The pose gradient of the cost (epnp_cost_pose_backward_f32 and its cluster-split form) against float64 autograd, per
object and per pose, in the manner of test_backward_matrix_gpu.py (whose case builders and clamp placement this file
uses).

The resident kernel walks the poses in tiles of its 128 threads, the split kernel in tiles of 512 exchanged in passes
of 128; the matrix puts a case on each side of those boundaries and of the resident point limit, in 6DoF and 4DoF,
unbounded, with scalar and per-object bounds, with depths below z_min, both Huber branches and non-unit quaternions.
The reference is the oracle's float64 autograd with respect to the poses (pinned to the reference's own autograd by
test_oracle_cost_pose_grad_cpu.py); the bound is max|a - b| / max|b| within ONE pose's gradient under
max(2e-4, 5 * floor), floor = the same autograd in float32 for that pose.

Then the exact properties of a kernel in which each thread owns its row, and the layer: evaluate_pnp and
monte_carlo_forward hand the kernels' gradients to autograd, at sizes the torch composite cannot run, and under CUDA
graph capture."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import AdaptiveHuberPnPCost, HuberPnPCost
from epropnp.epropnp import EProPnP4DoF, EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

TILE = 128                  # poses per tile of cost_pose_backward_kernel (NT)
SPLIT_TILE = 512            # COST_SPLIT_TILE


def pose_grads(c, dtype, census=False):
    """up[b, p] * d cost_b(poses[b, p]) / d poses[b, p] (B, P, D) by the oracle's autograd in `dtype`, in chunks."""
    B, P, N = c["B"], c["P"], c["N"]
    ob = max(1, min(B, bm.CHUNK // (N * P) if N * P < bm.CHUNK else 1))
    pp = max(1, min(P, bm.CHUNK // (N * ob)))
    out = torch.zeros(B, P, c["poses"].shape[-1], dtype=dtype, device=c["poses"].device)
    counts = torch.zeros(3, dtype=torch.float64)
    for b0 in range(0, B, ob):
        sl = slice(b0, min(B, b0 + ob))
        x3d, x2d, w2d, delta = (c[k][sl].to(dtype) for k in ("x3d", "x2d", "w2d", "delta"))
        cam = bm._camera(c["cam_mats"], c["z_min"], c["lb"], c["ub"], sl, dtype)
        for p0 in range(0, P, pp):
            ps = c["poses"][sl, p0:p0 + pp].transpose(0, 1).to(dtype).clone().requires_grad_(True)
            cost = orc.evaluate(x3d, x2d, w2d, ps, cam, delta)["cost"]
            (cost * c["up"][sl, p0:p0 + pp].T.to(dtype)).sum().backward()
            out[sl, p0:p0 + pp] = ps.grad.transpose(0, 1)
            if census:
                with torch.no_grad():
                    zh, u = bm.project(x3d, ps, cam.cam_mats, c["z_min"])
                    counts[0] += float((zh < c["z_min"]).sum())
                    if cam.lb is not None:
                        lo, hi = orc._bound(cam.lb, u), orc._bound(cam.ub, u)
                        counts[1] += float(((u < lo) | (u > hi)).any(-1).sum())
                        u = torch.minimum(torch.maximum(u, lo), hi)
                    counts[2] += float((((u - x2d) * w2d).norm(dim=-1) > delta[:, None]).sum())
    fr = (counts / (B * P * N)).tolist()
    return out, dict(below_zmin=fr[0], clamped=fr[1], outlier=fr[2])


def per_pose(a, b):
    """max|a - b| / max|b| within every pose's gradient (last axis); 0 where both are zero."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().amax(-1) / b.abs().amax(-1).clamp(min=1e-300)).numpy()


def assert_per_pose(got, g64, g32, what):
    assert torch.isfinite(got).all(), what
    err, floor = per_pose(got, g64), per_pose(g32, g64)
    bound = np.maximum(bm.REL_MIN, bm.K_FLOOR * floor)
    bad = np.argwhere(err >= bound)
    assert bad.size == 0, (what, bad[:6].tolist(), [float(err[tuple(i)]) for i in bad[:6]],
                           [float(floor[tuple(i)]) for i in bad[:6]])
    return dict(grad_pose_rel_max_per_pose=float(err.max()), f32_oracle_floor_max=float(floor.max()),
                grad_pose_over_bound_max=float((err / bound).max()))


# N: a number, "max" = max_points(dof) (the largest resident object) or "max+4" (the smallest split one); B = mult * G
# + add with G = 4 * SMs (more CTAs than the device holds at once); nonunit: quaternions of norm 0.8 .. 1.25.  Bounds and
# depth offsets go where an object has at most some 600 000 (pose, point) pairs: beyond that no gap between their
# float64 projections is wide enough to place one with the margin asserted.
CASES = [
    dict(id="d6_N1_P1_B1", dof=6, bounds=None, N=1, P=1, B=(0, 1)),
    dict(id="d6_tensor_N511_P127_Gp1", dof=6, bounds="tensor", N=511, P=TILE - 1, B=(1, 1), outliers=0.1),
    dict(id="d4_tensor_N512_P128_B3", dof=4, bounds="tensor", N=512, P=TILE, B=(0, 3), outliers=0.1),
    dict(id="d6_tensor_nonunit_N513_P129_B2", dof=6, bounds="tensor", N=513, P=TILE + 1, B=(0, 2), outliers=0.1,
         nonunit=True),
    dict(id="d6_N4096_P259_B2", dof=6, bounds=None, N=4096, P=2 * TILE + 3, B=(0, 2), outliers=0.1),
    dict(id="d6_zmin_N1000_P129_B2", dof=6, bounds=None, N=1000, P=TILE + 1, B=(0, 2), zmin=True, outliers=0.1),
    dict(id="d4_zmin_scalar_Nmax_P1_B2", dof=4, bounds="scalar", N="max", P=1, B=(0, 2), zmin=True),
    dict(id="d6_Nmax4_P511_B2", dof=6, bounds=None, N="max+4", P=SPLIT_TILE - 1, B=(0, 2), outliers=0.1, split=True),
    dict(id="d4_zmin_tensor_Nmax4_P33_B2", dof=4, bounds="tensor", N="max+4", P=33, B=(0, 2), zmin=True, outliers=0.1,
         split=True),
    dict(id="d4_Nmax4_P513_B1", dof=4, bounds=None, N="max+4", P=SPLIT_TILE + 1, B=(0, 1), outliers=0.1, split=True),
    dict(id="d4_N8192_P512_B1", dof=4, bounds=None, N=8192, P=SPLIT_TILE, B=(0, 1), split=True),
    dict(id="d6_nonunit_N16384_P1027_B2", dof=6, bounds=None, N=16384, P=2 * SPLIT_TILE + 3, B=(0, 2), outliers=0.1,
         nonunit=True, split=True),
    dict(id="d6_tensor_N16384_P33_B3", dof=6, bounds="tensor", N=16384, P=33, B=(0, 3), outliers=0.1, split=True),
]


def upstream(B, P, gen):
    """Upstream gradients of mixed sign, about 10 % exact zeros where an object has several poses, times a per-object
    scale of 1 .. 1e-6.  (Every pose is judged on its own here, so none is given a weight near the float32 denormals.)"""
    up = torch.randn(B, P, generator=gen)
    up = torch.where(up.abs() < 0.05, torch.full_like(up, 0.05), up)
    if P > 1:
        up = up.masked_fill(torch.rand(B, P, generator=gen) < 0.1, 0.0)
    return up * 10.0 ** (-6.0 * torch.rand(B, 1, generator=gen))


def build_case(case, dev, seed=11):
    N = case["N"]
    if isinstance(N, str):
        N = native.max_points(case["dof"]) + (4 if N.endswith("+4") else 0)
    G = bm.resident_grid(dev)
    B, P, dof = case["B"][0] * G + case["B"][1], case["P"], case["dof"]
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=case.get("outliers", 0.0))
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, P, 1)
    poses[..., :3] += 0.03 * torch.randn(B, P, 3, generator=gen)
    if dof == 6:
        q = poses[..., 3:] + 0.02 * torch.randn(B, P, 4, generator=gen)
        q = q / q.norm(dim=-1, keepdim=True)
        if case.get("nonunit"):
            q = q * (0.8 + 0.45 * torch.rand(B, P, 1, generator=gen))
        poses[..., 3:] = q
    else:
        poses[..., 3] += 0.05 * torch.randn(B, P, generator=gen)
    c = {k: v.to(dev) for k, v in pc.items()}
    c.update(B=B, N=N, P=P, dof=dof, poses=poses.to(dev), up=upstream(B, P, gen).to(dev), z_min=0.1, lb=None, ub=None)
    margins = {}
    if case.get("zmin"):
        c["z_min"] = 4.0
        c["poses"], margins["zmin_margin"] = bm.place_depths(c["x3d"], c["poses"], c["cam_mats"], c["z_min"])
        assert margins["zmin_margin"] > bm.ZMIN_GAP, margins
    if case["bounds"]:
        c["lb"], c["ub"], margins["bound_margin"] = bm.place_bounds(c["x3d"], c["poses"], c["cam_mats"], c["z_min"],
                                                                    case["bounds"] == "tensor")
        assert margins["bound_margin"] > bm.BOUND_GAP, margins
    c["delta"] = native.adaptive_delta(c["x2d"], c["w2d"], 0.5) if N > 1 else torch.full((B,), 4.0, device=dev)
    c["margins"] = margins
    return c


def run_kernel(c, **over):
    x = dict(c, **over)
    prob = native.Problem(x["x3d"], x["x2d"], x["w2d"], x["cam_mats"], x["lb"], x["ub"], x["delta"])
    return native.cost_pose_backward(prob, x["dof"], x["z_min"], x["poses"], x["up"], x.get("cluster_ctas", 0))


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_pose_gradient_matrix(cuda_device, case):
    c = build_case(case, cuda_device)
    assert (c["N"] > native.max_points(c["dof"])) == bool(case.get("split"))
    got = run_kernel(c)
    g64, fr = pose_grads(c, torch.float64, census=True)
    g32, _ = pose_grads(c, torch.float32)
    if case["bounds"]:
        assert 0.03 <= fr["clamped"] <= 0.25, fr
    if case.get("zmin"):
        assert 0.05 <= fr["below_zmin"] <= 0.3, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if case.get("outliers"):
        assert 0.01 <= fr["outlier"] <= 0.99, fr
    if case.get("nonunit"):
        assert float((c["poses"][..., 3:].norm(dim=-1) - 1).abs().max()) > 0.1
    stats = assert_per_pose(got, g64, g32, case["id"])
    record_parity(f"pose_grad/{case['id']}", B=c["B"], N=c["N"], P=c["P"], dof=c["dof"],
                  bounds=case["bounds"] or "none", split=bool(case.get("split")), bound_k=bm.K_FLOOR,
                  rel_min=bm.REL_MIN, **fr, **c["margins"], **stats)


def test_exact_properties_resident(cuda_device):
    """Each thread owns its row: an object alone equals its row of the batch, the plain loader equals the TMA path,
    P poses at once equal P calls of one."""
    c = build_case(dict(dof=6, bounds="tensor", N=512, P=TILE + 2, B=(0, 5), outliers=0.1), cuda_device)
    full = run_kernel(c)
    pick = lambda b: {k: (v[b:b + 1].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v)
                      for k, v in c.items()}
    for b in (0, 3):
        one = pick(b)
        one["B"] = 1
        assert torch.equal(run_kernel(one), full[b:b + 1])
    off = {}
    for k in ("x3d", "x2d", "w2d"):                     # 4-byte offset: not 16-byte aligned -> the plain loader
        flat = torch.empty(c[k].numel() + 1, device=cuda_device)
        flat[1:] = c[k].reshape(-1)
        off[k] = flat[1:].view(c[k].shape)
        assert off[k].data_ptr() % 16 != 0 and off[k].is_contiguous()
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    prob.x3d, prob.x2d, prob.w2d = off["x3d"], off["x2d"], off["w2d"]
    assert torch.equal(native.cost_pose_backward(prob, 6, c["z_min"], c["poses"], c["up"]), full)
    for p in (0, TILE - 1, TILE, TILE + 1):
        single = run_kernel(c, poses=c["poses"][:, p:p + 1].contiguous(), up=c["up"][:, p:p + 1].contiguous(), P=1)
        assert torch.equal(single, full[:, p:p + 1])


def test_exact_properties_split(cuda_device):
    """A repeated split call gives the same bits, for every object whatever the batch; at N = 4096 on C = 2 the split
    result differs from the resident one by fp32 rounding only."""
    c = build_case(dict(dof=6, bounds=None, N="max+4", P=SPLIT_TILE + 5, B=(0, 3), outliers=0.1), cuda_device)
    a, b = run_kernel(c), run_kernel(c)
    assert torch.equal(a, b)
    one = {k: (v[1:2].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == 3 else v) for k, v in c.items()}
    one["B"] = 1
    assert torch.equal(run_kernel(one), a[1:2])
    d = build_case(dict(dof=6, bounds="tensor", N=4096, P=TILE + 1, B=(0, 2), outliers=0.1), cuda_device)
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], d["lb"], d["ub"], d["delta"])
    res = native.cost_pose_backward(prob, 6, d["z_min"], d["poses"], d["up"])
    out = prob.empty(*res.shape)
    import ctypes
    native.check(native.lib().epnp_cost_pose_backward_split_f32(
        *prob.common_ptrs(), native.ptr(d["poses"]), native.ptr(d["up"]), native.ptr(out), d["P"], d["B"], d["N"], 6,
        ctypes.c_float(d["z_min"]), 2, native.stream_ptr(cuda_device)), "epnp_cost_pose_backward_split_f32")
    err = per_pose(out, res)
    assert 0 < err.max() < 2e-5, err.max()
    record_parity("pose_grad/split_vs_resident_N4096_C2", rel_max_per_pose=float(err.max()))


def _layer_case(dev, dof, B, N, seed=5):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.1)
    x3d, x2d, w2d = (pc[k].to(dev) for k in ("x3d", "x2d", "w2d"))
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"].to(dev), z_min=0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(x2d, w2d)
    return pc, x3d, x2d, w2d, camera, cost_fun


@pytest.mark.parametrize("dof,N", [(6, 512), (4, 256), (6, 16384)])
def test_monte_carlo_forward_differentiates_cost_init(cuda_device, dof, N):
    """pose_init.grad of monte_carlo_forward's cost_init = the kernel's direct result; with the correspondences also
    requiring grad the step returns every gradient, the correspondences' unchanged by the pose's presence."""
    dev, B, M = cuda_device, 4, 128
    pc, x3d, x2d, w2d, camera, cost_fun = _layer_case(dev, dof, B, N)
    layer = (EProPnP6DoF if dof == 6 else EProPnP4DoF)(mc_samples=M, num_iter=4, solver=LMSolver(dof=dof, num_iter=5))
    coef = torch.randn(B, generator=torch.Generator().manual_seed(1)).to(dev)
    pose_init = pc["pose_init"].to(dev).requires_grad_(True)
    out = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=pose_init, force_init_solve=False,
                                    amis_seed=3)
    pose_opt, samples, logw, cost_init = out[0], out[3], out[4], out[5]
    assert cost_init.requires_grad and not pose_opt.requires_grad and not samples.requires_grad
    (coef * cost_init).sum().backward()
    prob = native.Problem(x3d, x2d, w2d, camera.cam_mats, None, None, cost_fun.delta)
    direct = native.cost_pose_backward(prob, dof, 0.1, pose_init.detach()[:, None].contiguous(), coef[:, None])[:, 0]
    assert torch.equal(pose_init.grad, direct) and pose_init.grad.abs().sum() > 0
    # a training step: pose and correspondences
    leaves = [t.clone().requires_grad_(True) for t in (x3d, x2d, w2d)]
    pose2 = pc["pose_init"].to(dev).requires_grad_(True)
    out = layer.monte_carlo_forward(*leaves, camera, cost_fun, pose_init=pose2, force_init_solve=False, amis_seed=3)
    loss = (coef * out[5]).sum() + torch.logsumexp(out[4], dim=0).sum()
    loss.backward()
    assert torch.equal(pose2.grad, direct)
    for t in leaves:
        assert t.grad is not None and torch.isfinite(t.grad).all() and t.grad.abs().sum() > 0
    ref = [t.clone().requires_grad_(True) for t in (x3d, x2d, w2d)]
    out = layer.monte_carlo_forward(*ref, camera, cost_fun, pose_init=pc["pose_init"].to(dev), force_init_solve=False,
                                    amis_seed=3)
    ((coef * out[5]).sum() + torch.logsumexp(out[4], dim=0).sum()).backward()
    for t, r in zip(leaves, ref):
        assert torch.equal(t.grad, r.grad)


def test_evaluate_pnp_takes_the_native_pose_gradient(cuda_device, monkeypatch):
    """evaluate_pnp(out_cost=True) with a pose that requires grad runs the kernel (not the composite), and agrees with
    the float64 composite; float64 inputs keep the composite."""
    dev, B, S = cuda_device, 3, 5
    pc, x3d, x2d, w2d, camera, cost_fun = _layer_case(dev, 6, B, 300)
    poses = pc["pose_gt"].to(dev)[None].repeat(S, 1, 1)
    poses[..., :3] += 0.03 * torch.randn(S, B, 3, device=dev)
    calls = []
    real = native.cost_pose_backward
    monkeypatch.setattr(native, "cost_pose_backward", lambda *a, **k: calls.append(1) or real(*a, **k))
    pg = poses.clone().requires_grad_(True)
    cost = evaluate_pnp(x3d, x2d, w2d, pg, camera, cost_fun, out_cost=True)[1]
    up = torch.randn(S, B, device=dev)
    (cost * up).sum().backward()
    assert calls == [1]
    d = torch.float64
    p64 = poses.to(d).requires_grad_(True)
    cam64 = PerspectiveCamera(cam_mats=camera.cam_mats.to(d), z_min=0.1)
    c64 = evaluate_pnp(x3d.to(d), x2d.to(d), w2d.to(d), p64, cam64, HuberPnPCost(delta=cost_fun.delta.to(d)),
                       out_cost=True)[1]
    (c64 * up.to(d)).sum().backward()
    assert calls == [1]
    assert per_pose(pg.grad, p64.grad).max() < 2e-4


def test_stack_of_hypotheses_at_dense_size(cuda_device):
    """(512, 32, 7) hypotheses on N = 16 384 points: 3.2 GB per intermediate for the composite; the kernel's working set
    is the inputs and the output."""
    dev, B, N, S = cuda_device, 32, 16384, 512
    pc, x3d, x2d, w2d, camera, cost_fun = _layer_case(dev, 6, B, N)
    poses = pc["pose_gt"].to(dev)[None].repeat(S, 1, 1)
    poses[..., :3] += 0.03 * torch.randn(S, B, 3, device=dev)
    poses.requires_grad_(True)
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    cost = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_cost=True)[1]
    cost.sum().backward()
    torch.cuda.synchronize(dev)
    assert poses.grad.shape == (S, B, 7) and torch.isfinite(poses.grad).all() and (poses.grad.abs().amax(-1) > 0).all()
    assert torch.cuda.max_memory_allocated(dev) - base < 64 << 20
    # a few rows against float64
    c = dict(B=2, N=N, P=3, x3d=x3d[:2], x2d=x2d[:2], w2d=w2d[:2], cam_mats=camera.cam_mats[:2], lb=None, ub=None,
             delta=cost_fun.delta[:2], z_min=0.1, poses=poses.detach()[:3, :2].transpose(0, 1).contiguous(),
             up=torch.ones(2, 3, device=dev))
    g64, _ = pose_grads(c, torch.float64)
    g32, _ = pose_grads(c, torch.float32)
    assert_per_pose(poses.grad[:3, :2].transpose(0, 1), g64, g32, "stack")


@pytest.mark.parametrize("N", [512, 8192])
def test_backward_replays_under_graph_capture(cuda_device, N):
    dev, B, S = cuda_device, 4, 130
    pc, x3d, x2d, w2d, camera, cost_fun = _layer_case(dev, 6, B, N)
    poses = pc["pose_gt"].to(dev)[None].repeat(S, 1, 1).contiguous().requires_grad_(True)
    up = torch.randn(S, B, device=dev)

    def step():
        cost = evaluate_pnp(x3d, x2d, w2d, poses, camera, cost_fun, out_cost=True)[1]
        return torch.autograd.grad((cost * up).sum(), poses)[0]
    eager = step().clone()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    with torch.no_grad():
        poses[..., :3] += 0.01
    graph.replay()
    torch.cuda.synchronize(dev)
    moved = step()
    assert torch.equal(captured, moved) and not torch.equal(moved, eager)
