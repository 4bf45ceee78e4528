"""The camera gradients (epnp_cost_camera_backward_f32, epnp_gn_plus_camera_backward_f32 and their cluster-split forms)
against float64 autograd, per object, in the manner of test_backward_matrix_gpu.py (whose case builders and clamp
placement this file uses).

The cost backward sums over the poses of an object, so the reference is the oracle's float64 autograd with respect to
cam_mats and the tensor bounds (pinned to the reference's own autograd by test_oracle_cost_camera_grad_cpu.py).  The
bound is max|a - b| / max|b| within one object's gradient of one output under max(2e-4, 5 * floor), floor = the same
autograd in float32 for that object.  The matrix crosses the pose tiles (128 threads resident, 512 split), the
resident point limit, batches on either side of the grid, 6DoF and 4DoF, scalar and per-object bounds, depths below
z_min, both Huber branches, and the Monte-Carlo form (512 samples and the cost_init pose in one launch).

Then the layer: the 6DoF training step of EPro-PnP-6DoF/lib/train.py with a camera and bounds that require grad against
a float64 reference built from the kernels' own samples, exact properties, and CUDA-graph replay."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
import test_pose_grad_gpu as pg
from conftest import record_parity
from oracle import pnp_oracle as orc
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.epropnp import EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

OUTPUTS = ("cam", "lb", "ub")
EPS, HUBER_EPS = 1e-5, 1e-10


def camera_grads(c, dtype, census=False):
    """sum_p up[b, p] * d cost_b(poses[b, p]) / d (cam_mats[b], lb[b], ub[b]) by the oracle's autograd in `dtype`, in
    chunks of objects and poses (linear in `up`).  -> [(B, 3, 3), (B, 2) | None, (B, 2) | None], census fractions."""
    B, P, N = c["B"], c["P"], c["N"]
    ob = max(1, min(B, bm.CHUNK // (N * P) if N * P < bm.CHUNK else 1))
    pp = max(1, min(P, bm.CHUNK // (N * ob)))
    tensor_bounds = torch.is_tensor(c["lb"])
    out = [torch.zeros(B, 3, 3, dtype=dtype, device=c["x3d"].device)]
    out += [torch.zeros(B, 2, dtype=dtype, device=c["x3d"].device) if tensor_bounds else None for _ in range(2)]
    counts = torch.zeros(3, dtype=torch.float64)
    for b0 in range(0, B, ob):
        sl = slice(b0, min(B, b0 + ob))
        x3d, x2d, w2d, delta = (c[k][sl].to(dtype) for k in ("x3d", "x2d", "w2d", "delta"))
        leaves = [c["cam_mats"][sl].to(dtype).clone().requires_grad_(True)]
        leaves += [c[k][sl].to(dtype).clone().requires_grad_(True) if tensor_bounds else c[k] for k in ("lb", "ub")]
        cam = orc.Camera(leaves[0], c["z_min"], leaves[1], leaves[2])
        for p0 in range(0, P, pp):
            ps = c["poses"][sl, p0:p0 + pp].transpose(0, 1).to(dtype)
            cost = orc.evaluate(x3d, x2d, w2d, ps, cam, delta)["cost"]
            (cost * c["up"][sl, p0:p0 + pp].T.to(dtype)).sum().backward()
            if census:
                with torch.no_grad():
                    zh, u = bm.project(x3d, ps, cam.cam_mats, c["z_min"])
                    counts[0] += float((zh < c["z_min"]).sum())
                    if cam.lb is not None:
                        lo, hi = orc._bound(cam.lb, u), orc._bound(cam.ub, u)
                        counts[1] += float(((u < lo) | (u > hi)).any(-1).sum())
                        u = torch.minimum(torch.maximum(u, lo), hi)
                    counts[2] += float((((u - x2d) * w2d).norm(dim=-1) > delta[:, None]).sum())
        for o, l in zip(out, leaves):
            if o is not None:
                o[sl] = l.grad
    fr = (counts / (B * P * N)).tolist()
    return out, dict(below_zmin=fr[0], clamped=fr[1], outlier=fr[2])


def assert_per_object(got, g64, g32, what, objs=None):
    """got / g64 / g32: lists over OUTPUTS (None = not compared).  Returns the recorded numbers."""
    stats = {}
    for name, a, b, c in zip(OUTPUTS, got, g64, g32):
        if a is None or b is None:
            continue
        a = a[objs] if objs is not None else a
        assert torch.isfinite(a).all(), (what, name)
        err, floor = bm.per_object(a, b), bm.per_object(c, b)
        bound = np.maximum(bm.REL_MIN, bm.K_FLOOR * floor)
        bad = np.nonzero(err >= bound)[0]
        assert bad.size == 0, (what, name, bad[:8].tolist(), err[bad[:8]].tolist(), floor[bad[:8]].tolist())
        stats[f"grad_{name}_rel_max_per_object"] = float(err.max())
        stats[f"f32_oracle_floor_{name}_max"] = float(floor.max())
        stats[f"grad_{name}_over_bound_max"] = float((err / bound).max())
    return stats


def run_kernel(c, PA=None, **over):
    """native.cost_camera_backward on c's poses, the first PA as set a and the rest as set b (PA = None: all in a)."""
    x = dict(c, **over)
    prob = native.Problem(x["x3d"], x["x2d"], x["w2d"], x["cam_mats"], x["lb"], x["ub"], x["delta"])
    want = (True,) + (torch.is_tensor(x["lb"]),) * 2
    PA = x["P"] if PA is None else PA
    pa, ga = x["poses"][:, :PA].contiguous(), x["up"][:, :PA].contiguous()
    pb = gb = None
    if PA < x["P"]:
        pb, gb = x["poses"][:, PA:].contiguous(), x["up"][:, PA:].contiguous()
    return native.cost_camera_backward(prob, x["dof"], x["z_min"], pa, ga, pb, gb, want=want,
                                       cluster_ctas=x.get("cluster_ctas", 0))


# B = mult * G + add with G = 4 * SMs; N: a number, "max" = max_points(dof), "max+1" (the smallest split object);
# mc: the upstream of the Monte-Carlo backward (P - 1 samples and the cost_init pose, in two sets).
CASES = [
    dict(id="d6_tensor_N511_P1_B1", dof=6, bounds="tensor", N=511, P=1, B=(0, 1)),
    dict(id="d6_tensor_N512_P128_Gm1", dof=6, bounds="tensor", N=512, P=128, B=(1, -1), outliers=0.1),
    dict(id="d4_N513_P129_Gp1", dof=4, bounds=None, N=513, P=129, B=(1, 1), outliers=0.1),
    dict(id="d6_scalar_N513_P129_B2", dof=6, bounds="scalar", N=513, P=129, B=(0, 2), outliers=0.1),
    dict(id="d6_mc_tensor_N512_M512_B3", dof=6, bounds="tensor", N=512, P=513, B=(0, 3), outliers=0.1, mc=True),
    dict(id="d4_mc_zmin_N513_M512_B2", dof=4, bounds=None, N=513, P=513, B=(0, 2), zmin=True, outliers=0.1, mc=True),
    dict(id="d6_zmin_tensor_N1000_P129_B2", dof=6, bounds="tensor", N=1000, P=129, B=(0, 2), zmin=True),
    dict(id="d4_N511_P1025_B2", dof=4, bounds=None, N=511, P=1025, B=(0, 2), outliers=0.1),
    dict(id="d6_tensor_Nmax_P33_B2", dof=6, bounds="tensor", N="max", P=33, B=(0, 2), outliers=0.1),
    dict(id="d6_tensor_Nmax1_P33_B2", dof=6, bounds="tensor", N="max+1", P=33, B=(0, 2), outliers=0.1, split=True),
    dict(id="d4_zmin_Nmax1_P129_B2", dof=4, bounds=None, N="max+1", P=129, B=(0, 2), zmin=True, split=True),
    dict(id="d6_mc_N16384_M512_B2", dof=6, bounds=None, N=16384, P=513, B=(0, 2), outliers=0.1, mc=True, split=True),
    dict(id="d4_tensor_N16384_P33_B3", dof=4, bounds="tensor", N=16384, P=33, B=(0, 3), outliers=0.1, split=True),
]


def build_case(case, dev, seed=13):
    N = case["N"]
    if isinstance(N, str):
        N = native.max_points(case["dof"]) + (1 if N.endswith("+1") else 0)
    c = pg.build_case(dict(case, N=N), dev, seed=seed)
    if case.get("mc"):         # softmax-weighted samples first, the cost_init pose last
        gen = torch.Generator().manual_seed(seed + 2)
        c["up"] = bm.softmax_like(c["B"], c["P"] - 1, 1, gen).to(dev)
    return c


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_camera_gradient_matrix(cuda_device, case):
    c = build_case(case, cuda_device)
    assert (c["N"] > native.max_points(c["dof"])) == bool(case.get("split"))
    got = run_kernel(c, PA=c["P"] - 1 if case.get("mc") else None)
    g64, fr = camera_grads(c, torch.float64, census=True)
    g32, _ = camera_grads(c, torch.float32)
    if case["bounds"]:
        assert 0.03 <= fr["clamped"] <= 0.25, fr
    if case.get("zmin"):
        assert 0.05 <= fr["below_zmin"] <= 0.3, fr
    else:
        assert fr["below_zmin"] == 0.0, fr
    if case.get("outliers"):
        assert 0.01 <= fr["outlier"] <= 0.99, fr
    if case["bounds"] == "tensor":
        assert (got[1].abs().amax(1) > 0).all() and (got[2].abs().amax(1) > 0).all()
    stats = assert_per_object(got, g64, g32, case["id"])
    record_parity(f"camera_grad/cost/{case['id']}", B=c["B"], N=c["N"], P=c["P"], dof=c["dof"],
                  bounds=case["bounds"] or "none", split=bool(case.get("split")), bound_k=bm.K_FLOOR,
                  rel_min=bm.REL_MIN, **fr, **c["margins"], **stats)


def gn_composite(c, gp, dtype):
    """dL/d(cam_mats, lb, ub) of L = <gp, pose (+) gn_step(pose)> through the torch composite, in `dtype`."""
    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
    K = leaf(c["cam_mats"])
    lb, ub = (leaf(c[k]) if torch.is_tensor(c[k]) else c[k] for k in ("lb", "ub"))
    cast = lambda k: c[k].detach().to(dtype)
    camera = PerspectiveCamera(cam_mats=K, z_min=c["z_min"], lb=lb, ub=ub)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1, eps=HUBER_EPS)
    cost_fun.delta = cast("delta")
    solver = LMSolver(dof=c["dof"], eps=EPS)
    pose = c["pose"].detach().to(dtype)
    plus = solver.pose_add(pose, ag.gn_step_autograd(solver, cast("x3d"), cast("x2d"), cast("w2d"), pose, camera,
                                                     cost_fun), camera)
    (plus * gp.to(dtype)).sum().backward()
    return [K.grad] + [t.grad if torch.is_tensor(t) else None for t in (lb, ub)]


GN_CASES = [
    dict(id="d6_N5_outlier", dof=6, N=5, bounds=False, outliers=0.2),
    dict(id="d6_N513_bounded_outliers", dof=6, N=513, bounds=True, outliers=0.1),
    dict(id="d4_N512_zmin_bounded", dof=4, N=512, bounds=True, zmin=True),
    dict(id="d6_Nmax_zmin", dof=6, N="max", bounds=False, zmin=True, outliers=0.1),
    dict(id="d6_N16384_bounded", dof=6, N=16384, bounds=True, outliers=0.1),
    dict(id="d4_N16384_zmin", dof=4, N=16384, bounds=False, zmin=True),
]


@pytest.mark.parametrize("case", GN_CASES, ids=[c["id"] for c in GN_CASES])
def test_gn_plus_camera_gradient_matrix(cuda_device, case):
    c, gp = bm.build_gn_case(case, cuda_device)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    want = (True, bool(case["bounds"]), bool(case["bounds"]))
    got = native.gn_plus_camera_backward(prob, c["pose"], gp, c["dof"], c["z_min"], EPS, HUBER_EPS, want=want)
    c64, c32 = gn_composite(c, gp, torch.float64), gn_composite(c, gp, torch.float32)
    with torch.no_grad():
        zh, u = bm.project(c["x3d"].double(), c["pose"][None].double(), c["cam_mats"].double(), c["z_min"])
        below = float((zh < c["z_min"]).double().mean())
        clamped = 0.0
        if case["bounds"]:
            clamped = float(((u < c["lb"].double()[None, :, None]) | (u > c["ub"].double()[None, :, None]))
                            .any(-1).double().mean())
    if case.get("zmin"):
        assert 0.05 <= below <= 0.3, below
    if case["bounds"]:
        assert 0.01 <= clamped <= 0.3, clamped
    stats = assert_per_object(list(got), c64, c32, case["id"])
    record_parity(f"camera_grad/gn_plus/{case['id']}", N=c["N"], dof=c["dof"], bound_k=bm.K_FLOOR, rel_min=bm.REL_MIN,
                  split=c["N"] > native.max_points(c["dof"]), below_zmin=below, clamped=clamped, **c["margins"],
                  **stats)


def test_exact_properties(cuda_device):
    """An object alone equals its row of the batch; two runs give the same bits; set b's poses in set a give the same
    sum order only when nothing else moves, so the two-set launch is checked against float64 by the matrix instead."""
    for N in (513, native.max_points(6) + 1):
        c = build_case(dict(dof=6, bounds="tensor", N=N, P=130 if N == 513 else 33, B=(0, 5), outliers=0.1),
                       cuda_device)
        full = run_kernel(c, PA=c["P"] - 1)
        again = run_kernel(c, PA=c["P"] - 1)
        for a, b in zip(full, again):
            assert torch.equal(a, b)
        for b in (0, 3):
            one = {k: (v[b:b + 1].contiguous() if torch.is_tensor(v) and v.dim() and v.shape[0] == c["B"] else v)
                   for k, v in c.items()}
            one["B"] = 1
            for x, y in zip(run_kernel(one, PA=c["P"] - 1), full):
                assert torch.equal(x, y[b:b + 1])


def _train_step(dev, B, N, M, camera_grad, seed=31):
    """The 6DoF objective of EPro-PnP-6DoF/lib/train.py: monte_carlo_forward(pose_init=gt, force_init_solve=True,
    with_pose_opt_plus=True), MonteCarloPoseLoss and the loss_t / loss_r terms on pose_opt_plus, with cam_mats expanded
    from one (3, 3) and per-object lb / ub (requiring grad when `camera_grad`)."""
    import test_gn_plus_split_gpu as gs
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=seed, grid2d=round(N ** 0.5) ** 2 == N).items()}
    lb0, ub0 = gs.train_bounds(pc["x2d"])
    K = pc["cam_mats"][0].clone().requires_grad_(camera_grad)
    lb, ub = lb0.clone().requires_grad_(camera_grad), ub0.clone().requires_grad_(camera_grad)
    camera = PerspectiveCamera(cam_mats=K[None].expand(B, -1, -1), z_min=0.01, lb=lb, ub=ub)
    x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(x2d, w2d)
    cost_fun.delta.retain_grad()                            # delta: a function of w2d, and compared on its own
    init = RSLMSolver(dof=6, num_points=16, num_proposals=64, num_iter=3, cluster_split=True)
    layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=5, init_solver=init))
    pose_gt = pc["pose_gt"].clone().requires_grad_(True)    # cost_init and the loss terms differentiate the pose too
    torch.manual_seed(seed)                                 # the RSLM draws: the same in every run
    pose_opt, _, plus, samples, logw, cost_tgt = layer.monte_carlo_forward(
        x3d, x2d, w2d, camera, cost_fun, pose_init=pose_gt, force_init_solve=True, with_pose_opt_plus=True, amis_seed=7)
    loss_mc = MonteCarloPoseLoss().to(dev)(logw, cost_tgt, torch.tensor(1.0, device=dev))
    loss_t = (plus[:, :3] - pose_gt[:, :3]).norm(dim=-1)
    loss_t = torch.where(loss_t < 0.05, 0.5 * loss_t.square() / 0.05, loss_t - 0.025).mean()
    loss_r = ((1 - (plus[:, None, 3:] @ pose_gt[:, 3:, None]).squeeze(-1).squeeze(-1).square()) * 2).mean()
    loss = loss_mc + loss_t + loss_r
    ups = torch.autograd.grad(loss, [logw, cost_tgt, plus], retain_graph=True)
    loss.backward()
    grads = [t.grad for t in (x3d, x2d, w2d, cost_fun.delta, pose_gt)]
    cam = [t.grad for t in (K, lb, ub)] if camera_grad else None
    return dict(pc=pc, K=K.detach()[None].expand(B, -1, -1).contiguous(), lb=lb0, ub=ub0, delta=cost_fun.delta.detach(),
                grads=grads, cam=cam, ups=ups,
                pose_opt=pose_opt.detach(), samples=samples.detach())


@pytest.mark.parametrize("N", [512, 16384])
def test_training_step_drop_in(cuda_device, N):
    dev, B, M = cuda_device, 8, 512
    run = _train_step(dev, B, N, M, True)
    plain = _train_step(dev, B, N, M, False)
    for a, b in zip(run["grads"], plain["grads"]):          # x3d, x2d, w2d, delta, pose: unmoved by the camera's
        assert a is not None and a.abs().sum() > 0 and torch.equal(a, b)
    pc = run["pc"]
    g_logw, g_cost, g_plus = run["ups"]
    poses = torch.cat((pc["pose_gt"][:, None], run["samples"].transpose(0, 1)), 1)
    up = torch.cat((g_cost.reshape(B, 1), -g_logw.T), 1)
    c = dict(B=B, N=N, P=M + 1, x3d=pc["x3d"], x2d=pc["x2d"], w2d=pc["w2d"], cam_mats=run["K"], lb=run["lb"],
             ub=run["ub"], delta=run["delta"], z_min=0.01, poses=poses, up=up)
    g = dict(c, dof=6, pose=run["pose_opt"])
    refs = []
    for dt in (torch.float64, torch.float32):
        mc, _ = camera_grads(c, dt)
        gn = gn_composite(g, g_plus, dt)
        refs.append([a + b for a, b in zip(mc, gn)])
    # the (3, 3) camera is shared: its gradient is the sum over objects, judged as one object
    got = [run["cam"][0][None], run["cam"][1], run["cam"][2]]
    ref64 = [refs[0][0].sum(0, keepdim=True), refs[0][1], refs[0][2]]
    ref32 = [refs[1][0].sum(0, keepdim=True), refs[1][1], refs[1][2]]
    stats = assert_per_object(got, ref64, ref32, f"train N={N}")
    record_parity(f"camera_grad/train/6dof_B{B}_N{N}_M{M}", bound_k=bm.K_FLOOR, rel_min=bm.REL_MIN, **stats)


def test_evaluate_pnp_with_only_the_camera_requiring_grad(cuda_device):
    pc = {k: v.to(cuda_device) for k, v in make_problem(3, 200, seed=3).items()}
    K = pc["cam_mats"].clone().requires_grad_(True)
    camera = PerspectiveCamera(cam_mats=K, z_min=0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    cost = evaluate_pnp(pc["x3d"], pc["x2d"], pc["w2d"], pc["pose_gt"], camera, cost_fun, out_cost=True)[1]
    assert cost.grad_fn is not None
    cost.sum().backward()
    assert K.grad is not None and torch.isfinite(K.grad).all() and K.grad.abs().sum() > 0


def test_training_step_replays_under_graph_capture(cuda_device):
    dev, B, N, M = cuda_device, 4, 512, 128
    pc = {k: v.to(dev) for k, v in make_problem(B, N, seed=5).items()}
    K = pc["cam_mats"][0].clone().requires_grad_(True)
    lb, ub = (t.clone().requires_grad_(True) for t in (pc["x2d"].amin(1) + 5.0, pc["x2d"].amax(1) - 5.0))
    x3d, x2d, w2d = (pc[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
    layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=5))

    def step():
        camera = PerspectiveCamera(cam_mats=K[None].expand(B, -1, -1), z_min=0.01, lb=lb, ub=ub)
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
        cost_fun.set_param(x2d, w2d)
        _, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun,
                                                                  pose_init=pc["pose_gt"], force_init_solve=False,
                                                                  with_pose_opt_plus=True, amis_seed=11)
        loss = (cost_tgt + torch.logsumexp(-logw, 0)).sum() + plus.square().sum()
        return torch.autograd.grad(loss, [K, lb, ub, x2d])
    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize(dev)
    for a, b in zip(captured, eager):
        assert torch.equal(a, b)
