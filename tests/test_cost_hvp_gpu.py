"""Second order through the cost: the Hessian-vector-product kernels (epnp_cost_hvp_f32) and the autograd formulas of
cost_backward, cost_pose_backward, cost_camera_backward and mc_lse_backward that call them.

The reference is the oracle's float64 double backward of f = sum_p g_p cost(pose_p): grad f with create_graph, then the
gradient of grad f . v with respect to every input and to g.  The oracle forms the rotation as the kernels do
(ww + xx - yy - zz, ...), so every block, quaternion-quaternion included, is compared as it is.  Bound: per object and
output (per pose for the pose rows), max|a - b| / max|b| under max(REL_MIN, K_FLOOR * floor), floor = the same double
backward in float32.  Depths and bounds are kept off their clamps and the residuals off the Huber threshold by margins,
as in the first-order tests.

Then the layer: evaluate_pnp(out_cost=True) and cost_init / the Monte-Carlo loss differentiated twice, the exact
properties (run-to-run bits, first order unchanged by create_graph, a third backward raises, CUDA-graph replay) and
torch.library.opcheck."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
from oracle import pnp_oracle as orc
from epropnp_b200 import native, ops
from epropnp_b200.synth import make_problem

K_FLOOR = 10
REL_MIN = 5e-4
HUBER_GAP = 1e-6            # least relative distance of a float64 residual norm from delta (8 float32 ulps)
TANGENTS = native.HVP_TANGENTS
OUTPUTS = native.HVP_OUTPUTS


def build_case(dof, N, P, B, dev, bounds=False, zmin=False, seed=5, outliers=0.2):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outliers)
    gen = torch.Generator().manual_seed(seed + 1)
    poses = pc["pose_gt"][:, None, :].repeat(1, P, 1)
    poses[..., :3] += 0.03 * torch.randn(B, P, 3, generator=gen)
    if dof == 6:
        q = poses[..., 3:] + 0.02 * torch.randn(B, P, 4, generator=gen)
        poses[..., 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        poses[..., 3] += 0.05 * torch.randn(B, P, generator=gen)
    c = {k: v.to(dev) for k, v in pc.items()}
    up = torch.randn(B, P, generator=gen)
    c.update(B=B, N=N, P=P, dof=dof, poses=poses.to(dev), up=up.to(dev), z_min=0.1, lb=None, ub=None)
    if zmin:
        c["z_min"] = 4.0
        c["poses"], margin = bm.place_depths(c["x3d"], c["poses"], c["cam_mats"], c["z_min"])
        assert margin > bm.ZMIN_GAP, margin
    if bounds:
        c["lb"], c["ub"], margin = bm.place_bounds(c["x3d"], c["poses"], c["cam_mats"], c["z_min"], True)
        assert margin > bm.BOUND_GAP, margin
    c["delta"] = orc.adaptive_delta(c["x2d"], c["w2d"], 0.1)
    D = c["poses"].shape[-1]
    shapes = dict(x3d=(B, N, 3), x2d=(B, N, 2), w2d=(B, N, 2), delta=(B,), pose=(B, P, D), cam=(B, 3, 3), lb=(B, 2),
                  ub=(B, 2))
    c["t"] = {k: torch.randn(shapes[k], generator=gen).to(dev) for k in TANGENTS if bounds or k not in ("lb", "ub")}
    c["t"]["cam"] *= 10.0                   # K is O(100): a tangent of a comparable relative size
    return c


def oracle_hvp(c, dtype, t=None, census=False):
    """The float64 (or float32) double backward: dict of the nine outputs of cost_hvp."""
    t = c["t"] if t is None else t
    leaf = lambda x: x.detach().to(dtype).clone().requires_grad_(True)
    x3d, x2d, w2d, delta, poses, cam, up = (leaf(c[k]) for k in ("x3d", "x2d", "w2d", "delta", "poses", "cam_mats",
                                                                  "up"))
    lb = ub = None
    if c["lb"] is not None:
        lb, ub = leaf(c["lb"]), leaf(c["ub"])
    camera = orc.Camera(cam, c["z_min"], lb, ub)
    cost = orc.evaluate(x3d, x2d, w2d, poses.transpose(0, 1), camera, delta)["cost"]          # (P, B)
    f = (cost * up.T).sum()
    ins = [x3d, x2d, w2d, delta, poses, cam] + ([lb, ub] if lb is not None else [])
    g = torch.autograd.grad(f, ins, create_graph=True)
    dot = sum((gi * t[k].to(dtype)).sum() for gi, k in zip(g, TANGENTS) if t.get(k) is not None)
    h = torch.autograd.grad(dot, ins + [up], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = dict(zip(("x3d", "x2d", "w2d", "delta", "pose", "cam") + (("lb", "ub") if lb is not None else ()),
                   (z(hi, x) for hi, x in zip(h[:-1], ins))))
    out["grad"] = z(h[-1], up)
    if census:
        with torch.no_grad():
            zh, u = bm.project(x3d, poses.transpose(0, 1), cam, c["z_min"])
            if lb is not None:
                u = torch.minimum(torch.maximum(u, orc._bound(lb, u)), orc._bound(ub, u))
            s = ((u - x2d) * w2d).norm(dim=-1)
            dl = delta[:, None]
            out["census"] = dict(outlier=float((s > dl).double().mean()),
                                 huber_gap=float(((s - dl).abs() / dl).min()))
    return out


def run_hvp(c, want=None, t=None):
    if want is None:                                     # every output the problem has
        want = tuple(k not in ("lb", "ub") or c["lb"] is not None for k in OUTPUTS)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    return dict(zip(OUTPUTS, native.cost_hvp(prob, c["dof"], c["z_min"], c["poses"], c["up"],
                                             c["t"] if t is None else t, want)))


def rel_rows(a, b, lead):
    """max|a - b| / max|b| over all but the first `lead` axes."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    a, b = a.reshape(b.shape[:lead] + (-1,)), b.reshape(b.shape[:lead] + (-1,))
    return ((a - b).abs().amax(-1) / b.abs().amax(-1).clamp(min=1e-300)).numpy()


def assert_close(got, c, what):
    ref64, ref32 = oracle_hvp(c, torch.float64, census=True), oracle_hvp(c, torch.float32)
    fr = ref64.pop("census")
    assert fr["huber_gap"] > HUBER_GAP, (what, fr)
    ratios = {}
    for k in OUTPUTS:
        if k not in ref64 or got.get(k) is None:
            continue
        assert torch.isfinite(got[k]).all(), (what, k)
        lead = 2 if k in ("pose", "grad") else 1
        if k == "grad":                                  # one value per pose: relative to its object's largest
            err = rel_rows(got[k], ref64[k], 1)
            floor = rel_rows(ref32[k], ref64[k], 1)
        else:
            err, floor = rel_rows(got[k], ref64[k], lead), rel_rows(ref32[k], ref64[k], lead)
        bound = np.maximum(REL_MIN, K_FLOOR * floor)
        bad = np.argwhere(err >= bound)
        assert bad.size == 0, (what, k, bad[:4].tolist(), err.max(), floor.max())
        ratios[k] = float((err / bound).max())
    return fr, ratios


CASES = [
    dict(id="d6_N64_P5_B3", dof=6, N=64, P=5, B=3),
    dict(id="d6_tensor_N300_P7_B4", dof=6, N=300, P=7, B=4, bounds=True),
    dict(id="d6_zmin_tensor_N129_P130_B2", dof=6, N=129, P=130, B=2, zmin=True, bounds=True),
    dict(id="d4_N200_P9_B3", dof=4, N=200, P=9, B=3),
    dict(id="d4_zmin_tensor_N257_P3_B3", dof=4, N=257, P=3, B=3, zmin=True, bounds=True),
    dict(id="d6_N16384_P3_B2", dof=6, N=16384, P=3, B=2),
]


def _build(case, dev):
    kw = {k: v for k, v in case.items() if k != "id"}
    return build_case(dev=dev, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_cost_hvp_against_float64(cuda_device, case):
    c = _build(case, cuda_device)
    got = run_hvp(c)
    fr, ratios = assert_close(got, c, case["id"])
    assert 0.01 < fr["outlier"] < 0.99, fr
    # run to run: the same bits
    again = run_hvp(c)
    for k in OUTPUTS:
        if got[k] is not None:
            assert torch.equal(got[k], again[k]), k


THIRD = "no autograd formula was registered"       # custom_op's error: cost_hvp has no formula of its own


def _layer_case(dev, dof, S, float_bounds, B=3, N=96, seed=3):
    """S poses per object (stacked (S, B, D) through evaluate_pnp) and bounds: per-object tensors, or Python floats
    (they clamp, but take no gradient)."""
    c = build_case(dof, N, S, B, dev, bounds=not float_bounds, seed=seed)
    if float_bounds:
        c["lb"], c["ub"], margin = bm.place_bounds(c["x3d"], c["poses"], c["cam_mats"], c["z_min"], False)
        assert margin > bm.BOUND_GAP, margin
    return c


def _evaluate_second_order(c, dtype, native_path, create_graph=True):
    """The inputs' gradients of sum up * cost, and the inputs' gradients of (those gradients . v), through
    evaluate_pnp(out_cost=True) (native) or the oracle (float64 / float32), poses (S, B, D)."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import HuberPnPCost
    leaf = lambda x: x.detach().to(dtype).clone().requires_grad_(True) if torch.is_tensor(x) else x
    x3d, x2d, w2d, cam, delta, lb, ub = (leaf(c[k]) for k in ("x3d", "x2d", "w2d", "cam_mats", "delta", "lb", "ub"))
    pose = leaf(c["poses"].transpose(0, 1))
    if native_path:
        camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
        cost = evaluate_pnp(x3d, x2d, w2d, pose, camera, HuberPnPCost(delta=delta), out_cost=True)[1]
    else:
        cost = orc.evaluate(x3d, x2d, w2d, pose, orc.Camera(cam, c["z_min"], lb, ub), delta)["cost"]
    names = ["x3d", "x2d", "w2d", "delta", "pose", "cam"] + (["lb", "ub"] if torch.is_tensor(lb) else [])
    ins = [x3d, x2d, w2d, delta, pose, cam] + ([lb, ub] if torch.is_tensor(lb) else [])
    g = torch.autograd.grad((cost * c["up"].T.to(dtype)).sum(), ins, create_graph=create_graph)
    if not create_graph:
        return g, None, ins
    t = [c["t"][k].transpose(0, 1) if k == "pose" else c["t"][k] for k in names]
    loss = sum((gi * ti.to(dtype)).sum() for gi, ti in zip(g, t))
    return [gi.detach() for gi in g], torch.autograd.grad(loss, ins, create_graph=native_path), ins


def _assert_rows(got, ref64, ref32, what):
    for i, (a, b, f) in enumerate(zip(got, ref64, ref32)):
        err, floor = rel_rows(a, b, 1), rel_rows(f, b, 1)
        assert (err < np.maximum(REL_MIN, K_FLOOR * floor)).all(), (what, i, err.max(), floor.max())


@pytest.mark.gpu
@pytest.mark.parametrize("dof,S,float_bounds", [(6, 1, False), (4, 1, False), (6, 3, True), (4, 2, True)])
def test_evaluate_pnp_second_order(cuda_device, dof, S, float_bounds):
    c = _layer_case(cuda_device, dof, S, float_bounds)
    g_nat, h_nat, ins = _evaluate_second_order(c, torch.float32, True)
    _, h64, _ = _evaluate_second_order(c, torch.float64, False)
    _, h32, _ = _evaluate_second_order(c, torch.float32, False)
    _assert_rows(h_nat, h64, h32, (dof, S, float_bounds))
    # the first-order gradients with and without create_graph: the same bits
    plain, _, _ = _evaluate_second_order(c, torch.float32, True, create_graph=False)
    for a, b in zip(plain, g_nat):
        assert torch.equal(a, b)
    # a third derivative raises from cost_hvp's missing formula (not from a gradient that lost its graph)
    with pytest.raises(RuntimeError, match=THIRD):
        torch.autograd.grad(sum(hi.sum() for hi in h_nat), ins)


def _mc_leaves(pc, dev, dtype=torch.float32):
    """x3d, x2d, w2d, delta (B), pose_init, cam_mats, lb, ub: every input of cost_init + logsumexp(logw) as a leaf.
    The bounds are wide: they clamp no projection, and take a zero gradient."""
    B = pc["x3d"].shape[0]
    x2d = pc["x2d"].to(dev, dtype)
    delta = orc.adaptive_delta(pc["x2d"], pc["w2d"], 0.5).to(dev, dtype)
    vals = [pc["x3d"].to(dev, dtype), x2d, pc["w2d"].to(dev, dtype), delta, pc["pose_init"].to(dev, dtype),
            pc["cam_mats"].to(dev, dtype), (x2d.amin(1) - 400.0).reshape(B, 2), (x2d.amax(1) + 400.0).reshape(B, 2)]
    return [v.detach().clone().requires_grad_(True) for v in vals]


def _mc_layer_loss(leaves, noise, layer, loss_fn=None):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    x3d, x2d, w2d, delta, pose_init, cam, lb, ub = leaves
    camera = PerspectiveCamera(cam_mats=cam, lb=lb, ub=ub)
    _, _, _, samples, logw, cost_init = layer.monte_carlo_forward(
        x3d, x2d, w2d, camera, HuberPnPCost(delta=delta), pose_init=pose_init, force_init_solve=False,
        with_cost=True, amis_noise=noise)
    loss_fn = MonteCarloPoseLoss().to(x3d.device) if loss_fn is None else loss_fn
    loss = loss_fn(logw, cost_init, 1.0)
    return loss, samples, logw


def _mc_setup(dev, B=4, N=128, M=128, seed=21):
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp_b200.synth import make_noise
    pc = make_problem(B, N, seed=seed)
    noise = tuple(t.to(dev) for t in make_noise(B, M, seed=seed + 1))
    gen = torch.Generator().manual_seed(seed + 2)
    leaves = _mc_leaves(pc, dev)
    tangents = [torch.randn(x.shape, generator=gen).to(dev) for x in leaves]
    tangents[5] *= 10.0
    return pc, noise, EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=5)), tangents


@pytest.mark.gpu
def test_monte_carlo_loss_second_order(cuda_device):
    """A create_graph step through MonteCarloPoseLoss(logw, cost_init) with every input a leaf (x3d, x2d, w2d, delta,
    pose_init, cam_mats, tensor bounds), then grad . v, differentiated per input against the oracle's float64 double
    backward.  The oracle reuses the kernel's samples and treats the proposal log-density as a constant, as the
    reference does: logw = (logw + cost)(kernel's samples, inputs held) - cost(oracle)."""
    dev = cuda_device
    pc, noise, layer, tangents = _mc_setup(dev)
    leaves = _mc_leaves(pc, dev)
    loss, samples, logw = _mc_layer_loss(leaves, noise, layer)
    g = torch.autograd.grad(loss, leaves, create_graph=True)
    h_nat = torch.autograd.grad(sum((gi * ti).sum() for gi, ti in zip(g, tangents)), leaves)
    # first order: the same bits with and without create_graph
    plain = _mc_leaves(pc, dev)
    g0 = torch.autograd.grad(_mc_layer_loss(plain, noise, layer)[0], plain)
    for a, b in zip(g0, g):
        assert torch.equal(a, b.detach())

    samples_sb = samples.detach().double()                                    # (M, B, 7)

    def oracle(dtype):
        lv = _mc_leaves(pc, dev, dtype)
        x3d, x2d, w2d, delta, pose_init, cam, lb, ub = lv
        camera = orc.Camera(cam, 0.1, lb, ub)
        with torch.no_grad():
            c_k = orc.evaluate(x3d, x2d, w2d, samples_sb.to(dtype), camera, delta)["cost"]
            logq = -(logw.detach().to(dtype) + c_k)                           # the proposal log-density, held
        c = orc.evaluate(x3d, x2d, w2d, samples_sb.to(dtype), camera, delta)["cost"]     # (M, B)
        ci = orc.evaluate(x3d, x2d, w2d, pose_init, camera, delta)["cost"]
        loss = (ci + torch.logsumexp(-c - logq, dim=0)).mean()                # MonteCarloPoseLoss, reduction 'mean'
        go = torch.autograd.grad(loss, lv, create_graph=True)
        return torch.autograd.grad(sum((gi * ti.to(dtype)).sum() for gi, ti in zip(go, tangents)), lv,
                                   allow_unused=True)

    z = lambda hs, like: [torch.zeros_like(x) if h is None else h for h, x in zip(hs, like)]
    h64, h32 = z(oracle(torch.float64), h_nat), z(oracle(torch.float32), h_nat)
    names = ("x3d", "x2d", "w2d", "delta", "pose_init", "cam_mats", "lb", "ub")
    for name, a, b, f in zip(names, h_nat, h64, h32):
        if name in ("lb", "ub"):                                              # nothing is clamped
            assert torch.equal(a, torch.zeros_like(a)) and float(b.abs().max()) == 0.0, name
            continue
        assert float(b.abs().max()) > 0, name
        err, floor = rel_rows(a, b, 1), rel_rows(f, b, 1)
        assert (err < np.maximum(2e-3, K_FLOOR * floor)).all(), (name, err.max(), floor.max())


@pytest.mark.gpu
def test_graph_replay_of_a_second_order_step(cuda_device):
    """A create_graph step through MonteCarloPoseLoss (forward, first gradient, gradient . v and its gradient: the
    cost_hvp launches and mc_lse_backward's formula) captured in a CUDA graph, then replayed on NEW inputs copied into
    the static leaves: the same bits as the eager step on those inputs."""
    dev = cuda_device
    pc, noise, layer, tangents = _mc_setup(dev)
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    loss_fn = MonteCarloPoseLoss().to(dev)                  # its buffers are moved once, outside the capture

    def step(leaves):
        loss, _, _ = _mc_layer_loss(leaves, noise, layer, loss_fn)
        g = torch.autograd.grad(loss, leaves, create_graph=True)
        return torch.autograd.grad(sum((gi * ti).sum() for gi, ti in zip(g, tangents)), leaves[:6])

    static = _mc_leaves(pc, dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(static)
    pc2 = dict(pc, x2d=pc["x2d"] + 0.5 * torch.randn(pc["x2d"].shape, generator=torch.Generator().manual_seed(7)))
    new = _mc_leaves(pc2, dev)
    with torch.no_grad():
        for a, b in zip(static, new):
            a.copy_(b)
    graph.replay()
    torch.cuda.synchronize()
    eager = step(_mc_leaves(pc2, dev))
    for a, b in zip(out, eager):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_opcheck_cost_hvp(cuda_device):
    c = build_case(6, 40, 3, 2, cuda_device, bounds=True)
    t = c["t"]
    args = (c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"], c["poses"], c["up"],
            *(t.get(k) for k in TANGENTS), 6, c["z_min"], [True] * 9)
    torch.library.opcheck(ops.cost_hvp.op, args)
