"""Second order through pose_opt_plus = pose (+) gn_step(pose): the Hessian-vector-product kernel
(epnp_gn_plus_hvp_f32) and the autograd formulas of gn_plus_backward and gn_plus_camera_backward that call it.

The reference is the oracle's float64 double backward of f = <gplus, pose_add(pose, gn_step(pose))> at a detached pose:
grad f with create_graph with respect to x3d, x2d, w2d, delta, cam_mats, lb, ub, then the gradient of grad f . u with
respect to those inputs and gplus.  Bound: per object and output, max|a - b| / max|b| under max(REL_MIN, K_FLOOR * floor)
(test_cost_hvp_gpu.py's REL_MIN and K_FLOOR), floor = the largest error of the same double backward in float32 over
four orders of the points (the delta row sums per-point terms that largely cancel, and the order of that float32 sum
alone moves it by its own size in the small-delta cases).  Depths, bounds and residual
norms are kept off z_min, the bounds and delta by margins that each case asserts.  An object whose cond(H + eps I)
exceeds 1e6 is counted and not compared: there the float32 solve itself is the error.

Then the layer: LMSolver's pose_opt_plus differentiated twice, a gradient penalty on a loss linear in pose_opt_plus
plus the Monte-Carlo loss, the 6DoF training loss with a create_graph penalty against the torch composite
(EPNP_NATIVE_GN_STEP=0), and the exact properties (first order unchanged by create_graph, run-to-run bits, a third
backward raises, CUDA-graph replay) and torch.library.opcheck."""
import numpy as np
import pytest
import torch

import test_backward_matrix_gpu as bm
from oracle import pnp_oracle as orc
from epropnp_b200 import native, ops
from epropnp_b200.synth import make_problem
from test_cost_hvp_gpu import HUBER_GAP, K_FLOOR, REL_MIN, THIRD, rel_rows

TANGENTS = native.GN_HVP_TANGENTS
OUTPUTS = native.GN_HVP_OUTPUTS
EPS, HUBER_EPS = 1e-5, 1e-10
COND_MAX = 1e6


def build_case(dof, N, B, dev, bounds=None, zmin=False, seed=5, outliers=0.2, relative_delta=0.1):
    """bounds: None, "scalar" (one value for every object and coordinate, passed as (B, 2)) or "tensor"."""
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=outliers)
    gen = torch.Generator().manual_seed(seed + 1)
    pose = pc["pose_gt"].clone()
    pose[:, :3] += 0.03 * torch.randn(B, 3, generator=gen)
    if dof == 6:
        q = pose[:, 3:] + 0.02 * torch.randn(B, 4, generator=gen)
        pose[:, 3:] = q / q.norm(dim=-1, keepdim=True)
    else:
        pose[:, 3] += 0.05 * torch.randn(B, generator=gen)
    c = {k: v.to(dev) for k, v in pc.items()}
    c.update(B=B, N=N, dof=dof, pose=pose.to(dev), z_min=0.1, lb=None, ub=None)
    if zmin:
        c["z_min"] = 4.0
        p, margin = bm.place_depths(c["x3d"], c["pose"][:, None], c["cam_mats"], c["z_min"])
        c["pose"] = p[:, 0]
        assert margin > bm.ZMIN_GAP, margin
    if bounds is not None:
        lb, ub, margin = bm.place_bounds(c["x3d"], c["pose"][:, None], c["cam_mats"], c["z_min"], bounds == "tensor")
        assert margin > bm.BOUND_GAP, margin
        full = lambda b: b if torch.is_tensor(b) else torch.full((B, 2), float(b), device=dev)
        c["lb"], c["ub"] = full(lb).to(dev), full(ub).to(dev)
    c["delta"] = orc.adaptive_delta(c["x2d"], c["w2d"], relative_delta)
    D = c["pose"].shape[-1]
    c["gplus"] = torch.randn(B, D, generator=gen).to(dev)
    shapes = dict(x3d=(B, N, 3), x2d=(B, N, 2), w2d=(B, N, 2), delta=(B,), cam=(B, 3, 3), lb=(B, 2), ub=(B, 2))
    c["t"] = {k: torch.randn(shapes[k], generator=gen).to(dev) for k in TANGENTS
              if bounds is not None or k not in ("lb", "ub")}
    c["t"]["cam"] *= 10.0                   # K is O(100): a tangent of a comparable relative size
    return c


def oracle_hvp(c, dtype, t=None, census=False):
    """The double backward in `dtype`, on the CPU (the oracle's solve is CPU-only): dict of gn_plus_hvp's eight outputs
    (and the census)."""
    t = {k: v.cpu() for k, v in (c["t"] if t is None else t).items()}
    leaf = lambda x: x.detach().cpu().to(dtype).clone().requires_grad_(True)
    x3d, x2d, w2d, delta, cam, gplus = (leaf(c[k]) for k in ("x3d", "x2d", "w2d", "delta", "cam_mats", "gplus"))
    lb = ub = None
    if c["lb"] is not None:
        lb, ub = leaf(c["lb"]), leaf(c["ub"])
    pose = c["pose"].detach().cpu().to(dtype)
    camera = orc.Camera(cam, c["z_min"], lb, ub)
    plus = orc.pose_add(pose, orc.gn_step(x3d, x2d, w2d, camera, delta, pose, EPS))
    ins = [x3d, x2d, w2d, delta, cam] + ([lb, ub] if lb is not None else [])
    g = torch.autograd.grad((plus * gplus).sum(), ins, create_graph=True)
    dot = sum((gi * t[k].to(dtype)).sum() for gi, k in zip(g, TANGENTS) if t.get(k) is not None)
    h = torch.autograd.grad(dot, ins + [gplus], allow_unused=True)
    z = lambda hi, x: torch.zeros_like(x) if hi is None else hi
    out = dict(zip(TANGENTS, (z(hi, x) for hi, x in zip(h[:-1], ins))))
    out["grad"] = z(h[-1], gplus)
    if census:
        with torch.no_grad():
            zh, u = bm.project(x3d, pose[None], cam, c["z_min"])
            u_c = u
            if lb is not None:
                u_c = torch.minimum(torch.maximum(u, orc._bound(lb, u)), orc._bound(ub, u))
            s = ((u_c - x2d) * w2d).norm(dim=-1)
            dl = delta[:, None]
            e = orc.evaluate(x3d, x2d, w2d, pose, camera, delta, want_jac=True)
            jtj = e["jac"].transpose(-1, -2) @ e["jac"] + EPS * torch.eye(e["jac"].shape[-1], dtype=dtype)
            out["census"] = dict(outlier=float((s > dl).double().mean()), huber_gap=float(((s - dl).abs() / dl).min()),
                                 below_zmin=float((zh < c["z_min"]).double().mean()),
                                 clamped=float((u_c != u).any(-1).double().mean()),
                                 cond=torch.linalg.cond(jtj).cpu().numpy())
    return out


def run_hvp(c, want=None, t=None):
    if want is None:                                     # every output the problem has
        want = tuple(k not in ("lb", "ub") or c["lb"] is not None for k in OUTPUTS)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    return dict(zip(OUTPUTS, native.gn_plus_hvp(prob, c["pose"], c["gplus"], c["dof"], c["z_min"], EPS, HUBER_EPS,
                                                c["t"] if t is None else t, want)))


ORDERS = 4
POINT_OUTPUTS = ("x3d", "x2d", "w2d")


def floors(c, ref64):
    """Per output and object: the largest relative error of the float32 double backward over ORDERS orders of the
    points (the first the identity)."""
    N = c["x3d"].shape[1]
    out = {}
    for s in range(ORDERS):
        perm = torch.arange(N) if s == 0 else torch.randperm(N, generator=torch.Generator().manual_seed(s))
        perm = perm.to(c["x3d"].device)
        cc = dict(c, t=dict(c["t"]))
        for k in POINT_OUTPUTS:
            cc[k], cc["t"][k] = c[k][:, perm], c["t"][k][:, perm]
        r = oracle_hvp(cc, torch.float32)
        inv = torch.argsort(perm).cpu()                  # the oracle's outputs live on the CPU
        for k in POINT_OUTPUTS:
            r[k] = r[k][:, inv]
        for k, v in r.items():
            e = rel_rows(v, ref64[k], 1)
            out[k] = e if k not in out else np.maximum(out[k], e)
    return out


def assert_close(got, c, what):
    """Every output of every well-conditioned object within max(REL_MIN, K_FLOOR * floor).  Returns the census and the
    largest share of the bound used per output."""
    ref64 = oracle_hvp(c, torch.float64, census=True)
    fr = ref64.pop("census")
    fl = floors(c, ref64)
    assert fr["huber_gap"] > HUBER_GAP, (what, fr["huber_gap"])
    ok = fr["cond"] <= COND_MAX
    ratios = {}
    for k in OUTPUTS:
        if k not in ref64 or got.get(k) is None:
            continue
        assert torch.isfinite(got[k]).all(), (what, k)
        err, floor = rel_rows(got[k], ref64[k], 1), fl[k]
        bound = np.maximum(REL_MIN, K_FLOOR * floor)
        bad = np.argwhere((err >= bound) & ok)
        assert bad.size == 0, (what, k, bad[:4].tolist(), err[ok].max(), floor.max())
        ratios[k] = float((err / bound)[ok].max())
    fr["ill_conditioned"] = int((~ok).sum())
    return fr, ratios


def grid(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


CASES = [
    dict(id="d6_N5_B3", dof=6, N=5, B=3, outliers=0.0, relative_delta=0.5),
    dict(id="d6_tensor_N512_B6", dof=6, N=512, B=6, bounds="tensor"),
    dict(id="d6_scalar_N300_B4", dof=6, N=300, B=4, bounds="scalar"),
    dict(id="d6_zmin_tensor_N2048_B3", dof=6, N=2048, B=3, zmin=True, bounds="tensor", relative_delta=1.0),
    dict(id="d6_small_delta_N257_B4", dof=6, N=257, B=4, relative_delta=0.02, outliers=0.1),
    dict(id="d4_N200_B4", dof=4, N=200, B=4),
    dict(id="d4_zmin_tensor_N513_B3", dof=4, N=513, B=3, zmin=True, bounds="tensor", relative_delta=1.0),
    dict(id="d6_N16384_B2", dof=6, N=16384, B=2),
]


def _build(case, dev):
    return build_case(dev=dev, **{k: v for k, v in case.items() if k != "id"})


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_gn_plus_hvp_against_float64(cuda_device, case):
    c = _build(case, cuda_device)
    got = run_hvp(c)
    fr, ratios = assert_close(got, c, case["id"])
    assert fr["ill_conditioned"] < c["B"], fr
    if case["N"] > 5:
        assert 0.01 < fr["outlier"] < 0.99, fr
    if case.get("zmin"):
        assert fr["below_zmin"] > 0.01, fr
    if case.get("bounds"):
        assert fr["clamped"] > 0.01, fr
    again = run_hvp(c)
    for k in OUTPUTS:
        if got[k] is not None:
            assert torch.equal(got[k], again[k]), k


@pytest.mark.gpu
def test_batch_larger_than_the_grid(cuda_device):
    """B above one wave of CTAs: every object equals its own run alone, bit for bit."""
    B = 2 * grid(cuda_device) + 3
    c = build_case(6, 40, B, cuda_device, bounds="tensor", seed=9)
    got = run_hvp(c)
    for b in (0, B // 2, B - 1):
        one = {k: (v[b:b + 1] if torch.is_tensor(v) and v.dim() and v.shape[0] == B else v) for k, v in c.items()}
        one["t"] = {k: v[b:b + 1] for k, v in c["t"].items()}
        one["B"] = 1
        alone = run_hvp(one)
        for k in OUTPUTS:
            assert torch.equal(alone[k], got[k][b:b + 1]), (b, k)
    assert_close(got, c, "B>grid")


# ------------------------------------------------------------------------------------------------------------ the layer
def _leaves(c, dtype=torch.float32, dev=None):
    vals = [c[k] for k in ("x3d", "x2d", "w2d", "delta", "cam_mats")] + ([c["lb"], c["ub"]] if c["lb"] is not None
                                                                          else [])
    return [v.detach().to(dev or v.device, dtype).clone().requires_grad_(True) for v in vals]


def _plus(leaves, c, native_path, dof):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.levenberg_marquardt import LMSolver
    x3d, x2d, w2d, delta, cam = leaves[:5]
    lb, ub = (leaves[5], leaves[6]) if len(leaves) > 5 else (None, None)
    camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
    pose = c["pose"].to(x3d.device, x3d.dtype)
    if native_path:
        from epropnp import autograd as ag
        return ag.pose_plus_autograd(LMSolver(dof=dof, num_iter=0), x3d, x2d, w2d, pose, camera,
                                     HuberPnPCost(delta=delta))
    return orc.pose_add(pose, orc.gn_step(x3d, x2d, w2d, orc.Camera(cam, c["z_min"], lb, ub), delta, pose, EPS))


def _second_order(c, dtype, native_path):
    """The native layer on the problem's device, the oracle composite on the CPU."""
    leaves = _leaves(c, dtype, None if native_path else torch.device("cpu"))
    dev = leaves[0].device
    plus = _plus(leaves, c, native_path, c["dof"])
    g = torch.autograd.grad((plus * c["gplus"].to(dev, dtype)).sum(), leaves, create_graph=True)
    t = [c["t"][k] for k in TANGENTS[:len(leaves)]]
    loss = sum((gi * ti.to(dev, dtype)).sum() for gi, ti in zip(g, t))
    return [gi.detach() for gi in g], torch.autograd.grad(loss, leaves, create_graph=native_path), leaves


@pytest.mark.gpu
@pytest.mark.parametrize("dof,bounds", [(6, "tensor"), (4, None)])
def test_pose_opt_plus_twice_through_the_layer(cuda_device, monkeypatch, dof, bounds):
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    c = build_case(dof, 96, 3, cuda_device, bounds=bounds, seed=13)
    g_nat, h_nat, leaves = _second_order(c, torch.float32, True)
    _, h64, _ = _second_order(c, torch.float64, False)
    _, h32, _ = _second_order(c, torch.float32, False)
    for name, a, b, f in zip(TANGENTS, h_nat, h64, h32):
        err, floor = rel_rows(a, b, 1), rel_rows(f, b, 1)
        assert (err < np.maximum(REL_MIN, K_FLOOR * floor)).all(), (name, err.max(), floor.max())
    # first order: the same bits with and without create_graph
    plain = _leaves(c)
    g0 = torch.autograd.grad((_plus(plain, c, True, dof) * c["gplus"]).sum(), plain)
    for a, b in zip(g0, g_nat):
        assert torch.equal(a, b)
    # a third derivative raises from gn_plus_hvp's missing formula
    with pytest.raises(RuntimeError, match=THIRD):
        torch.autograd.grad(sum(hi.sum() for hi in h_nat), leaves)


def _mc_inputs(dev, B=4, N=128, M=128, seed=21):
    from epropnp_b200.synth import make_noise
    pc = make_problem(B, N, seed=seed)
    noise = tuple(t.to(dev) for t in make_noise(B, M, seed=seed + 1))
    x2d = pc["x2d"].to(dev)
    delta = orc.adaptive_delta(pc["x2d"], pc["w2d"], 0.5).to(dev)
    vals = [pc["x3d"].to(dev), x2d, pc["w2d"].to(dev), delta, pc["cam_mats"].to(dev)]
    return pc, noise, vals


def _train_loss(vals, pc, noise, dev, linear, dtype=torch.float32, seed=0):
    """The 6DoF training loss (train.py:178-193): MonteCarloPoseLoss + loss_t / loss_r on pose_opt_plus, or, with
    `linear`, the Monte-Carlo loss plus a loss linear in pose_opt_plus.  -> loss, leaves."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in vals]
    x3d, x2d, w2d, delta, cam = leaves
    layer = EProPnP6DoF(mc_samples=noise[0].shape[1], num_iter=4, solver=LMSolver(dof=6, num_iter=5)).to(dev)
    torch.manual_seed(seed)
    _, _, pose_opt_plus, _, logw, cost_init = layer.monte_carlo_forward(
        x3d, x2d, w2d, PerspectiveCamera(cam_mats=cam), HuberPnPCost(delta=delta),
        pose_init=pc["pose_init"].to(dev, dtype), force_init_solve=False, with_pose_opt_plus=True, with_cost=True,
        amis_noise=tuple(n.to(dev) for n in noise))
    loss_mc = MonteCarloPoseLoss().to(dev)(logw, cost_init, 1.0)
    gt = pc["pose_gt"].to(dev, dtype)
    if linear:
        w = 100.0 * torch.linspace(-1.0, 1.0, pose_opt_plus.numel(), device=dev, dtype=dtype)
        return loss_mc + (pose_opt_plus * w.reshape(pose_opt_plus.shape)).sum(), leaves
    loss_t = torch.nn.functional.smooth_l1_loss(pose_opt_plus[:, :3], gt[:, :3], beta=0.05)
    dot = (pose_opt_plus[:, 3:] * gt[:, 3:]).sum(-1)
    loss_r = (1 - dot * dot).mean()
    return loss_mc + loss_t + loss_r, leaves


def _penalised_step(vals, pc, noise, dev, linear, dtype=torch.float32):
    loss, leaves = _train_loss(vals, pc, noise, dev, linear, dtype)
    g = torch.autograd.grad(loss, leaves, create_graph=True)
    penalty = sum((gi * gi).sum() for gi in g)
    return [gi.detach() for gi in g], torch.autograd.grad(loss + penalty, leaves)


@pytest.mark.gpu
@pytest.mark.parametrize("linear", [True, False], ids=["linear_in_plus", "train_py_loss"])
def test_penalised_training_step_matches_the_composite(cuda_device, monkeypatch, linear):
    """A create_graph gradient-norm penalty over the training loss: native against EPNP_NATIVE_GN_STEP=0 (the same
    forward, samples and pose_opt_plus; only pose_opt_plus's derivatives are formed differently), per object and input
    within 2e-3 relative (the bound of test_cost_hvp_gpu.py's Monte-Carlo step).  Where pose_opt_plus's first gradient
    had no graph the penalty's gradient would lack the pose_opt_plus Hessian term and miss the composite by far more."""
    dev = cuda_device
    pc, noise, vals = _mc_inputs(dev)
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    g_nat, h_nat = _penalised_step(vals, pc, noise, dev, linear)
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "0")
    g_cmp, h_cmp = _penalised_step(vals, pc, noise, dev, linear)
    for name, a, b in zip(("x3d", "x2d", "w2d", "delta", "cam_mats"), h_nat, h_cmp):
        assert torch.isfinite(a).all(), name
        err = rel_rows(a, b, 1)
        assert (err < 2e-3).all(), (name, err.max())
    for a, b in zip(g_nat, g_cmp):
        assert (rel_rows(a, b, 1) < 2e-3).all()


@pytest.mark.gpu
def test_graph_replay_of_a_second_order_step(cuda_device, monkeypatch):
    """pose_opt_plus's create_graph step (forward, first gradient, gradient . u and its gradient: the gn_plus backward
    and gn_plus_hvp launches) captured in a CUDA graph, then replayed on NEW inputs copied into the static leaves: the
    same bits as the eager step on those inputs."""
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    dev = cuda_device
    c = build_case(6, 64, 4, dev, bounds="tensor", seed=17)

    def step(leaves):
        plus = _plus(leaves, c, True, 6)
        g = torch.autograd.grad((plus * c["gplus"]).sum(), leaves, create_graph=True)
        return torch.autograd.grad(sum((gi * c["t"][k]).sum() for gi, k in zip(g, TANGENTS)), leaves)

    static = _leaves(c)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(static)
    c2 = dict(c, x2d=c["x2d"] + 0.3 * torch.randn(c["x2d"].shape, generator=torch.Generator().manual_seed(7)).to(dev))
    new = _leaves(c2)
    with torch.no_grad():
        for a, b in zip(static, new):
            a.copy_(b)
    graph.replay()
    torch.cuda.synchronize()
    eager = step(_leaves(c2))
    for a, b in zip(out, eager):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_opcheck_gn_plus_hvp(cuda_device):
    c = build_case(6, 40, 2, cuda_device, bounds="tensor")
    args = (c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"], c["pose"], c["gplus"],
            *(c["t"].get(k) for k in TANGENTS), 6, c["z_min"], EPS, HUBER_EPS, [True] * 8)
    torch.library.opcheck(ops.gn_plus_hvp.op, args)
