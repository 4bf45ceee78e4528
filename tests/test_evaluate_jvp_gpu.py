"""Forward mode through the layer: the Jacobian-vector-product kernel (epnp_evaluate_jvp_f32) and the jvp formulas of the
eager autograd.Functions that call it.

The kernel is held to the oracle's float64 forward-mode derivative (torch.func.jvp of orc.evaluate, which forms the
rotation as the kernels do) per pose and object and output, under max(REL_MIN, K_FLOOR * floor), floor = the same
derivative in float32.  Depths, bounds and residuals are kept off their clamps by the margins of the cost tests.  Every
formula is then tied to the existing native backwards by the adjoint identity <g, J v> = <J^T g, v>, per object."""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

import test_backward_matrix_gpu as bm
import test_cost_hvp_gpu as hv
from oracle import pnp_oracle as orc
from epropnp_b200 import native, ops

K_FLOOR = 10
REL_MIN = 5e-4
ADJ_TOL = 2e-4              # |<g, J v> - <J^T g, v>| / sum |terms|, per object
OUTPUTS = native.JVP_OUTPUTS


def build_case(dof, N, S, B, dev, bounds=False, zmin=False, seed=5, clip=True):
    """hv.build_case with the poses stacked (S, B, D), as evaluate_pnp takes them."""
    c = hv.build_case(dof, N, S, B, dev, bounds=bounds, zmin=zmin, seed=seed)
    c["poses"] = c["poses"].transpose(0, 1).contiguous()
    c["t"]["pose"] = c["t"]["pose"].transpose(0, 1).contiguous()
    c["S"], c["clip"] = S, clip
    return c


def _oracle_fn(c, dtype):
    lb = None if c["lb"] is None else c["lb"].to(dtype)
    ub = None if c["ub"] is None else c["ub"].to(dtype)
    names = ["x3d", "x2d", "w2d", "delta", "pose", "cam"] + (["lb", "ub"] if lb is not None else [])

    def f(x3d, x2d, w2d, delta, poses, cam, *bnd):
        lo, hi = bnd if bnd else (None, None)
        out = orc.evaluate(x3d, x2d, w2d, poses, orc.Camera(cam, c["z_min"], lo, hi), delta, want_jac=True,
                           clip_jac=c["clip"])
        return out["residual"], out["jac"], out["cost"]
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], pose=c["poses"], cam=c["cam_mats"],
               lb=c["lb"], ub=c["ub"])
    return f, names, [src[k].detach().to(dtype) for k in names]


def oracle_jvp(c, dtype, t=None):
    """The oracle's forward-mode derivative in `dtype`: dict residual (S, B, 2N), jac (S, B, 2N, dof), cost (S, B)."""
    t = c["t"] if t is None else t
    f, names, primals = _oracle_fn(c, dtype)
    tangents = [t[k].to(dtype) if t.get(k) is not None else torch.zeros_like(p) for k, p in zip(names, primals)]
    _, out = torch.func.jvp(f, tuple(primals), tuple(tangents))
    return dict(zip(OUTPUTS, out))


def run_jvp(c, want=(True, True, True), t=None):
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    return dict(zip(OUTPUTS, native.evaluate_jvp(prob, c["poses"], c["dof"], c["z_min"], 1e-10, c["clip"],
                                                 c["t"] if t is None else t, want)))


def assert_close(got, c, what):
    ref64, ref32 = oracle_jvp(c, torch.float64), oracle_jvp(c, torch.float32)
    for k in OUTPUTS:
        if got.get(k) is None:
            continue
        assert torch.isfinite(got[k]).all(), (what, k)
        lead = 1 if k == "cost" else 2                   # cost: per pose, relative to its largest object
        err, floor = hv.rel_rows(got[k], ref64[k], lead), hv.rel_rows(ref32[k], ref64[k], lead)
        bound = np.maximum(REL_MIN, K_FLOOR * floor)
        bad = np.argwhere(err >= bound)
        assert bad.size == 0, (what, k, bad[:4].tolist(), err.max(), floor.max())


def huber_margin(c):
    """Least relative distance of a float64 residual norm from delta (the cost tests' margin)."""
    zh, u = bm.project(c["x3d"].double(), c["poses"].double(), c["cam_mats"].double(), c["z_min"])
    if c["lb"] is not None:
        u = torch.minimum(torch.maximum(u, orc._bound(c["lb"].double(), u)), orc._bound(c["ub"].double(), u))
    s = ((u - c["x2d"].double()) * c["w2d"].double()).norm(dim=-1)
    dl = c["delta"].double()[:, None]
    return float(((s - dl).abs() / dl).min())


def adjoint_gap(c, seed=11):
    """max over objects of |<g, J v> - <J^T g, v>| / sum |terms| for random upstream g of all three outputs, J^T g by
    epnp_evaluate_backward_f32."""
    gen = torch.Generator().manual_seed(seed)
    S, B, N, dof = c["S"], c["B"], c["N"], c["dof"]
    dev = c["x3d"].device
    g = dict(residual=torch.randn(S, B, 2 * N, generator=gen).to(dev),
             jac=torch.randn(S, B, 2 * N, dof, generator=gen).to(dev), cost=torch.randn(S, B, generator=gen).to(dev))
    jv = run_jvp(c)
    prob = native.Problem(c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"])
    bounded = c["lb"] is not None
    want = (True,) * 6 + (bounded, bounded)
    vjp = native.evaluate_backward(prob, c["poses"], dof, c["z_min"], 1e-10, c["clip"], g["residual"], g["jac"],
                                   g["cost"], want)
    lhs = torch.zeros(B, dtype=torch.float64)
    mag = torch.zeros(B, dtype=torch.float64)
    for k in OUTPUTS:
        term = (g[k].double() * jv[k].double()).reshape(S, B, -1).cpu()
        lhs += term.sum((0, 2))
        mag += term.abs().sum((0, 2))
    rhs = torch.zeros(B, dtype=torch.float64)
    for name, gr in zip(("x3d", "x2d", "w2d", "delta", "pose", "cam", "lb", "ub"), vjp):
        if gr is None or c["t"].get(name) is None:
            continue
        term = gr.double().cpu() * c["t"][name].double().cpu()
        term = term.transpose(0, 1) if name == "pose" else term
        term = term.reshape(B, -1)
        rhs += term.sum(1)
        mag += term.abs().sum(1)
    return float(((lhs - rhs).abs() / mag).max())


CASES = [
    dict(id="d6_N64_S1_B3", dof=6, N=64, S=1, B=3),
    dict(id="d6_tensor_N300_S3_B4", dof=6, N=300, S=3, B=4, bounds=True),
    dict(id="d6_zmin_tensor_N129_S130_B2", dof=6, N=129, S=130, B=2, zmin=True, bounds=True),
    dict(id="d6_noclip_zmin_N100_S2_B3", dof=6, N=100, S=2, B=3, zmin=True, clip=False),
    dict(id="d4_N200_S9_B3", dof=4, N=200, S=9, B=3),
    dict(id="d4_zmin_tensor_N257_S3_B3", dof=4, N=257, S=3, B=3, zmin=True, bounds=True),
    dict(id="d6_N5_S1_B300", dof=6, N=5, S=1, B=300),
    dict(id="d6_N16384_S2_B2", dof=6, N=16384, S=2, B=2),
]


def _build(case, dev):
    return build_case(dev=dev, **{k: v for k, v in case.items() if k != "id"})


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_evaluate_jvp_against_float64(cuda_device, case):
    c = _build(case, cuda_device)
    assert huber_margin(c) > hv.HUBER_GAP
    got = run_jvp(c)
    assert_close(got, c, case["id"])
    # d cost alone (pose-major from 64 poses on) agrees with the cost of the full call
    alone = run_jvp(c, want=(False, False, True))["cost"]
    assert torch.allclose(alone, got["cost"], rtol=1e-4, atol=1e-4 * float(got["cost"].abs().max()))
    assert adjoint_gap(c) < ADJ_TOL
    again = run_jvp(c)
    for k in OUTPUTS:
        assert torch.equal(got[k], again[k]), k


# ------------------------------------------------------------------------------------------------------------- layer
def _dual(x, t):
    return fwAD.make_dual(x, t.to(x.device, x.dtype))


def forward_mode(f, primals, tangents, mode):
    """The tangents of f's outputs: mode 'fwad' (torch.autograd.forward_ad), 'jvp' (torch.func.jvp) or 'linearize'
    (torch.func.linearize, its linear function applied to the tangents)."""
    if mode == "jvp":
        return tuple(torch.func.jvp(f, tuple(primals), tuple(tangents))[1])
    if mode == "linearize":
        _, lin = torch.func.linearize(f, *primals)
        return tuple(lin(*tangents))
    with fwAD.dual_level():
        out = f(*(_dual(p, t) for p, t in zip(primals, tangents)))
        return tuple(fwAD.unpack_dual(o).tangent for o in out)


def _evaluate_layer(c, dtype, dev, out_jac, mode="fwad"):
    """Tangents of evaluate_pnp's outputs with every input given one (forward_mode)."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import HuberPnPCost
    tensor_bounds = torch.is_tensor(c["lb"])
    names = ["x3d", "x2d", "w2d", "delta", "pose", "cam"] + (["lb", "ub"] if tensor_bounds else [])
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], pose=c["poses"], cam=c["cam_mats"],
               lb=c["lb"], ub=c["ub"])
    primals = [src[k].detach().to(dev, dtype) for k in names]
    tangents = [c["t"][k].to(dev, dtype) for k in names]

    def f(x3d, x2d, w2d, delta, pose, cam, *bnd):
        lb, ub = bnd if bnd else (c["lb"], c["ub"])
        camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
        r, cost, j = evaluate_pnp(x3d, x2d, w2d, pose, camera, HuberPnPCost(delta=delta), out_residual=out_jac,
                                  out_jacobian=out_jac, out_cost=True)
        return (r, j, cost) if out_jac else (cost,)
    return forward_mode(f, primals, tangents, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fwad", "jvp", "linearize"])
@pytest.mark.parametrize("dof,S,float_bounds,out_jac", [(6, 1, False, True), (6, 3, True, True), (4, 2, False, True),
                                                        (6, 3, False, False), (4, 1, True, False)])
def test_evaluate_pnp_forward_mode(cuda_device, mode, dof, S, float_bounds, out_jac):
    c = build_case(dof, 96, S, 3, cuda_device, bounds=not float_bounds)
    if float_bounds:
        poses_bm = c["poses"].transpose(0, 1)
        c["lb"], c["ub"], margin = bm.place_bounds(c["x3d"], poses_bm, c["cam_mats"], c["z_min"], False)
        assert margin > bm.BOUND_GAP, margin
    got = _evaluate_layer(c, torch.float32, cuda_device, out_jac, mode)
    ref = _evaluate_layer(c, torch.float64, torch.device("cpu"), True)
    ref = dict(zip(OUTPUTS, ref))
    for k, g in zip(OUTPUTS if out_jac else ("cost",), got):
        assert g is not None and torch.isfinite(g).all(), k
        err = hv.rel_rows(g, ref[k], 1)
        assert (err < 2e-3).all(), (k, err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fwad", "jvp", "linearize"])
def test_gn_step_forward_mode(cuda_device, mode):
    """LMSolver.gn_step in forward mode (the residual / Jacobian tangents) against the float64 composite's forward AD."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.levenberg_marquardt import LMSolver
    c = build_case(6, 80, 1, 3, cuda_device, bounds=True)
    solver = LMSolver(dof=6, num_iter=3)
    names = ("x3d", "x2d", "w2d", "delta", "cam", "lb", "ub")
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], cam=c["cam_mats"], lb=c["lb"], ub=c["ub"])

    def step(dev, dtype, mode):
        def f(x3d, x2d, w2d, delta, cam, lb, ub):
            camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
            return (solver.gn_step(x3d, x2d, w2d, c["poses"][0].to(dev, dtype), camera, HuberPnPCost(delta=delta)),)
        return forward_mode(f, [src[k].to(dev, dtype) for k in names], [c["t"][k].to(dev, dtype) for k in names],
                            mode)[0]
    got, ref = step(cuda_device, torch.float32, mode), step(torch.device("cpu"), torch.float64, "fwad")
    assert got is not None
    err = hv.rel_rows(got, ref, 1)
    assert (err < 5e-3).all(), err.max()


def _mc_problem(dev, B=4, N=128, M=128, seed=21):
    return hv._mc_setup(dev, B=B, N=N, M=M, seed=seed)


def _mc_outputs(leaves, noise, layer, with_plus):
    """logw (M, B), cost_init (B), pose_opt_plus (B, 7) | None and the Monte-Carlo loss of the 6DoF training step."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
    x3d, x2d, w2d, delta, pose_init, cam, lb, ub = leaves
    camera = PerspectiveCamera(cam_mats=cam, lb=lb, ub=ub)
    _, _, plus, _, logw, cost_init = layer.monte_carlo_forward(
        x3d, x2d, w2d, camera, HuberPnPCost(delta=delta), pose_init=pose_init, force_init_solve=False,
        with_cost=True, with_pose_opt_plus=with_plus, amis_noise=noise)
    loss = MonteCarloPoseLoss().to(x3d.device)(logw, cost_init, 1.0)
    return [logw, cost_init, loss] + ([plus] if with_plus else [])


@pytest.mark.gpu
@pytest.mark.parametrize("N", [512, 16384])
def test_training_step_adjoint_identity(cuda_device, N):
    """The 6DoF training step's logw, cost_init (pose_init with a tangent), pose_opt_plus and MonteCarloPoseLoss under
    forward AD against the same outputs' native reverse mode: <g, J v> = <J^T g, v>."""
    dev = cuda_device
    pc, noise, layer, tangents = _mc_problem(dev, B=3, N=N, M=128)
    gen = torch.Generator().manual_seed(5)
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x.detach(), t) for x, t in zip(hv._mc_leaves(pc, dev), tangents)]
        outs = _mc_outputs(duals, noise, layer, True)
        jv = [fwAD.unpack_dual(o).tangent for o in outs]
        prim = [fwAD.unpack_dual(o).primal for o in outs]
    assert all(t is not None for t in jv)
    gs = [torch.randn(p.shape, generator=gen).to(dev) for p in prim]
    leaves = hv._mc_leaves(pc, dev)
    outs = _mc_outputs(leaves, noise, layer, True)
    for o, p in zip(outs, prim):
        assert torch.equal(o.detach(), p.detach())
    for i, (g, t) in enumerate(zip(gs, jv)):
        vjp = torch.autograd.grad((outs[i] * g).sum(), leaves, retain_graph=True, allow_unused=True)
        lhs = float((g.double() * t.double()).sum())
        terms = [(a.double() * v.double()).sum() for a, v in zip(vjp, tangents) if a is not None]
        rhs = float(sum(terms))
        mag = float((g.double() * t.double()).abs().sum()) + float(sum(x.abs() for x in terms))
        assert abs(lhs - rhs) <= 1e-3 * mag, (i, lhs, rhs, mag)


@pytest.mark.gpu
def test_adaptive_delta_tangent_reaches_the_cost(cuda_device):
    """AdaptiveHuberPnPCost.set_param keeps w2d's tangent in delta (the torch path), and the cost sees it."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    c = build_case(6, 64, 1, 3, cuda_device)

    def cost_tangent(dev, dtype):
        with fwAD.dual_level():
            w2d = _dual(c["w2d"].to(dev, dtype), c["t"]["w2d"].to(dev))
            cf = AdaptiveHuberPnPCost(relative_delta=0.1)
            cf.set_param(c["x2d"].to(dev, dtype), w2d)
            assert fwAD.unpack_dual(cf.delta).tangent is not None
            cost = evaluate_pnp(c["x3d"].to(dev, dtype), c["x2d"].to(dev, dtype), w2d,
                                _dual(c["poses"].to(dev, dtype), torch.zeros_like(c["poses"])),
                                PerspectiveCamera(cam_mats=c["cam_mats"].to(dev, dtype)), cf, out_cost=True)[1]
            return fwAD.unpack_dual(cost).tangent
    got, ref = cost_tangent(cuda_device, torch.float32), cost_tangent(torch.device("cpu"), torch.float64)
    assert (hv.rel_rows(got, ref, 1) < 2e-3).all()


@pytest.mark.gpu
def test_traced_forward_mode_raises_or_matches(cuda_device):
    """Under torch.compile a forward tangent through evaluate_pnp raises a clear error or gives the eager tangent,
    never a silent zero."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import HuberPnPCost
    c = build_case(6, 64, 1, 2, cuda_device)
    camera = PerspectiveCamera(cam_mats=c["cam_mats"], z_min=c["z_min"])

    def f(x2d, pose):
        return evaluate_pnp(c["x3d"], x2d, c["w2d"], pose, camera, HuberPnPCost(delta=c["delta"]), out_cost=True)[1]
    with fwAD.dual_level():
        args = (fwAD.make_dual(c["x2d"], c["t"]["x2d"]), fwAD.make_dual(c["poses"], c["t"]["pose"]))
        eager = fwAD.unpack_dual(f(*args)).tangent
        try:
            traced = fwAD.unpack_dual(torch.compile(f, backend="eager")(*args)).tangent
        except Exception as e:                                     # noqa: BLE001 -- the error must name the cause
            assert "forward-mode" in str(e), e
            return
    assert traced is not None and torch.allclose(traced, eager, rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_opcheck_evaluate_jvp(cuda_device):
    c = build_case(6, 40, 3, 2, cuda_device, bounds=True)
    t = c["t"]
    args = (c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"], c["poses"],
            *(t.get(k) for k in native.JVP_TANGENTS), 6, c["z_min"], 1e-10, True, [True, True, True])
    torch.library.opcheck(ops.evaluate_jvp.op, args)


def _adjoint(fn, leaves, tangents, seed=7):
    """|<g, J v> - <J^T g, v>| / sum |terms| per object (axis 0 of the output) for fn(*leaves) -> one tensor: J v by
    forward AD, J^T g by the layer's reverse mode."""
    with fwAD.dual_level():
        out = fn(*(fwAD.make_dual(x.detach(), t) for x, t in zip(leaves, tangents)))
        jv = fwAD.unpack_dual(out).tangent
    assert jv is not None
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).to(out.device)
    ls = [x.detach().clone().requires_grad_(True) for x in leaves]
    vjp = torch.autograd.grad((fn(*ls) * g).sum(), ls, allow_unused=True)
    lhs = (g.double() * jv.double()).reshape(out.shape[0], -1)
    B = out.shape[0]
    rhs = [(a.double() * v.double()).reshape(B, -1) for a, v in zip(vjp, tangents) if a is not None]
    gap = (lhs.sum(1) - sum(r.sum(1) for r in rhs)).abs()
    mag = lhs.abs().sum(1) + sum(r.abs().sum(1) for r in rhs)
    return float((gap / mag).max())


def _problem_leaves(c):
    return [c["x3d"], c["x2d"], c["w2d"], c["cam_mats"], c["lb"], c["ub"], c["delta"]]


def _problem_tangents(c):
    return [c["t"][k] for k in ("x3d", "x2d", "w2d", "cam", "lb", "ub", "delta")]


@pytest.mark.gpu
@pytest.mark.parametrize("N", [512, 16384])
def test_evaluate_cost_adjoint_identity(cuda_device, N):
    """The evaluate_cost formula (poses with a tangent, tensor bounds) against cost_backward / cost_pose_backward /
    cost_camera_backward."""
    c = build_case(6, N, 3, 3, cuda_device, bounds=True)
    fn = lambda *a: ops.evaluate_cost(*a[:7], a[7].transpose(0, 1), 6, c["z_min"]).transpose(0, 1)       # (B, S)
    poses, t_pose = (x.transpose(0, 1).contiguous() for x in (c["poses"], c["t"]["pose"]))           # object-major
    assert _adjoint(fn, _problem_leaves(c) + [poses], _problem_tangents(c) + [t_pose]) < ADJ_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("N", [512, 16384])
def test_lm_solve_pose_opt_plus_adjoint_identity(cuda_device, N):
    """The lm_solve formula's pose_opt_plus tangent (gn_plus_hvp's J u) against its backward (gn_plus_backward /
    gn_plus_camera_backward)."""
    c = build_case(6, N, 1, 3, cuda_device, bounds=True)
    ints, floats = ops.param_lists(None, 6, lm_iter=0, z_min=c["z_min"])
    pose = c["poses"][0]
    fn = lambda *a: ops.lm_solve(*a, pose, ints, floats, False, False, True)[3]
    assert _adjoint(fn, _problem_leaves(c), _problem_tangents(c)) < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("N", [512, 16384])
def test_pose_opt_plus_tangent_against_float64(cuda_device, N):
    """pose_opt_plus's tangent through the layer (_PosePlus under forward AD, every problem input with a tangent, the
    pose held constant) against the oracle's float64 forward AD of pose_add(pose, gn_step(pose)), per object."""
    from epropnp.autograd import pose_plus_autograd
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.levenberg_marquardt import LMSolver
    c = build_case(6, N, 1, 4, cuda_device, bounds=True)
    solver = LMSolver(dof=6, num_iter=3)
    pose = c["poses"][0]
    names = ("x3d", "x2d", "w2d", "delta", "cam", "lb", "ub")
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], cam=c["cam_mats"], lb=c["lb"], ub=c["ub"])
    with fwAD.dual_level():
        d = {k: _dual(src[k], c["t"][k]) for k in names}
        camera = PerspectiveCamera(cam_mats=d["cam"], z_min=c["z_min"], lb=d["lb"], ub=d["ub"])
        got = fwAD.unpack_dual(pose_plus_autograd(solver, d["x3d"], d["x2d"], d["w2d"], pose, camera,
                                                  HuberPnPCost(delta=d["delta"]))).tangent
    assert got is not None

    def oracle(dtype):
        def plus(x3d, x2d, w2d, delta, cam, lb, ub):
            p = pose.cpu().to(dtype)
            return orc.pose_add(p, orc.gn_step(x3d, x2d, w2d, orc.Camera(cam, c["z_min"], lb, ub), delta, p,
                                               eps=solver.eps))
        return torch.func.jvp(plus, tuple(src[k].detach().cpu().to(dtype) for k in names),
                              tuple(c["t"][k].cpu().to(dtype) for k in names))[1]
    ref64, ref32 = oracle(torch.float64), oracle(torch.float32)
    err, floor = hv.rel_rows(got, ref64, 1), hv.rel_rows(ref32, ref64, 1)
    assert (err < np.maximum(REL_MIN, K_FLOOR * floor)).all(), (err.max(), floor.max())


@pytest.mark.gpu
def test_mc_epilogue_loss_and_weights_refuse_a_tangent(cuda_device):
    """The epilogue's loss and sample weights have no forward formula: a tangent raises instead of going missing; lse
    has one."""
    logw = torch.randn(3, 16, device=cuda_device)
    t = torch.randn(3, 16, device=cuda_device)
    with fwAD.dual_level():
        d = fwAD.make_dual(logw, t)
        lse = ops.mc_epilogue(d, None, None, None, True, False, False, False)[0]
        ref = (torch.softmax(logw, 1) * t).sum(1)
        assert torch.allclose(fwAD.unpack_dual(lse).tangent, ref, rtol=1e-5, atol=1e-6)
        with pytest.raises(RuntimeError, match="no forward-mode formula"):
            ops.mc_epilogue(d, None, None, torch.zeros(3, device=cuda_device), False, True, False, False)
        with pytest.raises(RuntimeError, match="no forward-mode formula"):
            ops.mc_epilogue(d, None, None, None, False, False, True, False)
