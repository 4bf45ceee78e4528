"""torch.compile over the layer, with the kernels under the CPU SIMT emulator and CPU tensors: the four call sequences of
tests/compile_flows.py trace without a graph break, compile (aot_eager, dynamic shapes, fullgraph) to the same bits as
eager in outputs and gradients, keep one graph while the batch varies, and raise the library's refusals as eager does.
Every epropnp operator passes torch.library.opcheck.  aot_eager needs no C++ toolchain; inductor runs in the GPU suite."""
import pytest
import torch
import torch._dynamo.testing
import torch.fx.experimental._config

import compile_flows as cf
import simt_native
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import HuberPnPCost
from epropnp.epropnp import EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import capi, native, ops
from epropnp_b200.synth import make_problem

SIZES = dict(B=3, N=32)


@pytest.fixture
def dev(monkeypatch):
    torch._dynamo.reset()
    yield simt_native.install(monkeypatch)
    torch._dynamo.reset()


@pytest.mark.parametrize("kind", cf.KINDS)
def test_no_graph_breaks(dev, kind):
    flow = cf.build(kind, dev, **SIZES)
    explained = torch._dynamo.explain(flow.fn)(*flow.args)
    assert explained.graph_break_count == 0, explained.break_reasons
    assert explained.graph_count == 1


@pytest.mark.parametrize("kind", cf.KINDS)
def test_compiled_equals_eager_bit_for_bit(dev, kind):
    eager = cf.run(cf.build(kind, dev, **SIZES))
    flow = cf.build(kind, dev, **SIZES)
    compiled = cf.run(flow, torch.compile(flow.fn, backend="aot_eager", fullgraph=True, dynamic=True))
    for a, b in zip(eager[0] + eager[1], compiled[0] + compiled[1]):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


@pytest.mark.parametrize("kind", ["det_infer", "train6"])
def test_varying_batch_keeps_one_graph(dev, monkeypatch, kind):
    # B = 3 equals the camera's 3 x 3: with duck shaping the two would share one symbol, and the rotation product
    # would pin it to 3
    monkeypatch.setattr(torch.fx.experimental._config, "use_duck_shape", False)
    counter = torch._dynamo.testing.CompileCounterWithBackend("aot_eager")
    compiled, frames = None, []
    for B in (3, 5, 7):
        flow = cf.build(kind, dev, B=B, N=SIZES["N"])
        compiled = compiled or torch.compile(flow.fn, backend=counter, fullgraph=True, dynamic=True)
        got = cf.run(flow, compiled)
        frames.append(counter.frame_count)
        want = cf.run(cf.build(kind, dev, B=B, N=SIZES["N"]))
        for a, b in zip(got[0] + got[1], want[0] + want[1]):
            assert torch.equal(a, b), B
    assert frames[0] > 0 and frames == frames[:1] * 3, frames


@pytest.mark.parametrize("kind", ["train6", "test6"])
def test_empty_batch(dev, kind):
    """B = 0: the reference's empty results (and, training, zero gradients) under compile as eagerly.  (The Det flows
    raise at B = 0 eagerly as well: the orientation grid's reshape, and LMSolver.forward's differentiable
    pose_opt_plus, which the library refuses for an empty batch.)"""
    want = cf.run(cf.build(kind, dev, B=0, N=SIZES["N"]))
    flow = cf.build(kind, dev, B=0, N=SIZES["N"])
    got = cf.run(flow, torch.compile(flow.fn, backend="aot_eager", dynamic=True))
    for a, b in zip(got[0] + got[1], want[0] + want[1]):
        torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)         # the loss: the mean of nothing


def test_refusals_raise_under_compile(dev, monkeypatch):
    """The library's refusals reach the caller unchanged: fast mode with lm_iter = 0, and RSLM above the resident
    limit without cluster_split."""
    pc = make_problem(2, 24, seed=3, dof=6)
    x3d, x2d, w2d = pc["x3d"], pc["x2d"], pc["w2d"]
    camera, cost_fun = PerspectiveCamera(cam_mats=pc["cam_mats"]), HuberPnPCost(delta=5.0)
    layer = EProPnP6DoF(mc_samples=16, num_iter=2, solver=LMSolver(dof=6, num_iter=0))
    fn = lambda x3d, pose: layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=pose,
                                                     force_init_solve=False, fast_mode=True, amis_seed=1)[0]
    with pytest.raises(native.NativeError) as eager:
        fn(x3d, pc["pose_init"])
    with pytest.raises(native.NativeError) as compiled:
        torch.compile(fn, backend="aot_eager", fullgraph=True)(x3d, pc["pose_init"])
    assert str(compiled.value) == str(eager.value)

    N = native.max_points(6) + 1
    pc = make_problem(1, N, seed=4, dof=6)
    rslm = cf.SeededRSLM(dof=6, num_points=8, num_proposals=2, num_iter=1)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"])
    fn = lambda x3d, x2d, w2d: rslm.solve(x3d, x2d, w2d, camera, cost_fun)[0]
    with pytest.raises(native.NativeError) as eager:
        fn(pc["x3d"], pc["x2d"], pc["w2d"])
    with pytest.raises(native.NativeError) as compiled:
        torch.compile(fn, backend="aot_eager", fullgraph=True)(pc["x3d"], pc["x2d"], pc["w2d"])
    assert str(compiled.value) == str(eager.value)


def opcheck_cases(dev, B=2, N=24, M=16, P=4, grad=True):
    """(operator, args) for every epropnp operator on one seeded problem; the forward operators with inputs requiring
    grad, so opcheck also checks their formulas."""
    pc = make_problem(B, N, seed=5, dof=6)
    f = lambda k: pc[k].to(dev)
    leaf = lambda t: t.clone().requires_grad_(grad)
    x3d, x2d, w2d, cam = leaf(f("x3d")), leaf(f("x2d")), leaf(f("w2d")), leaf(f("cam_mats"))
    lb, ub = leaf(torch.full((B, 2), -50.0, device=dev)), leaf(torch.full((B, 2), 700.0, device=dev))
    delta = leaf(torch.full((B,), 5.0, device=dev))
    prob = (x3d, x2d, w2d, cam, lb, ub, delta)
    plain = tuple(t.detach() for t in prob)
    pose = f("pose_init")
    poses = leaf(torch.stack((pose, pose + 0.01)))                                   # (S, B, 7)
    ints, floats = ops.param_lists(None, 6, lm_iter=4, mc_samples=M, mc_iter=2, z_min=0.1)
    samples = (pose[:, None] + 0.01 * torch.randn(B, M, 7, generator=torch.Generator().manual_seed(1)).to(dev))
    logw = torch.randn(B, M, generator=torch.Generator().manual_seed(2)).to(dev)
    lse = torch.logsumexp(logw, 1)
    g = lambda *s: torch.randn(*s, generator=torch.Generator().manual_seed(3)).to(dev)
    inds = torch.randint(0, N, (P, B, 8), generator=torch.Generator().manual_seed(4), dtype=torch.int32).to(dev)
    start = pose[None].expand(P, B, 7).contiguous()
    return [
        (ops.adaptive_delta.op, (plain[1], plain[2], 0.5)),
        (ops.evaluate_cost.op, prob + (poses, 6, 0.1)),
        (ops.evaluate_full.op, prob + (poses, 6, 0.1, 1e-10, True, True, True, True)),
        (ops.lm_solve.op, plain + (pose, ints, floats, True, True, True)),
        (ops.lm_amis_fused.op, prob + (pose, leaf(pose.clone()), None, None, None, 9, None, ints, floats, True, True,
                                    False)),
        (ops.rslm_draw.op, (f("x3d"), f("x2d"), f("w2d"), f("cam_mats"), None, P, 8, 6, 1e-5, 3, None)),
        (ops.rslm.op, plain + (inds, start, ints, floats, False)),
        (ops.epnp_init.op, (f("x3d"), f("x2d"), f("w2d"), f("cam_mats"), 0.5)),
        (ops.mc_epilogue.op, (leaf(logw), samples, pose, None, True, False, True, True)),
        (ops.cost_backward.op, plain + (samples, g(B, M), pose[:, None], g(B, 1), 6, 0.1, [True] * 4)),
        (ops.cost_pose_backward.op, plain + (samples, g(B, M), 6, 0.1)),
        (ops.cost_camera_backward.op, plain + (samples, g(B, M), None, None, 6, 0.1, [True] * 3)),
        (ops.gn_plus_backward.op, plain + (pose, g(B, 7), 6, 0.1, 1e-5, 1e-10, [True, False, True, True])),
        (ops.gn_plus_camera_backward.op, plain + (pose, g(B, 7), 6, 0.1, 1e-5, 1e-10, [True] * 3)),
        (ops.evaluate_backward.op, plain + (poses.detach(), 6, 0.1, 1e-10, True, g(2, B, 2 * N), None, g(2, B),
                                         [True] * 8)),
        (ops.mc_lse_backward.op, (logw, lse, g(B))),
    ]


def test_opcheck_every_operator(dev):
    cases = opcheck_cases(dev)
    assert {op for op, _ in cases} == set(ops.FORWARD + ops.BACKWARD)
    for op, args in cases:
        torch.library.opcheck(op, args)


def test_eager_calls_skip_the_dispatcher_only_where_nothing_is_lost(dev, monkeypatch):
    """Eagerly, with nothing requiring grad, the layer's entry points run the implementation directly; with an input
    requiring grad they go through the operator (its autograd formula), with the same values."""
    calls = []
    monkeypatch.setattr(native, "evaluate_cost", lambda *a, _f=native.evaluate_cost: calls.append(1) or _f(*a))
    pc = make_problem(2, 24, seed=6, dof=6)
    prob = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, torch.tensor(5.0))
    poses = pc["pose_init"][None]
    direct = ops.evaluate_cost(*prob, poses, 6, 0.1)
    assert direct.grad_fn is None and len(calls) == 1
    x3d = pc["x3d"].clone().requires_grad_(True)
    through = ops.evaluate_cost(x3d, *prob[1:], poses, 6, 0.1)
    assert through.grad_fn is not None and "epropnp_evaluate_cost" in type(through.grad_fn).__name__
    assert torch.equal(direct, through.detach()) and len(calls) == 2


def test_param_lists_round_trip(dev):
    """The (ints, floats) lists carry every field of EpnpParams, so the rebuilt block equals the library's own."""
    p = capi.default_params(4, lm_iter=7, z_min=0.25, mc_samples=96, acg_dispersion=0.002)
    q = ops.make_params(*ops.param_lists(p))
    assert bytes(q) == bytes(p)
    assert bytes(ops.make_params(*ops.param_lists(None, 4, lm_iter=7, z_min=0.25, mc_samples=96,
                                                  acg_dispersion=0.002))) == bytes(p)


@pytest.mark.parametrize("want", [(True, True, False), (False, True, False), (True, False, True)])
def test_requested_evaluate_outputs_are_differentiable(dev, want):
    """evaluate_full's formula: every requested output (residual, Jacobian, cost in any combination) carries a gradient,
    eagerly and compiled alike."""
    pc = make_problem(2, 24, seed=7, dof=6)
    want_r, want_j, want_c = want
    for compiled in (False, True):
        x3d = pc["x3d"].clone().requires_grad_(True)
        fn = lambda x3d: ops.evaluate_full(x3d, pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, torch.tensor(5.0),
                                           pc["pose_init"][None], 6, 0.1, 1e-10, True, want_r, want_j, want_c)
        r, c, j = (torch.compile(fn, backend="aot_eager", fullgraph=True) if compiled else fn)(x3d)
        live = [t for t, w in zip((r, c, j), (want_r, want_c, want_j)) if w]
        assert all(t.requires_grad for t in live) and not any(t.requires_grad for t in (r, c, j) if t.numel() == 0)
        sum(t.sum() for t in live).backward()
        assert x3d.grad is not None and x3d.grad.abs().sum() > 0
