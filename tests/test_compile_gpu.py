"""torch.compile / torch.export of the layer on the H100: every epropnp operator passes opcheck on CUDA tensors at a
resident (N = 512) and a cluster-split (N = 16 384) size; the four call sequences of tests/compile_flows.py compile with
aot_eager to eager's bits, and with inductor (default mode) to eager within the parity bounds (inductor's Triton code
covers only the caller's glue -- set_param's variance, pnp_normalize -- and may order it differently); the 6DoF training
step runs under mode="reduce-overhead" (CUDA graphs) and equals eager with seed tensors, or draws anew without; the
6DoF test-time module and monte_carlo_forward export with a dynamic batch; LMSolver.gn_step differentiates under
compile."""
import numpy as np
import pytest
import torch
import torch._dynamo.testing

import compile_flows as cf
from conftest import assert_lm_parity, err_vs, record_parity
from epropnp.camera import PerspectiveCamera
from epropnp.common import evaluate_pnp
from epropnp.cost_fun import AdaptiveHuberPnPCost, HuberPnPCost
from epropnp.epnp import EPnPSolver
from epropnp.epropnp import EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import ops
from epropnp_b200.synth import make_problem
from test_compile_simt_cpu import opcheck_cases

pytestmark = pytest.mark.gpu
FLOW = dict(B=32, N=512, M=512, P=4)


@pytest.fixture
def dev(cuda_device, monkeypatch):
    # Python floats (Huber and solver constants, loss weights) specialised, as the layer uses them: unspecialised, they
    # would become CPU scalar inputs whose arithmetic inductor compiles to host C++ kernels
    monkeypatch.setattr(torch._dynamo.config, "specialize_float", True)
    torch._dynamo.reset()
    yield cuda_device
    torch._dynamo.reset()


@pytest.mark.parametrize("N", [512, 16384])
def test_opcheck_every_operator_on_cuda(dev, N):
    cases = opcheck_cases(dev, B=2, N=N, M=64)
    for op, args in cases:
        if op is ops.rslm.op:
            args = args[:-1] + (True,)                   # above the resident limit: the cluster-split initialiser
        torch.library.opcheck(op, args)


@pytest.mark.parametrize("kind", cf.KINDS)
def test_aot_eager_equals_eager_bit_for_bit(dev, kind):
    eager = cf.run(cf.build(kind, dev, **FLOW))
    flow = cf.build(kind, dev, **FLOW)
    got = cf.run(flow, torch.compile(flow.fn, backend="aot_eager", fullgraph=True, dynamic=True))
    for a, b in zip(eager[0] + eager[1], got[0] + got[1]):
        assert a.shape == b.shape and torch.equal(a, b)


def _pose_cost(kind, flow, pose):
    """Per-object cost of `pose` on the flow's problem with a fixed Huber threshold (assert_lm_parity's flip clause)."""
    x3d, x2d, w2d, cam = (flow.args[i].detach() for i in range(4)) if kind != "det_train" else \
        (flow.args[0].detach(), flow.args[1], flow.args[2].detach(), flow.args[4])
    camera = PerspectiveCamera(cam_mats=cam, z_min=0.5 if pose.shape[-1] == 4 else 0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(x2d, w2d)
    with torch.no_grad():
        return evaluate_pnp(x3d, x2d, w2d, pose, camera, cost_fun, out_cost=True)[1]


def _compare_inductor(kind, flow, got, want, tag):
    stats = {}
    outs = dict(det_infer=("pose", "grid_cost"), det_train=("loss", "logw", "cost_init", "plus"),
                train6=("loss", "logw", "cost_init", "plus"), test6=("pose",))[kind]
    for name, a, b in zip(outs, got[0], want[0]):
        if name in ("pose", "plus"):
            stats[f"{name}_flip_frac"] = assert_lm_parity(a.cpu(), _pose_cost(kind, flow, a).cpu(), b.cpu(),
                                                          _pose_cost(kind, flow, b).cpu(), 1e-4, what=f"{tag} {name}")
        else:
            stats[f"{name}_rel"] = err_vs(a.cpu().numpy(), b.cpu().numpy())
    for i, (a, b) in enumerate(zip(got[1], want[1])):
        stats[f"grad{i}_rel"] = err_vs(a.cpu().numpy(), b.cpu().numpy())
    record_parity(f"compile/{tag}", **stats)
    for k, v in stats.items():
        if k.endswith("_rel"):
            assert v < 1e-4, (tag, k, v)


@pytest.mark.parametrize("kind", cf.KINDS)
def test_inductor_matches_eager(dev, kind):
    want = cf.run(cf.build(kind, dev, **FLOW))
    flow = cf.build(kind, dev, **FLOW)
    got = cf.run(flow, torch.compile(flow.fn))
    _compare_inductor(kind, flow, got, want, f"inductor/{kind}")


def test_inductor_det_batch_varies(dev):
    """torch.compile's default dynamic-shape policy: the second batch size recompiles with a symbolic batch, the third
    reuses that graph."""
    compiled, frames = None, []
    counter = torch._dynamo.testing.CompileCounterWithBackend("inductor")
    for B in (32, 48, 64):
        flow = cf.build("det_infer", dev, **dict(FLOW, B=B))
        compiled = compiled or torch.compile(flow.fn, backend=counter)
        got = cf.run(flow, compiled)
        frames.append(counter.frame_count)
        _compare_inductor("det_infer", flow, got, cf.run(cf.build("det_infer", dev, **dict(FLOW, B=B))),
                          f"inductor/det_infer_B{B}")
    assert frames[2] == frames[1], frames


@pytest.mark.parametrize("N", [512, 16384])
def test_reduce_overhead_training_step(dev, N):
    """mode="reduce-overhead": CUDA-graph replays on new inputs and seed tensors (written before each call) equal the
    same compiled step run without graphs bit for bit, and eager within the inductor bounds."""
    size = dict(FLOW, N=N, B=32 if N == 512 else 4)
    build = lambda data_seed: cf.build("train6", dev, seeds="tensor", data_seed=data_seed, cluster_split=N > 512,
                                       **size)
    flow, plain = build(1), build(1)
    step, plain_step = torch.compile(flow.fn, mode="reduce-overhead"), torch.compile(plain.fn)
    for trial in range(3):
        data = build(10 + trial)
        for f in (flow, plain, data):
            for i, t in enumerate(data.args):
                if f is not data:
                    (f.args[i].data if i in f.leaves else f.args[i]).copy_(t)
            f.args[-2].fill_(100 + trial)
            f.args[-1].fill_(200 + trial)
        got, same = cf.run(flow, step), cf.run(plain, plain_step)
        for a, b in zip(got[0] + got[1], same[0] + same[1]):
            assert torch.equal(a, b), trial
        _compare_inductor("train6", data, got, cf.run(data), f"reduce_overhead/train6_N{N}_trial{trial}")


def test_reduce_overhead_without_seed_draws_anew(dev):
    flow = cf.build("train6", dev, seeds="none", **FLOW)
    step = torch.compile(flow.fn, mode="reduce-overhead")
    logws = [cf.run(flow, step)[0][1] for _ in range(4)]
    for a, b in zip(logws, logws[1:]):
        assert not torch.equal(a, b)


class _Test6(torch.nn.Module):
    def __init__(self, M=64):
        super().__init__()
        self.layer = EProPnP6DoF(mc_samples=M, num_iter=4, solver=LMSolver(dof=6, num_iter=3, init_solver=EPnPSolver()))

    def forward(self, x3d, x2d, w2d, cam):
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d, w2d)
        return self.layer(x3d, x2d, w2d, PerspectiveCamera(cam_mats=cam), cost_fun, fast_mode=True)[0]


class _MonteCarlo(_Test6):
    def forward(self, x3d, x2d, w2d, cam, pose_init, seed):
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d, w2d)
        pose_opt, _, _, samples, logw, _ = self.layer.monte_carlo_forward(
            x3d, x2d, w2d, PerspectiveCamera(cam_mats=cam), cost_fun, pose_init=pose_init, force_init_solve=False,
            amis_seed=seed)
        return pose_opt, samples, logw


@pytest.mark.parametrize("module", [_Test6, _MonteCarlo])
def test_export_with_dynamic_batch(dev, module):
    def inputs(B, seed):
        pc = make_problem(B, 512, seed=seed, dof=6)
        args = tuple(pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats"))
        if module is _MonteCarlo:
            args += (pc["pose_init"].to(dev), torch.tensor([5], dtype=torch.int64, device=dev))
        return args
    m = module().to(dev)
    B = torch.export.Dim("B", min=2, max=4096)
    shapes = [{0: B}] * 4 + ([{0: B}, None] if module is _MonteCarlo else [])
    with torch.no_grad():
        ep = torch.export.export(m, inputs(16, 1), dynamic_shapes=shapes)
        for b, seed in ((16, 2), (40, 3)):
            args = inputs(b, seed)
            for a, e in zip(ep.module()(*args) if module is _MonteCarlo else (ep.module()(*args),),
                            m(*args) if module is _MonteCarlo else (m(*args),)):
                assert a.shape == e.shape and torch.equal(a, e), b


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_gn_step_under_compile(dev, backend):
    pc = make_problem(32, 512, seed=9, dof=6)
    solver = LMSolver(dof=6)

    def step(x3d, x2d, w2d, cam, pose):
        camera, cost_fun = PerspectiveCamera(cam_mats=cam), HuberPnPCost(delta=3.0)
        return solver.pose_add(pose, solver.gn_step(x3d, x2d, w2d, pose, camera, cost_fun), camera)

    def grads(fn):
        leaves = [pc[k].to(dev).requires_grad_(True) for k in ("x3d", "x2d", "w2d", "cam_mats")]
        out = fn(*leaves, pc["pose_init"].to(dev))
        (out * torch.linspace(-1, 1, out.numel(), device=dev).reshape(out.shape)).sum().backward()
        return [out.detach()] + [t.grad for t in leaves]
    want, got = grads(step), grads(torch.compile(step, backend=backend, dynamic=True))
    errs = [err_vs(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(got, want)]
    record_parity(f"compile/gn_step/{backend}", out_rel=errs[0], grad_rel_max=float(np.max(errs[1:])))
    if backend == "aot_eager":
        assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert max(errs) < 1e-4, errs
