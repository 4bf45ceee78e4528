"""LMSolver from stacked starts, pose_init (S, B, D) (lm_stacked_kernel through epnp_lm_solve_stacked_f32), against the
(B, D) solve (lm_warp_kernel through epnp_lm_solve_f32): start s of object b must give what the (B, D) call gives with
pose_init = pose_init[s], bit for bit, in pose_opt, pose_cov, cost, pose_opt_plus and cost_init -- and what the
replicate-and-flatten call (the points copied S times, S B objects) gives.  N covers the staged kernel (5, 300, 640),
one warp from global memory (641) and eight warps (4096); S = 1, 3 (one CTA per object) and 33 (five CTAs of seven
hypothesis warps, two idle); B is several waves of CTAs.  Also leading dimensions, empty stacks, every refusal, CUDA-graph
replay, torch.compile and opcheck.  tests/test_lm_stacked_simt_cpu.py runs the same checks under the SIMT emulator."""
import math

import pytest
import torch

from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import native, ops
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

OUTPUTS = ("pose_opt", "pose_cov", "cost", "pose_opt_plus", "cost_init")


def case(dof, N, S, B, bounds="none", mode="lm", outputs=OUTPUTS):
    return dict(dof=dof, N=N, S=S, B=B, bounds=bounds, mode=mode, outputs=outputs,
                id=f"dof{dof}-N{N}-S{S}-B{B}-{bounds}-{mode}-{len(outputs)}out")


CASES = [
    case(6, 5, 3, 3000, "none", "lm"),
    case(4, 5, 33, 300, "scalar", "fast"),
    case(6, 300, 33, 600, "tensor", "lm"),
    case(4, 300, 3, 3000, "none", "fast", ("pose_opt",)),
    case(6, 640, 1, 3000, "scalar", "fast"),
    case(4, 640, 33, 200, "tensor", "lm", ("pose_opt", "pose_opt_plus")),
    case(6, 641, 3, 1500, "tensor", "lm"),
    case(4, 641, 33, 100, "none", "fast"),
    case(6, 4096, 3, 300, "scalar", "lm", ("pose_opt", "cost")),
    case(4, 4096, 1, 200, "tensor", "fast"),
    case(6, 4096, 33, 40, "none", "fast"),
]


class Setup:
    """One seeded problem of B objects with S starts each (the given pose, and S - 1 perturbations of it; in 4DoF the
    second start is the yaw + pi twin), as native.Problem and as the LMSolver's camera / cost."""

    def __init__(self, dev, dof, N, S, B, bounds="none", seed=0):
        pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.1)
        t = {k: pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats", "pose_init")}
        self.dof, self.D, self.S, self.B, self.N = dof, (7 if dof == 6 else 4), S, B, N
        self.x3d, self.x2d, self.w2d, self.cam = t["x3d"], t["x2d"], t["w2d"], t["cam_mats"]
        if bounds == "scalar":
            self.lb, self.ub = -100.0, 800.0
        elif bounds == "tensor":
            g = torch.Generator().manual_seed(seed + 1)
            self.lb = (torch.rand(B, 2, generator=g) * 100.0 - 150.0).to(dev)
            self.ub = (torch.rand(B, 2, generator=g) * 100.0 + 600.0).to(dev)
        else:
            self.lb = self.ub = None
        self.camera = PerspectiveCamera(cam_mats=self.cam, z_min=0.1, lb=self.lb, ub=self.ub)
        self.cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        self.cost_fun.set_param(self.x2d, self.w2d)
        self.prob = native.Problem(self.x3d, self.x2d, self.w2d, self.cam, self.lb, self.ub, self.cost_fun.delta)
        self.starts = stack_starts(t["pose_init"], S, dof, seed)

    def args(self):
        return self.x3d, self.x2d, self.w2d, self.camera, self.cost_fun

    def flattened(self):
        """The problem replicated S times: S B objects, object s B + b a copy of object b."""
        rep = lambda v: None if v is None else v.unsqueeze(0).expand((self.S,) + v.shape).reshape(
            (self.S * v.shape[0],) + v.shape[1:])
        p = self.prob
        return native.Problem(rep(p.x3d), rep(p.x2d), rep(p.w2d), rep(p.cam), rep(p.lb), rep(p.ub), rep(p.delta))


def stack_starts(pose, S, dof, seed):
    g = torch.Generator().manual_seed(seed + 2)
    noise = lambda *s: torch.randn(*s, generator=g).to(pose.device)
    starts = [pose]
    for s in range(1, S):
        p = pose.clone()
        p[:, :3] += 0.1 * noise(pose.shape[0], 3)
        if dof == 6:
            q = p[:, 3:] + 0.2 * noise(pose.shape[0], 4)
            p[:, 3:] = q / q.norm(dim=-1, keepdim=True)
        else:
            p[:, 3] += math.pi if s == 1 else 0.5 * float(noise(1))
        starts.append(p)
    return torch.stack(starts)


def same(a, b):
    """Bit-for-bit equality, NaN payloads included (a start that diverges must diverge alike)."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def params(dof, mode, lm_iter=None):
    if mode == "lm":
        return native.default_params(dof, lm_iter=10 if lm_iter is None else lm_iter)
    return native.default_params(dof, lm_iter=5 if lm_iter is None else lm_iter, fast_mode=1)


def _want_kwargs(outputs):
    names = dict(pose_cov="cov", cost="cost", pose_opt_plus="plus", cost_init="cost_init")
    return {f"want_{names[k]}": True for k in outputs if k != "pose_opt"}


def check_case(dev, c):
    """Every start of every object against its own (B, D) call and against the replicate-and-flatten call."""
    st = Setup(dev, c["dof"], c["N"], c["S"], c["B"], c["bounds"], seed=c["N"] + c["S"])
    p, kw = params(c["dof"], c["mode"]), _want_kwargs(c["outputs"])
    got = native.lm_solve_stacked(st.prob, st.starts, p, **kw)
    flat = native.lm_solve(st.flattened(), st.starts.reshape(-1, st.D), p, **kw)
    for k in OUTPUTS:
        assert (got[k] is None) == (k not in c["outputs"]), k
    for s in range(c["S"]):
        one = native.lm_solve(st.prob, st.starts[s], p, **kw)
        for k in c["outputs"]:
            assert same(got[k][s], one[k]), (k, s)
    for k in c["outputs"]:
        assert same(got[k].reshape(flat[k].shape), flat[k]), k
    assert torch.isfinite(got["pose_opt"]).float().mean() > 0.9


def check_solver_leading_dims(dev, dof=6, N=64, B=5, mode="lm"):
    """LMSolver.forward / solve with pose_init (2, 3, B, D): outputs (2, 3, B, ...) equal to the six (B, D) calls."""
    st = Setup(dev, dof, N, 6, B, "scalar", seed=3)
    solver = LMSolver(dof=dof, num_iter=10 if mode == "lm" else 5)
    starts = st.starts.reshape(2, 3, B, st.D)
    fast = mode != "lm"
    pose, cov, cost, plus = solver(*st.args(), pose_init=starts, with_pose_opt_plus=True, with_pose_cov=True,
                                   with_cost=True, fast_mode=fast)
    assert pose.shape == (2, 3, B, st.D) and cov.shape == (2, 3, B, dof, dof) and cost.shape == (2, 3, B)
    assert plus.shape == (2, 3, B, st.D)
    for i in range(2):
        for j in range(3):
            one = solver(*st.args(), pose_init=starts[i, j], with_pose_opt_plus=True, with_pose_cov=True,
                         with_cost=True, fast_mode=fast)
            for a, b in zip((pose, cov, cost, plus), one):
                assert same(a[i, j], b)
    p2, c2, k2 = solver.solve(*st.args(), pose_init=starts, with_pose_cov=True, with_cost=True, fast_mode=fast)
    assert same(p2, pose) and same(c2, cov) and same(k2, cost)
    only, no_cov, no_cost = solver.solve(*st.args(), pose_init=starts[0], fast_mode=fast)
    assert same(only, pose[0]) and no_cov is None and no_cost is None


def check_empty(dev, dof=6, N=16):
    """S = 0 and B = 0 give empty outputs of the stacked shapes; nothing is launched."""
    solver = LMSolver(dof=dof, num_iter=3)
    D = 7 if dof == 6 else 4
    st = Setup(dev, dof, N, 1, 3, seed=4)
    pose, cov, cost, plus = solver(*st.args(), pose_init=st.starts[:0], with_pose_cov=True, with_cost=True,
                                   with_pose_opt_plus=True)
    assert pose.shape == (0, 3, D) and cov.shape == (0, 3, dof, dof) and cost.shape == (0, 3) and plus.shape == (0, 3, D)
    out = native.lm_solve_stacked(st.prob, st.starts[:0], params(dof, "lm"), want_cov=True, want_cost_init=True)
    assert out["pose_opt"].shape == (0, 3, D) and out["cost_init"].shape == (0, 3)
    z = lambda *s: torch.zeros(s, device=dev)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.delta = z(0)
    empty = (z(0, N, 3), z(0, N, 2), z(0, N, 2), PerspectiveCamera(cam_mats=z(0, 3, 3), z_min=0.1), cost_fun)
    pose, cov, cost, plus = solver(*empty, pose_init=z(4, 0, D), with_pose_cov=True, with_cost=True,
                                   with_pose_opt_plus=True)
    assert pose.shape == (4, 0, D) and cov.shape == (4, 0, dof, dof) and cost.shape == (4, 0) and plus.shape == (4, 0, D)
    assert solver.solve(*empty, pose_init=z(2, 3, 0, D))[0].shape == (2, 3, 0, D)


def check_refusals(dev, dof=6, N=16, B=3):
    st = Setup(dev, dof, N, 2, B, seed=5)
    solver = LMSolver(dof=dof, num_iter=3, init_solver=LMSolver(dof=dof, num_iter=1))
    with pytest.raises(ValueError, match="force_init_solve"):
        solver.solve(*st.args(), pose_init=st.starts, force_init_solve=True)
    with pytest.raises(ValueError, match="pose_init"):
        native.lm_solve_stacked(st.prob, None, params(dof, "lm"))
    with pytest.raises(ValueError, match="pose_init"):
        native.lm_solve_stacked(st.prob, st.starts[0], params(dof, "lm"))                  # (B, D): not stacked
    with pytest.raises(ValueError, match="pose_init"):
        native.lm_solve_stacked(st.prob, st.starts[..., :3], params(dof, "lm"))              # a pose of the wrong width
    with pytest.raises(ValueError, match="stacked pose_init"):
        solver.solve(*st.args(), pose_init=torch.zeros(2, B + 1, st.D, device=dev))
    # a differentiable pose_opt_plus from stacked starts is refused; without a derivative it is not
    x3d = st.x3d.clone().requires_grad_(True)
    with pytest.raises(ValueError, match="not differentiable"):
        solver(x3d, st.x2d, st.w2d, st.camera, st.cost_fun, pose_init=st.starts, with_pose_opt_plus=True)
    pose, _, _, plus = solver(x3d, st.x2d, st.w2d, st.camera, st.cost_fun, pose_init=st.starts)
    assert plus is None and not pose.requires_grad
    # fast mode without a Gauss-Newton step has no covariance, cost or cost_init
    p0 = params(dof, "fast", lm_iter=0)
    for want in ("want_cov", "want_cost", "want_cost_init"):
        with pytest.raises(native.NativeError):
            native.lm_solve_stacked(st.prob, st.starts, p0, **{want: True})
    with pytest.raises(native.NativeError):
        LMSolver(dof=dof, num_iter=0).solve(*st.args(), pose_init=st.starts, with_cost=True, fast_mode=True)
    got = native.lm_solve_stacked(st.prob, st.starts, p0, want_plus=True)
    assert same(got["pose_opt"], st.starts)
    for s in range(2):
        assert same(got["pose_opt_plus"][s], native.lm_solve(st.prob, st.starts[s], p0, want_plus=True)["pose_opt_plus"])


def check_compile(dev, dof=4, N=24, B=3):
    """torch.compile(fullgraph=True, dynamic=True) traces the stacked solve with no graph break, to eager's bits."""
    import torch._dynamo
    st = Setup(dev, dof, N, 3, B, "scalar", seed=6)
    solver = LMSolver(dof=dof, num_iter=5)

    def fn(x3d, x2d, w2d, cam, starts):
        camera = PerspectiveCamera(cam_mats=cam, z_min=0.1, lb=-100.0, ub=800.0)
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d, w2d)
        return solver(x3d, x2d, w2d, camera, cost_fun, pose_init=starts, with_pose_cov=True, with_cost=True,
                      with_pose_opt_plus=True, fast_mode=True)

    args = (st.x3d, st.x2d, st.w2d, st.cam, st.starts)
    torch._dynamo.reset()
    explained = torch._dynamo.explain(fn)(*args)
    assert explained.graph_break_count == 0, explained.break_reasons
    eager = fn(*args)
    compiled = torch.compile(fn, backend="aot_eager", fullgraph=True, dynamic=True)(*args)
    torch._dynamo.reset()
    for a, b in zip(eager, compiled):
        assert same(a, b)


def opcheck_args(dev, dof=6, N=24, B=2, S=3, grad=True):
    st = Setup(dev, dof, N, S, B, "tensor", seed=7)
    leaf = lambda v: v.clone().requires_grad_(grad)
    ints, floats = ops.param_lists(None, dof, lm_iter=4, z_min=0.1)
    prob = (leaf(st.x3d), leaf(st.x2d), leaf(st.w2d), leaf(st.cam), leaf(st.lb), leaf(st.ub),
            leaf(st.cost_fun.delta))
    return prob + (st.starts, ints, floats, True, True, True)


def check_opcheck(dev):
    for grad in (True, False):
        torch.library.opcheck(ops.lm_solve_stacked.op, opcheck_args(dev, grad=grad))
    out = ops.lm_solve_stacked(*opcheck_args(dev))
    assert not any(t.requires_grad for t in out)


@pytest.mark.parametrize("c", CASES, ids=[c["id"] for c in CASES])
def test_stacked_equals_per_start_and_flattened(cuda_device, c):
    check_case(cuda_device, c)


@pytest.mark.parametrize("dof,mode", [(6, "lm"), (4, "fast")])
def test_solver_leading_dimensions(cuda_device, dof, mode):
    check_solver_leading_dims(cuda_device, dof=dof, N=300, B=700, mode=mode)


def test_empty_stacks(cuda_device):
    check_empty(cuda_device)


def test_refusals(cuda_device):
    check_refusals(cuda_device)


def test_compile_no_graph_break(cuda_device):
    check_compile(cuda_device)


def test_opcheck(cuda_device):
    check_opcheck(cuda_device)


def test_graph_replay_equals_eager(cuda_device):
    """The stacked solve captured into a CUDA graph and replayed on new inputs gives the eager call's bits."""
    dev = cuda_device
    a, b = Setup(dev, 6, 300, 8, 512, "tensor", seed=8), Setup(dev, 6, 300, 8, 512, "tensor", seed=9)
    solver = LMSolver(dof=6, num_iter=10)
    static = [v.clone() for v in (a.x3d, a.x2d, a.w2d, a.cam, a.lb, a.ub, a.starts)]

    def run():
        x3d, x2d, w2d, cam, lb, ub, starts = static
        camera = PerspectiveCamera(cam_mats=cam, z_min=0.1, lb=lb, ub=ub)
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d, w2d)
        return solver(x3d, x2d, w2d, camera, cost_fun, pose_init=starts, with_pose_cov=True, with_cost=True,
                      with_pose_opt_plus=True)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = run()
    for src in (b, a):
        for dst, v in zip(static, (src.x3d, src.x2d, src.w2d, src.cam, src.lb, src.ub, src.starts)):
            dst.copy_(v)
        graph.replay()
        torch.cuda.synchronize()
        want = solver(*src.args(), pose_init=src.starts, with_pose_cov=True, with_cost=True, with_pose_opt_plus=True)
        for g, w in zip(outs, want):
            assert same(g, w)
