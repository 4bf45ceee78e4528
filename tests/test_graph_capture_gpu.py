"""CUDA-graph capture of the layer's flows on a real GPU.  Each flow is captured after a side-stream warm-up, replayed
with new inputs and seeds written into its static buffers, and must give what an eager call on those inputs, with the
same seeds as ints, gives -- bit for bit, outputs and gradients.  (The graph runs the seed-pointer kernels, the eager
call the by-value ones.)  Without given seeds, the graph draws its own on the device: two replays on the same inputs
sample differently."""
import pytest
import torch

from epropnp import common
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.epnp import EPnPSolver
from epropnp.epropnp import EProPnP4DoF, EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
from epropnp.monte_carlo_pose_loss import MonteCarloPoseLoss
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu


class _SeededRSLM(RSLMSolver):
    """RSLMSolver whose draws take `self.seed` (None: the solver draws its own), so a test can give the random-sample
    init of monte_carlo_forward the same seed in the graph and in the eager call."""
    seed = None

    def solve(self, *args, **kwargs):
        return super().solve(*args, rslm_seed=self.seed, **kwargs)


def _inputs(dev, B, N, dof, seed):
    pc = make_problem(B, N, seed=seed, dof=dof)
    return {k: pc[k].to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats", "pose_gt")}


def _capture(run, static, seeds):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            run(static, seeds)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = run(static, seeds)
    return g, out


def _check_replays_match_eager(dev, run, B, N, dof, seed_names, trials=2):
    static = _inputs(dev, B, N, dof, seed=100)
    seeds = {k: torch.zeros(1, dtype=torch.int64, device=dev) for k in seed_names}
    g, out = _capture(run, static, seeds)
    for t in range(trials):
        new = _inputs(dev, B, N, dof, seed=200 + t)
        values = {k: 0x0123_4567_89AB_CDEF + 7919 * t + i for i, k in enumerate(seed_names)}
        with torch.no_grad():
            for k, v in new.items():
                static[k].copy_(v)
        for k, v in values.items():
            seeds[k].fill_(v)
        g.replay()
        got = {k: v.clone() for k, v in out.items() if v is not None}
        want = run(new, values)
        torch.cuda.synchronize()
        for k, v in got.items():
            assert torch.equal(v, want[k]), f"trial {t}: {k}"
    return g, out, static


def _mc_forward(dof, init, force_init_solve, M=128, I=4, P=16):
    """monte_carlo_forward (no grad) with pose_init = pose_gt (init 'gt'), or with the RSLM init ('rslm')."""
    rslm = _SeededRSLM(dof=dof, num_points=8, num_proposals=P, num_iter=3)
    layer = (EProPnP6DoF if dof == 6 else EProPnP4DoF)(mc_samples=M, num_iter=I,
                                                       solver=LMSolver(dof=dof, num_iter=5, init_solver=rslm))

    def run(inp, seeds):
        rslm.seed = seeds.get("rslm")
        camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(inp["x2d"], inp["w2d"])
        pose_init = inp["pose_gt"] if init == "gt" else None
        r = layer.monte_carlo_forward(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun, pose_init=pose_init,
                                      force_init_solve=force_init_solve, with_cost=True, with_pose_opt_plus=True,
                                      amis_seed=seeds.get("amis"))
        return dict(zip(("pose_opt", "cost", "plus", "samples", "logw", "cost_init"), r))
    return run


@pytest.mark.parametrize("dof,init,force", [(6, "rslm", True), (4, "rslm", True), (6, "gt", True), (6, "gt", False),
                                            (4, "gt", False)])
def test_monte_carlo_forward_replays_match_eager(cuda_device, dof, init, force):
    seeds = ("amis", "rslm") if (init == "rslm" or force) else ("amis",)
    _check_replays_match_eager(cuda_device, _mc_forward(dof, init, force), 8, 96, dof, seeds)


def test_lmsolver_forward_with_epnp_init_replays_match_eager(cuda_device):
    solver = LMSolver(dof=6, num_iter=5, init_solver=EPnPSolver(conf_quantile=0.8))

    def run(inp, seeds):
        camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(inp["x2d"], inp["w2d"])
        pose, cov, cost, plus = solver(inp["x3d"], inp["x2d"], inp["w2d"], camera, cost_fun, with_pose_opt_plus=True,
                                       with_pose_cov=True, with_cost=True)
        return dict(pose=pose, cov=cov, cost=cost, plus=plus)
    _check_replays_match_eager(cuda_device, run, 8, 96, 6, ())


def _train_step(dof, N, force_init_solve, M=128, I=4, P=4):
    """The reference's training step (EPro-PnP-6DoF/lib/train.py): adaptive delta from the weights, monte_carlo_forward
    with the ground-truth pose as pose_init, the Monte-Carlo pose loss plus a loss on pose_opt_plus, backward."""
    rslm = _SeededRSLM(dof=dof, num_points=16, num_proposals=P, num_iter=3)
    layer = EProPnP6DoF(mc_samples=M, num_iter=I, solver=LMSolver(dof=dof, num_iter=5, init_solver=rslm))
    loss_fn = MonteCarloPoseLoss().to("cuda")

    def run(inp, seeds):
        rslm.seed = seeds.get("rslm")
        if inp.get("_leaves") is None:           # static inputs keep their leaves across replays
            inp["_leaves"] = tuple(inp[k].detach().requires_grad_(True) for k in ("x3d", "x2d", "w2d"))
        x3d, x2d, w2d = inp["_leaves"]
        for t in (x3d, x2d, w2d):
            t.grad = None
        loss_fn.norm_factor.fill_(1.0)
        camera = PerspectiveCamera(cam_mats=inp["cam_mats"])
        cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
        cost_fun.set_param(x2d.detach(), w2d)
        pose_opt, _, plus, _, logw, cost_tgt = layer.monte_carlo_forward(
            x3d, x2d, w2d, camera, cost_fun, pose_init=inp["pose_gt"], force_init_solve=force_init_solve,
            with_pose_opt_plus=True, amis_seed=seeds.get("amis"))
        loss = loss_fn(logw, cost_tgt, 1.0) + 0.1 * (plus - inp["pose_gt"]).abs().sum()
        loss.backward()
        return dict(loss=loss.detach(), pose_opt=pose_opt, gx3d=x3d.grad, gx2d=x2d.grad, gw2d=w2d.grad,
                    norm_factor=loss_fn.norm_factor)
    return run


def test_training_step_replays_match_eager(cuda_device):
    """B = 8, N = 96, RSLM init with force_init_solve (as the reference trains), pose_opt_plus and the backward."""
    _check_replays_match_eager(cuda_device, _train_step(6, 96, True), 8, 96, 6, ("amis", "rslm"))


def test_split_path_replays_match_eager(cuda_device):
    """N = 16 384 (a 128 x 128 coordinate map): the cluster-split AMIS, cost, GN-plus backward kernels under capture.
    RSLM init refuses this size, so pose_init is used as it is (force_init_solve=False)."""
    N = 16384
    assert N > native.max_points(6, 128, 4)
    _check_replays_match_eager(cuda_device, _train_step(6, N, False), 2, N, 6, ("amis",))
    _check_replays_match_eager(cuda_device, _mc_forward(6, "gt", False), 2, N, 6, ("amis",))


def test_in_graph_seeds_draw_new_samples_at_every_replay(cuda_device):
    dev = cuda_device
    static = _inputs(dev, 8, 96, 6, seed=5)
    g, out = _capture(_mc_forward(6, "rslm", True), static, {})
    g.replay()
    first = {k: v.clone() for k, v in out.items() if v is not None}
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(first["samples"], out["samples"]) and not torch.equal(first["logw"], out["logw"])
    assert torch.isfinite(out["logw"]).all()

    # the RSLM subsets and start poses themselves, seed drawn inside the graph
    def draw(inp, seeds):
        seed = common.philox_seed(None, dev)
        inds, start = native.rslm_draw(inp["x3d"], inp["x2d"], inp["w2d"], inp["cam_mats"], 32, 8, 6, seed=seed)
        return dict(inds=inds, start=start)
    g, out = _capture(draw, static, {})
    g.replay()
    first = {k: v.clone() for k, v in out.items()}
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(first["inds"], out["inds"]) and not torch.equal(first["start"], out["start"])


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")      # the refusal comes before anything is captured
def test_torch_draws_are_refused_under_capture(cuda_device):
    static = _inputs(cuda_device, 4, 64, 4, seed=3)
    solver = RSLMSolver(dof=4, num_points=8, num_proposals=8, draws='torch')
    camera = PerspectiveCamera(cam_mats=static["cam_mats"])
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(static["x2d"], static["w2d"])
    solver.solve(static["x3d"], static["x2d"], static["w2d"], camera, cost_fun)        # eager: as always
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="cannot be captured into a CUDA graph"):
        with torch.cuda.graph(g):
            solver.solve(static["x3d"], static["x2d"], static["w2d"], camera, cost_fun)
