"""The forward matrix of test_lm_matrix_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulator (tests/simt_native.py),
held to the same per-object float64 bounds, at sizes the emulator affords.  The three forms of lm_warp_kernel stay: N = 7
(staged, plain loader), 640 (staged), 641 (one warp from global memory) and 2049 (eight warps).  Also the refusal of a
fast-mode solve without a Gauss-Newton step, through the C ABI, native, LMSolver and EProPnP6DoF."""
import pytest
import torch

import simt_native
import test_lm_matrix_gpu as _lm
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

_c = _lm._c
S_LIST = (1, 129)


@pytest.fixture
def cuda_device(monkeypatch):
    return simt_native.install(monkeypatch)


CASES = [
    _c(6, 7, 3, "lm", outliers=0.2, mixed=True),
    _c(4, 7, 2, "fast"),
    _c(6, 640, 2, "fast", bounds="tensor"),
    _c(4, 640, 2, "lm", outliers=0.1),
    _c(6, 641, 2, "lm", zmin=True),
    _c(4, 641, 2, "fast", bounds="scalar", outliers=0.1),
    _c(6, 2049, 2, "lm", outliers=0.1, mixed=True),
    _c(4, 2049, 2, "fast"),
]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_lm_matrix(cuda_device, case):
    _lm.run_case(case, cuda_device, S_LIST, record="simt/lm_matrix")


def test_lm_exact_properties(cuda_device):
    _lm.check_exact_properties(cuda_device, 640, B=3)


def _problem(B=3, N=64, dof=6):
    pc = make_problem(B, N, seed=1, dof=dof)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
    return pc, native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta)


@pytest.mark.parametrize("want", ["cov", "cost", "cost_init"])
def test_fast_mode_without_steps_refuses_what_it_cannot_compute(cuda_device, want):
    pc, prob = _problem()
    p = native.default_params(6, lm_iter=0, fast_mode=1)
    with pytest.raises(native.NativeError):
        native.lm_solve(prob, pc["pose_init"], p, **{f"want_{want}": True})


def test_fast_mode_without_steps_returns_pose_init_and_the_gn_step(cuda_device):
    """pose_opt alone is pose_init; pose_opt_plus is pose_init (+) gn_step, as in LM mode with lm_iter = 0."""
    pc, prob = _problem(N=641)
    fast = native.lm_solve(prob, pc["pose_init"], native.default_params(6, lm_iter=0, fast_mode=1), want_plus=True)
    lm = native.lm_solve(prob, pc["pose_init"], native.default_params(6, lm_iter=0), want_plus=True)
    assert torch.equal(fast["pose_opt"], pc["pose_init"])
    assert torch.equal(fast["pose_opt_plus"], lm["pose_opt_plus"])


def test_fast_mode_without_steps_refused_through_the_layers(cuda_device):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    pc, _ = _problem(B=2, N=32)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"], z_min=0.1)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    solver = LMSolver(dof=6, num_iter=0)
    args = (pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun)
    pose, _, _ = solver.solve(*args, pose_init=pc["pose_init"], fast_mode=True)
    assert torch.equal(pose, pc["pose_init"])
    with pytest.raises(native.NativeError):
        solver.solve(*args, pose_init=pc["pose_init"], with_pose_cov=True, fast_mode=True)
    layer = EProPnP6DoF(mc_samples=16, num_iter=4, solver=solver)
    with pytest.raises(native.NativeError):
        layer.monte_carlo_forward(*args, pose_init=pc["pose_init"], force_init_solve=False, fast_mode=True)
