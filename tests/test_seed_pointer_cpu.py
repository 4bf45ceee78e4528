"""The seed-pointer entry points (epnp_lm_amis_fused_seedptr_f32, epnp_lm_amis_fused_split_seedptr_f32,
epnp_rslm_draw_seedptr_f32), which read the Philox seed from device memory so that a captured CUDA graph draws anew at
every replay, on the CPU: pnp_kernels.cu under the SIMT emulators (single CTA and cluster).  Given the same seed value,
each gives the by-value call's outputs bit for bit.  And the host logic: while a graph is being captured the layer draws
its seed on the device and takes the tensor-seed calls; eager calls keep the int seed from torch's CPU generator."""
import ctypes

import pytest
import torch

import simt_cluster_native
import simt_native
from epropnp import common
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import AdaptiveHuberPnPCost
from epropnp.epropnp import EProPnP6DoF
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver
from epropnp_b200 import capi, native
from epropnp_b200.synth import make_problem

SEED = 0x1234_5678_9ABC_DEF            # both halves of the Philox key in use


def _seed_tensor(dev, value=SEED):
    return torch.tensor([value], dtype=torch.int64, device=dev)


def _fused_pair(dev, fn, dof, B, N, M, I, **kw):
    pc = make_problem(B, N, seed=N + dof, dof=dof)
    pc = {k: v.to(dev) for k, v in pc.items()}
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None,
                          native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5))
    p = native.default_params(dof, lm_iter=3, mc_samples=M, mc_iter=I)
    args = dict(want_cost=True, want_plus=True, want_proposals=True, **kw)
    by_value = fn(prob, pc["pose_init"], p, seed=SEED, obj_offset=5, **args)
    by_ptr = fn(prob, pc["pose_init"], p, seed=_seed_tensor(dev), obj_offset=5, **args)
    other = fn(prob, pc["pose_init"], p, seed=_seed_tensor(dev, SEED + 1), obj_offset=5, **args)
    return by_value, by_ptr, other


def _assert_same(a, b):
    for k, v in a.items():
        if v is not None:
            assert torch.equal(v, b[k]), k


@pytest.mark.parametrize("dof,N", [(6, 40), (4, 40), (6, 2048)])      # 128-thread resident; N = 2048: the dense kernel
def test_fused_seed_pointer_matches_by_value(monkeypatch, dof, N):
    dev = simt_native.install(monkeypatch)
    B = 1 if N >= 2048 else 3
    by_value, by_ptr, other = _fused_pair(dev, native.lm_amis_fused, dof, B, N, 16, 2)
    _assert_same(by_value, by_ptr)
    assert not torch.equal(by_value["pose_samples"], other["pose_samples"])      # the kernel did read the pointer


@pytest.mark.parametrize("dof,N,ctas", [(6, 50, 3), (4, 37, 2)])
def test_split_seed_pointer_matches_by_value(monkeypatch, dof, N, ctas):
    dev = simt_cluster_native.install(monkeypatch)
    by_value, by_ptr, other = _fused_pair(dev, native.lm_amis_fused_split, dof, 2, N, 16, 2, cluster_ctas=ctas)
    _assert_same(by_value, by_ptr)
    assert not torch.equal(by_value["pose_samples"], other["pose_samples"])


@pytest.mark.parametrize("dof", [6, 4])
def test_rslm_draw_seed_pointer_matches_by_value(monkeypatch, dof):
    dev = simt_native.install(monkeypatch)
    pc = make_problem(3, 45, seed=3, dof=dof)
    args = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], 24, 6, dof)
    a = native.rslm_draw(*args, seed=SEED, obj_offset=2, want_t=True)
    b = native.rslm_draw(*args, seed=_seed_tensor(dev), obj_offset=2, want_t=True)
    c = native.rslm_draw(*args, seed=_seed_tensor(dev, SEED + 1), obj_offset=2, want_t=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[0], c[0])


def test_null_seed_pointer_and_bad_seed_tensors_are_refused(monkeypatch):
    dev = simt_native.install(monkeypatch)
    lib = simt_native.handle()
    w = torch.ones(1, 8, 2)
    out_i, out_s = torch.empty(1, 1, 4, dtype=torch.int32), torch.empty(1, 1, 7)
    seed = _seed_tensor(dev)
    for seed_ptr, want in ((None, -1), (ctypes.c_void_p(seed.data_ptr()), 0)):
        rc = lib.epnp_rslm_draw_seedptr_f32(None, None, capi.ptr(w), None, capi.ptr(torch.zeros(1, 3)), seed_ptr, 0,
                                            capi.iptr(out_i), capi.ptr(out_s), None, 1, 4, 1, 8, 6, ctypes.c_float(1e-5),
                                            None)
        assert rc == want
    p = native.default_params(6, mc_samples=16, mc_iter=2)
    for name in ("epnp_lm_amis_fused_seedptr_f32", "epnp_lm_amis_fused_split_seedptr_f32"):
        tail = ([0] if "split" in name else []) + [None]
        x = torch.zeros(1, 8, 3)
        rc = getattr(lib, name)(*[capi.ptr(x)] * 4, None, None, capi.ptr(torch.ones(1)), capi.ptr(torch.zeros(1, 7)),
                                None, None, None, None, 0, *[capi.ptr(torch.zeros(1, 16 * 7))] * 8, 1, 8,
                                ctypes.byref(p), *tail)
        assert rc == -1, name
    pc = make_problem(1, 16, seed=1)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, 1.0)
    for bad in (torch.tensor([1], dtype=torch.int32), torch.tensor([1, 2]), torch.tensor(1.0)):
        with pytest.raises(ValueError, match="seed tensor"):
            native.lm_amis_fused(prob, pc["pose_init"], p, seed=bad)


def test_philox_seed_eager_and_capturing(monkeypatch):
    torch.manual_seed(7)
    want = int(torch.randint(0, 2 ** 62, (1,)).item())
    torch.manual_seed(7)
    assert common.philox_seed(None, torch.device("cpu")) == want           # eager: today's draw from the CPU generator
    assert common.philox_seed(5, torch.device("cpu")) == 5
    assert common.philox_seed(torch.tensor(9), torch.device("cpu")) == 9   # a CPU tensor is a number, as before
    _pretend_capturing(monkeypatch, True)
    s = common.philox_seed(None, torch.device("cpu"))
    assert torch.is_tensor(s) and s.dtype == torch.int64 and s.shape == (1,) and 0 <= int(s) < 2 ** 62
    assert common.philox_seed(11, torch.device("cpu")) == 11                 # a given seed is kept under capture too


def _pretend_capturing(monkeypatch, capturing):
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: capturing)


def _record_calls(monkeypatch):
    """Names of the C-ABI calls the layer makes, through the emulated library."""
    calls = []
    real = capi._lib

    class Spy:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(real, name)
    monkeypatch.setattr(capi, "_lib", Spy())
    return calls


@pytest.mark.parametrize("capturing", [False, True])
def test_layer_takes_the_seed_pointer_calls_only_under_capture(monkeypatch, capturing):
    dev = simt_native.install(monkeypatch)
    calls = _record_calls(monkeypatch)
    _pretend_capturing(monkeypatch, capturing)
    pc = make_problem(2, 24, seed=4)
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"])
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    solver = LMSolver(dof=6, num_iter=3, init_solver=RSLMSolver(dof=6, num_points=8, num_proposals=4, num_iter=2))
    layer = EProPnP6DoF(mc_samples=16, num_iter=2, solver=solver)
    layer.monte_carlo_forward(pc["x3d"], pc["x2d"], pc["w2d"], camera, cost_fun, pose_init=pc["pose_init"],
                              force_init_solve=True)
    seedptr = {"epnp_rslm_draw_seedptr_f32", "epnp_lm_amis_fused_seedptr_f32"}
    by_value = {"epnp_rslm_draw_f32", "epnp_lm_amis_fused_f32"}
    assert (seedptr if capturing else by_value) <= set(calls)
    assert not (by_value if capturing else seedptr) & set(calls)


def test_torch_draws_are_refused_under_capture(monkeypatch):
    simt_native.install(monkeypatch)
    _pretend_capturing(monkeypatch, True)
    pc = make_problem(2, 24, seed=4, dof=4)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)
    cost_fun.set_param(pc["x2d"], pc["w2d"])
    solver = RSLMSolver(dof=4, num_points=8, num_proposals=4, draws='torch')
    with pytest.raises(RuntimeError, match="cannot be captured into a CUDA graph"):
        solver.solve(pc["x3d"], pc["x2d"], pc["w2d"], PerspectiveCamera(cam_mats=pc["cam_mats"]), cost_fun)
