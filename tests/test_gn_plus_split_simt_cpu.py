"""The cluster-split backward of pose_opt_plus (epnp_gn_plus_backward_split_f32) on the CPU: pnp_kernels.cu under the
cluster SIMT emulator (tests/simt_cluster_native.py).  The golden cases of test_gn_plus_backward_cpu with forced cluster
sizes against the float64 composite and against the resident kernel; synthetic point sets with a short last rank, an
odd count and empty ranks; the audit build (-DEPNP_SPLIT_AUDIT) checks that every rank ends with rank 0's normal
equations, step and v, that each rank stores the gradient rows of its own points only and that rank 0 alone stores
grad_delta; results do not depend on the fiber schedule; the argument checks and refusals."""
import ctypes
import functools
import itertools

import numpy as np
import pytest
import torch

import simt_cluster_native
import simt_native
import test_gn_plus_split_gpu as _gs
from conftest import err_vs
from test_gn_plus_backward_cpu import _case
from epropnp import autograd as ag
from epropnp.levenberg_marquardt import LMSolver
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

AUDIT = ("-DEPNP_SPLIT_AUDIT",)
GOLDEN = ["lm6_basic", "lm6_bounds", "lm6_scalar_bounds_fixed_delta", "lm4_basic", "mc6_basic", "mc4_basic"]


def _golden_grads(name, dev, monkeypatch, mode, ctas=0):
    """dL/d(x3d, x2d, w2d[, delta]) of L = <coef, pose_opt_plus> on golden case `name`: mode "composite64" /
    "composite32" (torch autograd through the composite), "resident" or "split" (the native kernels, fp32)."""
    dtype = torch.float64 if mode == "composite64" else torch.float32
    g, x3d, x2d, w2d, camera, cost_fun, pose = _case(name, dev, dtype)
    solver = LMSolver(dof=int(g["dof"]), num_iter=int(g["lm_iter"]))
    coef = torch.from_numpy(np.random.RandomState(3).randn(*pose.shape)).to(device=dev, dtype=dtype)
    leaves = [x3d, x2d, w2d] + ([cost_fun.delta] if torch.is_tensor(cost_fun.delta) else [])
    if mode.startswith("composite"):
        monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "0")
        (ag.pose_plus_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun) * coef).sum().backward()
        return [l.grad.detach() for l in leaves]
    p = solver.native_params(camera, cost_fun, False)
    prob = native.Problem(x3d, x2d, w2d, camera.cam_mats, camera.lb, camera.ub, cost_fun.delta)
    fn = native.gn_plus_backward if mode == "resident" else functools.partial(native.gn_plus_backward_split,
                                                                              cluster_ctas=ctas)
    return list(fn(prob, pose, coef, p.dof, p.z_min, p.eps, p.huber_eps)[:len(leaves)])


@pytest.mark.parametrize("name", GOLDEN)
def test_split_matches_composite_and_resident(monkeypatch, name):
    dev = simt_cluster_native.install(monkeypatch)
    c64 = _golden_grads(name, dev, monkeypatch, "composite64")
    c32 = _golden_grads(name, dev, monkeypatch, "composite32")
    res = _golden_grads(name, dev, monkeypatch, "resident")
    for ctas in (2, 3, 5):
        split = _golden_grads(name, dev, monkeypatch, "split", ctas)
        for gs, gr, g64, g32, what in zip(split, res, c64, c32, ("x3d", "x2d", "w2d", "delta")):
            assert torch.isfinite(gs).all(), (ctas, what)
            assert err_vs(gs.numpy(), g64.numpy()) < 1e-4, (ctas, what)
            floor = err_vs(g32.numpy(), g64.numpy())
            assert err_vs(gs.numpy(), gr.numpy()) < max(1e-5, 3 * floor), (ctas, what, floor)


def _synthetic(dof, N, B=2, seed=21, bounds=False):
    pc = make_problem(B, N, seed=seed, dof=dof, outlier_frac=0.2)     # outliers: grad_delta is more than rounding noise
    lb = ub = None
    if bounds:      # bounds that bind for some points, so the clipped branch runs
        lb, ub = pc["x2d"].amin(1) + 20.0, pc["x2d"].amax(1) - 20.0
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub,
                          native.adaptive_delta(pc["x2d"], pc["w2d"], 0.1))
    gp = torch.randn(B, 7 if dof == 6 else 4, generator=torch.Generator().manual_seed(seed))
    return prob, pc["pose_init"], gp


def _split(prob, pose, gp, dof, ctas, want=(True, True, True, True)):
    return native.gn_plus_backward_split(prob, pose, gp, dof, 0.1, 1e-5, 1e-10, want=want, cluster_ctas=ctas)


# N = 50 on 3 CTAs -> 24 + 24 + 2 points; 37 on 5 -> 8 x 4 + 5 (odd, padded); 48 on 5 -> 16 x 3 + two empty ranks
# (and the TMA loader, N % 4 == 0)
RANGES = [(6, 50, 3), (6, 37, 5), (6, 48, 5), (4, 37, 5), (4, 50, 3)]


@pytest.mark.parametrize("dof,N,ctas", RANGES)
def test_awkward_ranges_against_composite_and_resident(monkeypatch, dof, N, ctas):
    simt_cluster_native.install(monkeypatch)
    prob, pose, gp = _synthetic(dof, N, bounds=N == 50)
    split = _split(prob, pose, gp, dof, ctas)
    res = native.gn_plus_backward(prob, pose, gp, dof, 0.1, 1e-5, 1e-10)
    args = (prob.x3d, prob.x2d, prob.w2d, prob.cam, prob.lb, prob.ub, prob.delta, pose, gp, dof, 0.1)
    c64, c32 = _gs.composite_grads(*args, torch.float64), _gs.composite_grads(*args, torch.float32)
    for gs, gr, g64, g32, what in zip(split, res, c64, c32, ("x3d", "x2d", "w2d", "delta")):
        assert torch.isfinite(gs).all() and gs.abs().sum() > 0, what
        # (the bound against the resident kernel is the fp64 one here: with two objects, one whose delta gradient nearly
        # cancels, grad_delta carries rounding noise of about 1e-4 of the other's in either kernel)
        bound = max(1e-4, _gs.K_FLOOR * err_vs(g32.numpy(), g64.numpy()))
        assert err_vs(gs.numpy(), g64.numpy()) < bound, what
        assert err_vs(gs.numpy(), gr.numpy()) < bound, what


def _points_of_rank(N, ctas):
    share = ((N + ctas - 1) // ctas + 7) // 8 * 8
    return [max(0, min(N, (r + 1) * share) - min(N, r * share)) for r in range(8)]


@pytest.mark.parametrize("dof,N,ctas", [(6, 50, 3), (6, 48, 5), (4, 37, 5)])
def test_ranks_agree_and_write_only_their_rows(monkeypatch, dof, N, ctas):
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    B = 2
    prob, pose, gp = _synthetic(dof, N, B)
    full = _split(prob, pose, gp, dof, ctas)
    counts = (ctypes.c_longlong * 16)()
    pts = _points_of_rank(N, ctas)
    for want in itertools.product((False, True), repeat=4):
        lib.simt_audit_reset()
        out = _split(prob, pose, gp, dof, ctas, want=want)
        lib.simt_audit_read(counts)
        stores, mismatches = list(counts)[:8], list(counts)[8:]
        assert mismatches == [0] * 8, want                      # H, g, cost, step, v: rank 0's bits on every rank
        per_point = 3 * want[0] + 2 * want[1] + 2 * want[2]
        expect = [B * pts[r] * per_point + (B * want[3] if r == 0 else 0) for r in range(8)]
        assert stores == expect, (want, stores, expect)
        for o, f, w in zip(out, full, want):                    # the outputs asked for, the same bits as all four
            assert (o is None) == (not w) and (o is None or torch.equal(o, f))


def test_split_results_do_not_depend_on_fiber_schedule(monkeypatch):
    """Ascending, descending and random fiber orders across the whole cluster give the same bits: no rank reads another
    rank's partials without the cluster barrier in between."""
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    prob, pose, gp = _synthetic(6, 50, bounds=True)
    try:
        lib.simt_set_schedule(0, 1)
        base = _split(prob, pose, gp, 6, 3)
        for mode, seed in ((1, 1), (2, 5)):
            lib.simt_set_schedule(mode, seed)
            lib.simt_audit_reset()
            out = _split(prob, pose, gp, 6, 3)
            counts = (ctypes.c_longlong * 16)()
            lib.simt_audit_read(counts)
            assert list(counts)[8:] == [0] * 8
            for a, b in zip(out, base):
                assert torch.equal(a, b), mode
    finally:
        lib.simt_set_schedule(0, 1)


def test_arguments_and_refusals(monkeypatch):
    """A cluster size outside [minimum, 8] is a bad argument; a device that cannot co-schedule the cluster is refused
    before any launch; B = 0 launches nothing."""
    simt_cluster_native.install(monkeypatch)
    lib = simt_cluster_native.handle()
    prob, pose, gp = _synthetic(6, 40)
    for bad in (1, 9, -1):
        with pytest.raises(native.NativeError, match="bad argument"):
            _split(prob, pose, gp, 6, bad)

    def raw(B, ctas):      # pointers that would fault if anything read them: B = 0 must return before any launch
        one = ctypes.c_void_p(16)
        return lib.epnp_gn_plus_backward_split_f32(one, one, one, one, None, None, one, one, one, one, one, one, one,
                                                   B, 40, 6, ctypes.c_float(0.1), ctypes.c_float(1e-5),
                                                   ctypes.c_float(1e-10), ctas, None)
    assert raw(0, 0) == 0 and raw(0, 9) == -1
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "0")
    with pytest.raises(native.NativeError, match="not supported"):
        _split(prob, pose, gp, 6, 0)
    assert raw(0, 0) == 0


def test_single_cta_emulator_refuses_split_call(monkeypatch):
    """The single-CTA emulator build cannot run a cluster: the split call reports EPNP_ERR_UNSUPPORTED after its argument
    checks, as a device without cluster support does."""
    simt_native.install(monkeypatch)
    prob, pose, gp = _synthetic(6, 40)
    with pytest.raises(native.NativeError, match="not supported"):
        _split(prob, pose, gp, 6, 0)
    with pytest.raises(native.NativeError, match="bad argument"):
        _split(prob, pose, gp, 6, 9)


def test_autograd_takes_the_split_call_above_the_resident_limit(monkeypatch):
    """_PosePlus.backward routes through autograd.gn_plus_backward: with the resident limit lowered below N it takes the
    split call (automatic cluster size), and the gradients stay within the composite's bound."""
    dev = simt_cluster_native.install(monkeypatch)
    calls = []
    split = native.gn_plus_backward_split
    monkeypatch.setattr(native, "gn_plus_backward_split", lambda *a, **k: calls.append(1) or split(*a, **k))
    monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i: 0)
    c64 = _golden_grads("mc6_basic", dev, monkeypatch, "composite64")
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    g, x3d, x2d, w2d, camera, cost_fun, pose = _case("mc6_basic", dev, torch.float32)
    solver = LMSolver(dof=6, num_iter=int(g["lm_iter"]))
    coef = torch.from_numpy(np.random.RandomState(3).randn(*pose.shape)).to(torch.float32)
    (ag.pose_plus_autograd(solver, x3d, x2d, w2d, pose, camera, cost_fun) * coef).sum().backward()
    assert calls == [1]
    for gn, gc in zip((x3d.grad, x2d.grad, w2d.grad, cost_fun.delta.grad), c64):
        assert err_vs(gn.numpy(), gc.numpy()) < 1e-4
