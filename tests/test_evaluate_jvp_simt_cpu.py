"""The Jacobian-vector-product kernels (epnp_evaluate_jvp_f32) on the CPU: pnp_kernels.cu under the SIMT emulator, held
to the oracle's float64 forward-mode derivative with the bound of test_evaluate_jvp_gpu.py (whose helpers this file
uses), at small sizes, and tied to epnp_evaluate_backward_f32 by the adjoint identity."""
import pytest
import torch

import simt_native
import test_cost_hvp_gpu as hv
import test_evaluate_jvp_gpu as jv

CPU = torch.device("cpu")


@pytest.mark.parametrize("dof,N,S,B,bounds,zmin,clip", [(6, 7, 1, 2, False, False, True),
                                                        (6, 33, 70, 2, True, True, True),
                                                        (4, 129, 2, 3, True, False, True),
                                                        (4, 20, 3, 2, False, True, False),
                                                        (6, 5, 1, 3, False, True, False)])
def test_kernels_against_float64(monkeypatch, dof, N, S, B, bounds, zmin, clip):
    simt_native.install(monkeypatch)
    c = jv.build_case(dof, N, S, B, CPU, bounds=bounds, zmin=zmin, clip=clip)
    assert jv.huber_margin(c) > hv.HUBER_GAP
    got = jv.run_jvp(c)
    jv.assert_close(got, c, (dof, N, S, B))
    assert jv.adjoint_gap(c) < jv.ADJ_TOL
    # the outputs are linear in v: each tangent part alone sums to the whole
    parts = [jv.run_jvp(c, t={k: v}) for k, v in c["t"].items()]
    for out in jv.OUTPUTS:
        total = sum(p[out].double() for p in parts)
        assert torch.allclose(total, got[out].double(), rtol=1e-4, atol=1e-5 * float(got[out].abs().max())), out


def test_only_the_asked_outputs_are_written(monkeypatch):
    simt_native.install(monkeypatch)
    c = jv.build_case(6, 16, 3, 2, CPU, bounds=True)
    full = jv.run_jvp(c)
    for i, k in enumerate(jv.OUTPUTS):
        one = jv.run_jvp(c, want=[j == i for j in range(3)])
        assert all(one[o] is None for o in jv.OUTPUTS if o != k)
        assert torch.equal(one[k], full[k]), k


def test_pose_major_cost_matches_point_major(monkeypatch):
    """d cost alone at 64 poses and more runs pose-major; with the residual asked for too, point-major."""
    simt_native.install(monkeypatch)
    c = jv.build_case(6, 150, 64, 2, CPU, bounds=True)
    alone = jv.run_jvp(c, want=(False, False, True))["cost"]
    with_r = jv.run_jvp(c, want=(True, False, True))["cost"]
    assert torch.allclose(alone, with_r, rtol=1e-4, atol=1e-5 * float(with_r.abs().max()))


@pytest.mark.parametrize("mode", ["fwad", "jvp", "linearize"])
def test_forward_mode_through_evaluate_pnp(monkeypatch, mode):
    """torch.autograd.forward_ad, torch.func.jvp and torch.func.linearize through evaluate_pnp's residual, Jacobian and
    cost on the emulator: the eager jvp formula of the evaluate_full operator, against the oracle."""
    simt_native.install(monkeypatch)
    from epropnp.camera import PerspectiveCamera
    from epropnp.common import evaluate_pnp
    from epropnp.cost_fun import HuberPnPCost
    c = jv.build_case(6, 24, 2, 2, CPU, bounds=True)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    names = ("x3d", "x2d", "w2d", "delta", "pose", "cam", "lb", "ub")
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], pose=c["poses"], cam=c["cam_mats"],
               lb=c["lb"], ub=c["ub"])

    def f(x3d, x2d, w2d, delta, pose, cam, lb, ub):
        camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
        r, cost, j = evaluate_pnp(x3d, x2d, w2d, pose, camera, HuberPnPCost(delta=delta), out_residual=True,
                                  out_jacobian=True, out_cost=True)
        return r, j, cost
    got = jv.forward_mode(f, [src[k] for k in names], [c["t"][k] for k in names], mode)
    jv.assert_close(dict(zip(jv.OUTPUTS, got)), c, mode)


@pytest.mark.parametrize("mode", ["jvp", "linearize"])
def test_gn_step_under_torch_func(monkeypatch, mode):
    """LMSolver.gn_step's tangent under torch.func.jvp and torch.func.linearize equals torch.autograd.forward_ad's.
    linearize traces the step with make_fx and replays the graph, so every kernel call, the primal evaluation's
    included, must be in that graph.  Fresh native output buffers are filled with NaN here: a call the trace missed
    leaves them so in the replay."""
    simt_native.install(monkeypatch)
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp_b200 import native
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(native.Problem, "empty",
                        lambda self, *s: torch.full(s, float("nan"), dtype=torch.float32, device=self.device))
    c = jv.build_case(6, 40, 1, 3, CPU, bounds=True)
    solver = LMSolver(dof=6, num_iter=3)
    names = ("x3d", "x2d", "w2d", "delta", "cam", "lb", "ub")
    src = dict(x3d=c["x3d"], x2d=c["x2d"], w2d=c["w2d"], delta=c["delta"], cam=c["cam_mats"], lb=c["lb"], ub=c["ub"])

    def f(x3d, x2d, w2d, delta, cam, lb, ub):
        camera = PerspectiveCamera(cam_mats=cam, z_min=c["z_min"], lb=lb, ub=ub)
        return (solver.gn_step(x3d, x2d, w2d, c["poses"][0], camera, HuberPnPCost(delta=delta)),)
    run = lambda m: jv.forward_mode(f, [src[k] for k in names], [c["t"][k] for k in names], m)[0]
    ref, got = run("fwad"), run(mode)
    assert torch.isfinite(ref).all() and torch.isfinite(got).all(), mode
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6 * float(ref.abs().max())), mode


def test_needs_derivative():
    import torch.autograd.forward_ad as fwAD
    from epropnp_b200 import ops
    x = torch.ones(3)
    assert not ops.needs_derivative(x, None, 1.0)
    with fwAD.dual_level():
        assert ops.needs_derivative(fwAD.make_dual(x, torch.ones(3))) and not ops.needs_derivative(x)
    assert ops.needs_derivative(x.clone().requires_grad_(True))
    with torch.no_grad():
        assert not ops.needs_derivative(x.clone().requires_grad_(True))
