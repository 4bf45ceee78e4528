"""The Hessian-vector-product kernel of pose_opt_plus (epnp_gn_plus_hvp_f32) on the CPU: pnp_kernels.cu under the SIMT
emulator, held to the oracle's float64 double backward with the bound of test_gn_plus_hvp_gpu.py (whose helpers this
file uses), at small sizes; and the second-order formulas of gn_plus_backward / gn_plus_camera_backward end to end."""
import pytest
import torch

import simt_native
import test_gn_plus_hvp_gpu as hv

CPU = torch.device("cpu")


@pytest.mark.parametrize("dof,N,B,bounds,zmin,rd", [(6, 7, 2, None, False, 0.1), (6, 33, 2, "tensor", True, 0.1),
                                                    (4, 129, 3, "tensor", False, 0.1), (4, 21, 2, None, True, 0.5),
                                                    (6, 65, 2, "scalar", False, 0.02)])
def test_kernel_against_float64(monkeypatch, dof, N, B, bounds, zmin, rd):
    simt_native.install(monkeypatch)
    c = hv.build_case(dof, N, B, CPU, bounds=bounds, zmin=zmin, relative_delta=rd)
    got = hv.run_hvp(c)
    fr, _ = hv.assert_close(got, c, (dof, N, B, bounds, zmin))
    assert fr["ill_conditioned"] == 0, fr
    assert 0.0 < fr["outlier"] < 1.0, fr
    if bounds:
        assert fr["clamped"] > 0, fr
    if zmin:
        assert fr["below_zmin"] > 0, fr
    # each tangent part alone: the outputs are linear in u
    parts = {k: hv.run_hvp(c, t={k: v}) for k, v in c["t"].items()}
    for out in hv.OUTPUTS:
        if got[out] is not None:
            total = sum(p[out].double() for p in parts.values())
            assert torch.allclose(total, got[out].double(), rtol=1e-4, atol=1e-5 * float(got[out].abs().max())), out


def test_only_the_asked_outputs_are_written(monkeypatch):
    simt_native.install(monkeypatch)
    c = hv.build_case(6, 16, 2, CPU, bounds="tensor")
    full = hv.run_hvp(c)
    for i, k in enumerate(hv.OUTPUTS):
        want = [j == i for j in range(len(hv.OUTPUTS))]
        one = hv.run_hvp(c, want=want)
        assert all(one[o] is None for o in hv.OUTPUTS if o != k)
        assert torch.equal(one[k], full[k]), k


def test_second_order_through_the_layer(monkeypatch):
    """pose_opt_plus differentiated twice through LMSolver's native path, every problem input a leaf, on the
    emulator; then a third derivative raises."""
    simt_native.install(monkeypatch)
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    c = hv.build_case(6, 24, 2, CPU, bounds="tensor", seed=13)
    _, h_nat, leaves = hv._second_order(c, torch.float32, True)
    ref = hv.oracle_hvp(c, torch.float64)
    for k, v in zip(hv.TANGENTS, h_nat):
        err = hv.rel_rows(v, ref[k], 1)
        assert (err < 1e-3).all(), (k, err.max())
    with pytest.raises(RuntimeError, match=hv.THIRD):
        torch.autograd.grad(sum(hi.sum() for hi in h_nat), leaves)


def test_penalty_on_a_loss_linear_in_pose_opt_plus(monkeypatch):
    """The Monte-Carlo loss plus a loss linear in pose_opt_plus under a gradient-norm penalty: the native step against
    the torch composite (EPNP_NATIVE_GN_STEP=0) on the emulator.  Without a graph on pose_opt_plus's first gradient the
    penalty's gradient loses the pose_opt_plus Hessian term."""
    simt_native.install(monkeypatch)
    pc, noise, vals = hv._mc_inputs(CPU, B=2, N=24, M=32)
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "1")
    _, h_nat = hv._penalised_step(vals, pc, noise, CPU, True)
    monkeypatch.setenv("EPNP_NATIVE_GN_STEP", "0")
    _, h_cmp = hv._penalised_step(vals, pc, noise, CPU, True)
    for name, a, b in zip(("x3d", "x2d", "w2d", "delta", "cam_mats"), h_nat, h_cmp):
        err = hv.rel_rows(a, b, 1)
        assert (err < 2e-3).all(), (name, err.max())
