"""The Hessian-vector-product kernels (epnp_cost_hvp_f32) on the CPU: pnp_kernels.cu under the SIMT emulator, held to
the oracle's float64 double backward with the bound of test_cost_hvp_gpu.py (whose helpers this file uses), at small
sizes; and the second-order formula of the layer's cost backwards end to end."""
import pytest
import torch

import simt_native
import test_cost_hvp_gpu as hv

CPU = torch.device("cpu")


@pytest.mark.parametrize("dof,N,P,B,bounds,zmin", [(6, 7, 3, 2, False, False), (6, 33, 130, 2, True, True),
                                                    (4, 129, 2, 3, True, False), (4, 20, 5, 2, False, True)])
def test_kernels_against_float64(monkeypatch, dof, N, P, B, bounds, zmin):
    simt_native.install(monkeypatch)
    c = hv.build_case(dof, N, P, B, CPU, bounds=bounds, zmin=zmin)
    got = hv.run_hvp(c)
    hv.assert_close(got, c, (dof, N, P, B))
    # each tangent part alone: the outputs are linear in v
    parts = {k: hv.run_hvp(c, t={k: v}) for k, v in c["t"].items()}
    for out in hv.OUTPUTS:
        if got[out] is not None:
            total = sum(p[out].double() for p in parts.values())
            assert torch.allclose(total, got[out].double(), rtol=1e-4, atol=1e-5 * float(got[out].abs().max())), out


def test_only_the_asked_outputs_are_written(monkeypatch):
    simt_native.install(monkeypatch)
    c = hv.build_case(6, 16, 3, 2, CPU, bounds=True)
    full = hv.run_hvp(c)
    for i, k in enumerate(hv.OUTPUTS):
        want = [j == i for j in range(len(hv.OUTPUTS))]
        one = hv.run_hvp(c, want=want)
        assert all(one[o] is None for o in hv.OUTPUTS if o != k)
        assert torch.equal(one[k], full[k]), k


def test_second_order_through_the_layer(monkeypatch):
    """grad of (grad cost . v) through evaluate_pnp's cost with every input differentiable, on the emulator."""
    simt_native.install(monkeypatch)
    from epropnp_b200 import ops
    monkeypatch.setattr(ops.native, "max_points", lambda *a, **k: 1 << 20)
    c = hv.build_case(6, 24, 1, 2, CPU, bounds=True)
    c["t"].pop("pose")
    ins = {k: c[k].clone().requires_grad_(True) for k in ("x3d", "x2d", "w2d", "delta", "cam_mats", "lb", "ub")}
    poses = c["poses"].clone().requires_grad_(True)
    prob = ops.problem_args(ins["x3d"], ins["x2d"], ins["w2d"], ins["cam_mats"], ins["lb"], ins["ub"], ins["delta"])
    cost = ops.evaluate_cost(*prob, poses.transpose(0, 1), 6, c["z_min"])          # (1, B)
    leaves = list(ins.values()) + [poses]
    g = torch.autograd.grad((cost * c["up"].T).sum(), leaves, create_graph=True)
    t = [c["t"]["x3d"], c["t"]["x2d"], c["t"]["w2d"], c["t"]["delta"], c["t"]["cam"], c["t"]["lb"], c["t"]["ub"]]
    loss = sum((gi * ti).sum() for gi, ti in zip(g, t))
    h = dict(zip(("x3d", "x2d", "w2d", "delta", "cam", "lb", "ub", "pose"),
                 torch.autograd.grad(loss, leaves, retain_graph=True)))
    ref = hv.oracle_hvp(c, torch.float64)
    for k, v in h.items():
        err = hv.rel_rows(v, ref[k], 1)
        assert (err < 1e-3).all(), (k, err.max())
    # a third derivative raises from cost_hvp's missing formula
    h3 = torch.autograd.grad(loss, leaves, create_graph=True)
    with pytest.raises(RuntimeError, match=hv.THIRD):
        torch.autograd.grad(sum(x.sum() for x in h3), leaves)
