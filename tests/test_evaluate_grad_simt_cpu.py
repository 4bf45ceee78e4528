"""epnp_evaluate_backward_f32 on the CPU: pnp_kernels.cu under the single-CTA SIMT emulator (tests/simt_emul), held to
the oracle's float64 autograd per object with the bound of test_evaluate_grad_gpu.py (whose helpers this file uses),
and to the reference's own autograd (tests/golden/evaluate_grad).  The exact properties of the GPU suite hold here too:
an object alone equals its row of the batch, one gradient asked alone equals the same gradient asked with all, a zero
upstream gives zero.  Autograd: the Function's forward equals the no-grad call, its gradients are the kernel's reduced
to the inputs' shapes, and a broadcast (B, N, 1) weight receives the sum over its expanded axis."""
import numpy as np
import pytest
import torch

import simt_native
import test_evaluate_grad_gpu as eg
from conftest import golden_bounds, load_golden
from test_oracle_evaluate_grad_cpu import NAMES
from epropnp import autograd as ag
from epropnp.camera import PerspectiveCamera
from epropnp.cost_fun import HuberPnPCost
from epropnp_b200 import native


@pytest.mark.parametrize("dof,N,S,bounds,zmin,clip,ups", [
    (6, 1, 1, None, False, True, eg.UPS),
    (6, 200, 3, "tensor", False, True, eg.UPS),
    (4, 130, 2, "scalar", True, False, eg.UPS),
    (6, 150, 2, None, True, True, ("jac",)),
    (4, 160, 1, "shared", False, True, ("res",)),
    (6, 140, 2, "tensor", False, False, ("cost",)),
])
def test_kernel_against_float64(monkeypatch, dof, N, S, bounds, zmin, clip, ups):
    simt_native.install(monkeypatch)
    c = eg.build_case(dof, N, S, B=3, bounds=bounds, zmin=zmin, outliers=0.1 if N > 1 else 0.0, clip=clip, ups=ups)
    got = eg.run_kernel(c)
    g64, fr = eg.reference(c, torch.float64, census=True)
    g32, _ = eg.reference(c, torch.float32)
    if bounds:
        assert fr["clamped"] > 0.01, fr
    if zmin:
        assert fr["below_zmin"] > 0.03, fr
    if N > 1:
        assert 0.01 < fr["outlier"] < 0.99, fr
    eg.assert_per_object(got, g64, g32, (dof, N, S, bounds))
    eg.exact_properties(c)


@pytest.mark.parametrize("name", NAMES)
def test_kernel_against_reference_goldens(monkeypatch, name):
    """The reference's float64 autograd, with the bound max(2e-4, 5 * the reference's float32 floor) per object."""
    simt_native.install(monkeypatch)
    g = load_golden("evaluate_grad/" + name)
    t = lambda k: torch.from_numpy(g[k]).float()
    lb, ub = golden_bounds(g)
    prob = native.Problem(t("x3d"), t("x2d"), t("w2d"), t("cam_mats"), lb, ub, t("delta"))
    pose, dof = t("pose"), int(g["dof"])
    stacked = pose.dim() == 3
    S = pose.shape[0] if stacked else 1
    ups = [t(k) if stacked else t(k)[None] for k in ("g_res", "g_jac", "g_cost")]
    tensor_b = torch.is_tensor(lb)
    got = native.evaluate_backward(prob, pose if stacked else pose[None], dof, float(g["z_min"]), eg.HUBER_EPS,
                                   bool(g["clip_jac"]), *ups, want=(True,) * 6 + (tensor_b,) * 2)
    for name_k, a in zip(("x3d", "x2d", "w2d", "delta", "pose", "cam_mats", "lb", "ub"), got):
        if a is None:
            continue
        ref, ref32 = g[f"grad_{name_k}"], g[f"ref32_grad_{name_k}"]
        a = a.double().numpy()
        if name_k == "pose":
            a = a if stacked else a[0]
            # the reference's rotation form differs from the kernel's off the unit sphere only: compare without the
            # component along q (the goldens' quaternions are unit to float64 rounding)
            from test_oracle_cost_pose_grad_cpu import comparable
            a, ref, ref32 = (comparable(x, g["pose"]) for x in (a, ref, ref32))
            a, ref, ref32 = (np.moveaxis(x, -2, 0) if stacked else x for x in (a, ref, ref32))
        for o in range(ref.shape[0]):
            if not np.abs(ref[o]).any():
                assert not np.abs(a[o]).any(), (name, name_k, o)
                continue
            err = np.abs(a[o] - ref[o]).max() / np.abs(ref[o]).max()
            floor = np.abs(ref32[o] - ref[o]).max() / np.abs(ref[o]).max()
            assert err < max(2e-4, 5 * floor), (name, name_k, o, err, floor)


def test_autograd_forward_and_gradients(monkeypatch):
    simt_native.install(monkeypatch)
    c = eg.build_case(6, 90, 3, B=2, bounds="shared", outliers=0.1)
    (x3d, x2d, w2d), poses, camera, cost_fun = eg._layer_inputs(c)
    w1 = w2d[..., :1].detach().clone().requires_grad_(True)             # a broadcast weight
    K = c["cam_mats"][0].clone().requires_grad_(True)                   # one camera for every object
    camera = PerspectiveCamera(cam_mats=K, z_min=c["z_min"], lb=camera.lb, ub=camera.ub)
    for pose in (poses, poses[1]):
        args = (x3d, x2d, w1, pose, camera, cost_fun, True, True, True, True)
        live = ag.evaluate_autograd(*args)
        prob = native.Problem(x3d, x2d, w1, K, camera.lb, camera.ub, cost_fun.delta)
        if pose.dim() == 3:
            rep = lambda v: v.unsqueeze(0).expand((3,) + v.shape).reshape((6,) + v.shape[1:])
            prob = native.Problem(rep(prob.x3d), rep(prob.x2d), rep(prob.w2d), rep(prob.cam), rep(prob.lb),
                                  rep(prob.ub), rep(prob.delta))
        plain = native.evaluate_full(prob, pose.detach().reshape(-1, 7), 6, c["z_min"], eg.HUBER_EPS, True, True, True,
                                     True)
        for a, b in zip(live, plain):
            assert torch.equal(a.detach().reshape(-1), b.reshape(-1))
    r, cost, j = ag.evaluate_autograd(x3d, x2d, w1, poses, camera, cost_fun, True, True, True, True)
    u = c["ups"]
    ((r * u["res"]).sum() + (j * u["jac"]).sum() + (cost * u["cost"]).sum()).backward()
    direct = eg.run_kernel(dict(c, w2d=w1.detach().expand(2, 90, 2), cam_mats=K.detach().expand(2, 3, 3)))
    assert w1.grad.shape == (2, 90, 1) and torch.equal(w1.grad, direct[2].sum(-1, keepdim=True))
    assert torch.equal(K.grad, direct[5].sum(0)) and camera.lb.grad.shape == (2,)
    assert torch.equal(camera.lb.grad, direct[6].sum(0)) and torch.equal(camera.ub.grad, direct[7].sum(0))
    for a, b in ((x3d.grad, direct[0]), (x2d.grad, direct[1]), (cost_fun.delta.grad, direct[3]),
                 (poses.grad, direct[4])):
        assert torch.equal(a, b)


def test_broadcast_weight_receives_the_summed_gradient(monkeypatch):
    """The cost's native backward hands a (B, N, 1) weight the sum of its two columns' gradients (it raised before)."""
    simt_native.install(monkeypatch)
    c = eg.build_case(6, 40, 2, B=2, outliers=0.1)
    w1 = c["w2d"][..., :1].clone().requires_grad_(True)
    cost = ag.evaluate_cost_autograd(c["x3d"], c["x2d"], w1, c["poses"], PerspectiveCamera(cam_mats=c["cam_mats"]),
                                     HuberPnPCost(delta=c["delta"]))
    cost.sum().backward()
    prob = native.Problem(c["x3d"], c["x2d"], w1.detach(), c["cam_mats"], None, None, c["delta"])
    direct = native.cost_backward(prob, 6, 0.1, c["poses"].transpose(0, 1).contiguous(), torch.ones(2, 2))[2]
    assert w1.grad.shape == (2, 40, 1) and torch.equal(w1.grad, direct.sum(-1, keepdim=True))
