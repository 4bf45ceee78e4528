"""Cluster-split EPnP initialiser on the H100 (epnp_epnp_init_split_f32 / EPnPSolver above the resident limit): parity
with the cv2 goldens (dense16k: two 128 x 128 coordinate maps, and the resident kernel's six cases at C = 2 and 8), the
split call against the resident kernel, determinism, batch and cluster-size independence of the kept set, the largest
N, isolation of bad objects, and the reference's whole 6DoF test loop at N = 16,384."""
import os

import numpy as np
import pytest
import torch

from conftest import err_vs, load_golden, record_parity
from test_epnp_host_cpu import parity, quat_angle

pytestmark = pytest.mark.gpu
CASES = ("dense", "cube512", "camera", "select", "small", "outliers")


def tensors(g, dev):
    return tuple(torch.from_numpy(g[k]).to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats"))


def masks(g):
    return [c >= np.quantile(c, g["q"]) for c in g["w2d"].mean(-1)]


def numpy_counts(w2d, q):
    conf = np.asarray(w2d, np.float32).mean(-1)
    return [int((c >= np.quantile(c, np.float32(q))).sum()) for c in conf]


def pose_gaps(a, b):
    """max rotation angle (rad) and max relative translation difference between two pose batches"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ang = max(quat_angle(p[3:], r[3:]) for p, r in zip(a, b))
    trel = float((np.linalg.norm(a[:, :3] - b[:, :3], axis=1) / np.linalg.norm(b[:, :3], axis=1)).max())
    return ang, trel


def test_dense16k_golden_parity(cuda_device):
    from epropnp_b200 import native
    g = load_golden(os.path.join("epnp", "dense16k"))
    N = g["x3d"].shape[1]
    assert N > native.max_points(6)
    pose, n_sel = native.epnp_init_split(*tensors(g, cuda_device), float(g["q"]), want_n_sel=True)
    torch.cuda.synchronize()
    assert n_sel.cpu().tolist() == g["n_sel"].tolist()
    ang, trel, ties = parity(pose.cpu().numpy(), g, masks(g))
    record_parity("epnp_split_dense16k", max_rot_angle_rad=ang, max_rel_t=trel, near_ties=ties,
                  objects=int(g["x3d"].shape[0]), cluster_ctas=native.split_ctas(6, N))


@pytest.mark.parametrize("ctas", [2, 8])
@pytest.mark.parametrize("case", CASES)
def test_existing_goldens_through_the_split_call(cuda_device, case, ctas):
    from epropnp_b200 import native
    g = load_golden(os.path.join("epnp", case))
    pose, n_sel = native.epnp_init_split(*tensors(g, cuda_device), float(g["q"]), want_n_sel=True, cluster_ctas=ctas)
    torch.cuda.synchronize()
    assert n_sel.cpu().tolist() == g["n_sel"].tolist()
    parity(pose.cpu().numpy(), g, masks(g))


def _dense(B, N, seed, dev, grid2d=True):
    from epropnp_b200.synth import make_problem
    pc = make_problem(B, N, seed=seed, grid2d=grid2d)
    return {k: v.to(dev) for k, v in pc.items()}


def test_split_against_resident(cuda_device):
    from epropnp_b200 import native
    pc = _dense(256, 4096, 41, cuda_device)
    t = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"])
    res, n_res = native.epnp_init(*t, 0.8, want_n_sel=True)
    spl, n_spl = native.epnp_init_split(*t, 0.8, want_n_sel=True, cluster_ctas=2)
    torch.cuda.synchronize()
    assert torch.equal(n_spl, n_res)
    ang, trel = pose_gaps(spl.cpu(), res.cpu())
    record_parity("epnp_split_vs_resident_N4096", max_rot_angle_rad=ang, max_rel_t=trel, objects=256, cluster_ctas=2)
    assert ang < 1e-5 and trel < 1e-5, (ang, trel)


def test_deterministic_batch_and_cluster_size_independent(cuda_device):
    from epropnp_b200 import native
    N = 16384
    pc = _dense(64, N, 42, cuda_device)
    t = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"])
    a, na = native.epnp_init_split(*t, 0.8, want_n_sel=True)
    b = native.epnp_init_split(*t, 0.8)
    h = 32
    c = native.epnp_init_split(*(x[:h] for x in t), 0.8)
    torch.cuda.synchronize()
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and torch.equal(a[:h], c)
    assert na.cpu().tolist() == numpy_counts(pc["w2d"].cpu().numpy(), 0.8)
    worst = (0.0, 0.0)
    for ctas in range(native.split_ctas(6, N), 9):
        p, n = native.epnp_init_split(*t, 0.8, want_n_sel=True, cluster_ctas=ctas)
        torch.cuda.synchronize()
        assert torch.equal(n, na), ctas
        ang, trel = pose_gaps(p.cpu(), a.cpu())
        assert ang < 1e-5 and trel < 1e-5, (ctas, ang, trel)
        worst = (max(worst[0], ang), max(worst[1], trel))
    record_parity("epnp_split_cluster_sizes_N16384", max_rot_angle_rad=worst[0], max_rel_t=worst[1], objects=64)


def test_largest_object_and_refusal(cuda_device):
    from epropnp_b200 import native
    nmax = native.max_points_split(6)
    assert nmax >= 16384
    pc = _dense(2, nmax, 43, cuda_device, grid2d=False)            # the limit is not a square
    pose, n = native.epnp_init_split(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], 0.8, want_n_sel=True)
    torch.cuda.synchronize()
    assert torch.isfinite(pose).all()
    assert n.cpu().tolist() == numpy_counts(pc["w2d"].cpu().numpy(), 0.8)
    gt = pc["pose_gt"][:, :3]
    assert float(((pose[:, :3] - gt).norm(dim=1) / gt.norm(dim=1)).max()) < 1e-2
    big = _dense(1, nmax + 64, 43, cuda_device, grid2d=False)
    with pytest.raises(native.NativeError, match="shared memory"):
        native.epnp_init_split(big["x3d"], big["x2d"], big["w2d"], big["cam_mats"], 0.8)


def test_bad_objects_leave_the_others_unchanged(cuda_device):
    from epropnp_b200 import native
    pc = _dense(8, 16384, 44, cuda_device)
    x3d, x2d, w2d, cam = pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"]
    base, n0 = native.epnp_init_split(x3d, x2d, w2d, cam, 0.8, want_n_sel=True)
    x3d2, w2d2 = x3d.clone(), w2d.clone()
    x3d2[3, :, 2] = 0.0                                        # object 3: coplanar points
    w2d2[5, 16000, 1] = float("nan")                           # object 5: a NaN confidence, in the last rank's range
    pose, n = native.epnp_init_split(x3d2, x2d, w2d2, cam, 0.8, want_n_sel=True)
    torch.cuda.synchronize()
    keep = [i for i in range(8) if i not in (3, 5)]
    assert torch.equal(pose[keep], base[keep]) and torch.equal(n[keep], n0[keep])
    assert torch.isnan(pose[5]).all() and int(n[5]) == 0
    assert int(n[3]) == int(n0[3])


def test_reference_test_loop_at_16k(cuda_device, monkeypatch):
    """EPnP on the 20 % most confident points, GN(3), then the Monte-Carlo forward from that pose, as
    EPro-PnP-6DoF/lib/test.py:178-221 runs them, on two 128 x 128 coordinate maps."""
    from epropnp_b200 import native
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epnp import EPnPSolver
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    g = load_golden(os.path.join("epnp", "dense16k"))
    x3d, x2d, w2d, cam = tensors(g, cuda_device)
    camera = PerspectiveCamera(cam_mats=cam, z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(x2d, w2d)
    layer = EProPnP6DoF(mc_samples=512, num_iter=4, solver=LMSolver(6, 3, init_solver=EPnPSolver(0.8)))
    pose = layer(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]
    ref = LMSolver(6, 3)(x3d, x2d, w2d, camera, cost_fun, pose_init=torch.from_numpy(g["pose"]).float().to(cuda_device),
                         fast_mode=True)[0]
    e = err_vs(pose.cpu(), ref.cpu())
    record_parity("epnp_split_gn3_end_to_end_N16384", pose_rel_err=e)
    assert e < 1e-4, e
    out = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=pose, force_init_solve=False,
                                    fast_mode=True)
    torch.cuda.synchronize()
    assert torch.isfinite(out[4]).all() and torch.isfinite(out[0]).all()
    calls = []
    split_cost = native.evaluate_cost_split
    monkeypatch.setattr(native, "evaluate_cost_split", lambda *a, **k: calls.append(1) or split_cost(*a, **k))
    forced = layer.monte_carlo_forward(x3d, x2d, w2d, camera, cost_fun, pose_init=pose, force_init_solve=True,
                                       fast_mode=True)
    torch.cuda.synchronize()
    assert len(calls) >= 2                                      # the cost at pose_init and at the EPnP pose
    assert torch.isfinite(forced[0]).all() and torch.isfinite(forced[4]).all()
