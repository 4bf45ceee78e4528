"""EPnP initialiser on the H100 (epnp_epnp_init_f32 / EPnPSolver): parity with the cv2 goldens, the end-to-end test-time
path against the cv2-initialised solve, determinism and batch independence, isolation of bad objects, and refusals."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden, record_parity
from test_epnp_host_cpu import parity

pytestmark = pytest.mark.gpu
CASES = ("dense", "cube512", "camera", "select", "small", "outliers")


def tensors(g, dev):
    return tuple(torch.from_numpy(g[k]).to(dev) for k in ("x3d", "x2d", "w2d", "cam_mats"))


@pytest.mark.parametrize("case", CASES)
def test_golden_parity(cuda_device, case):
    from epropnp_b200 import native
    g = load_golden(os.path.join("epnp", case))
    pose, n_sel = native.epnp_init(*tensors(g, cuda_device), float(g["q"]), want_n_sel=True)
    torch.cuda.synchronize()
    assert n_sel.cpu().tolist() == g["n_sel"].tolist()
    conf = g["w2d"].mean(-1)
    masks = [c >= np.quantile(c, g["q"]) for c in conf]
    ang, trel, ties = parity(pose.cpu().numpy(), g, masks)
    record_parity(f"epnp_{case}", max_rot_angle_rad=ang, max_rel_t=trel, near_ties=ties, objects=int(g["x3d"].shape[0]))
    print(f"{case}: max angle {ang:.2e} rad, max |dt|/|t| {trel:.2e}, near-ties {ties}")


def test_test_time_path_matches_cv2_initialised_solve(cuda_device):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epnp import EPnPSolver
    from epropnp.epropnp import EProPnP6DoF
    from epropnp.levenberg_marquardt import LMSolver
    from conftest import err_vs
    g = load_golden(os.path.join("epnp", "dense"))
    x3d, x2d, w2d, cam = tensors(g, cuda_device)
    camera = PerspectiveCamera(cam_mats=cam, z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(x2d, w2d)
    layer = EProPnP6DoF(mc_samples=512, num_iter=4, solver=LMSolver(6, 3, init_solver=EPnPSolver(0.8)))
    pose = layer(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]
    ref = LMSolver(6, 3)(x3d, x2d, w2d, camera, cost_fun, pose_init=torch.from_numpy(g["pose"]).float().to(cuda_device),
                         fast_mode=True)[0]
    e = err_vs(pose.cpu(), ref.cpu())
    record_parity("epnp_gn3_end_to_end", pose_rel_err=e)
    assert e < 1e-4, e


def test_deterministic_and_batch_independent(cuda_device):
    from epropnp_b200 import native
    from epropnp_b200.synth import make_problem
    B, N = 4096, 4096
    pc = make_problem(256, N, seed=31, grid2d=True)            # 256 distinct objects, tiled to B
    x3d, x2d, w2d, cam = (pc[k].to(cuda_device).repeat(B // 256, *([1] * (pc[k].dim() - 1)))
                          for k in ("x3d", "x2d", "w2d", "cam_mats"))
    a = native.epnp_init(x3d, x2d, w2d, cam, 0.8)
    b = native.epnp_init(x3d, x2d, w2d, cam, 0.8)
    h = B // 2
    c = native.epnp_init(x3d[:h], x2d[:h], w2d[:h], cam[:h], 0.8)
    torch.cuda.synchronize()
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)
    assert torch.equal(a[:h], c)


def test_bad_objects_leave_the_others_unchanged(cuda_device):
    from epropnp_b200 import native
    g = load_golden(os.path.join("epnp", "cube512"))
    x3d, x2d, w2d, cam = tensors(g, cuda_device)
    base, n0 = native.epnp_init(x3d, x2d, w2d, cam, 0.8, want_n_sel=True)
    x3d2, w2d2 = x3d.clone(), w2d.clone()
    x3d2[3, :, 2] = 0.0                                        # object 3: coplanar points
    w2d2[7, 11, 1] = float("nan")                              # object 7: a NaN confidence
    pose, n = native.epnp_init(x3d2, x2d, w2d2, cam, 0.8, want_n_sel=True)
    torch.cuda.synchronize()
    keep = [i for i in range(x3d.shape[0]) if i not in (3, 7)]
    assert torch.equal(pose[keep], base[keep]) and torch.equal(n[keep], n0[keep])
    assert torch.isnan(pose[7]).all() and int(n[7]) == 0
    assert int(n[3]) == int(n0[3])                             # the selection does not look at x3d


def test_shapes_and_refusals(cuda_device):
    from epropnp_b200 import capi, native
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import HuberPnPCost
    from epropnp.epnp import EPnPSolver
    from epropnp.levenberg_marquardt import LMSolver
    from epropnp_b200.synth import make_problem
    dev = cuda_device
    nmax = capi.lib().epnp_max_points(6, 0, 0)
    assert nmax >= 4096
    pc = {k: v.to(dev) for k, v in make_problem(2, nmax, seed=4).items()}
    pose, n = native.epnp_init(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], 0.8, want_n_sel=True)
    torch.cuda.synchronize()
    assert torch.isfinite(pose).all() and (n > 0).all()
    assert native.epnp_init(pc["x3d"][:0], pc["x2d"][:0], pc["w2d"][:0], pc["cam_mats"][:0]).shape == (0, 7)
    big = {k: v.to(dev) for k, v in make_problem(1, nmax + 4, seed=4).items()}
    with pytest.raises(native.NativeError):
        native.epnp_init(big["x3d"], big["x2d"], big["w2d"], big["cam_mats"], 0.8)
    with pytest.raises(native.NativeError):                    # 20 points at q = 0.9 keep at most 2
        native.epnp_init(pc["x3d"][:, :20], pc["x2d"][:, :20], pc["w2d"][:, :20], pc["cam_mats"], 0.9)
    with pytest.raises(native.NativeError):
        native.epnp_init(pc["x3d"].cpu(), pc["x2d"].cpu(), pc["w2d"].cpu(), pc["cam_mats"].cpu())
    camera = PerspectiveCamera(cam_mats=pc["cam_mats"])
    with pytest.raises(ValueError):
        LMSolver(4, 3, init_solver=EPnPSolver())(pc["x3d"], pc["x2d"], pc["w2d"], camera, HuberPnPCost(), fast_mode=True)
