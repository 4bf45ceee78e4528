"""The EPnP initialiser's per-object math (csrc/pnp_epnp.cuh) built with g++ through tests/epnp_host.cpp: the point
selection against np.quantile (the kept set must be exactly equal), the poses against the cv2 goldens
(tests/golden/epnp, oracle/make_golden_epnp.py), and a live cross-check against cv2 where OpenCV is installed."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN_DIR, ROOT, load_golden

CASES = ("dense", "cube512", "camera", "select", "small", "outliers")
ANG_TOL, T_TOL, TIE_TOL = 1e-4, 1e-4, 1e-6


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("epnp_host") / "libepnp_host.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                    os.path.join(ROOT, "tests", "epnp_host.cpp")], check=True)
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.epnp_host_select.argtypes = [P, ctypes.c_int, ctypes.c_float, P]
    lib.epnp_host_min_selected.argtypes = [ctypes.c_int, ctypes.c_float]
    lib.epnp_host_solve.argtypes = [P, P, P, P, ctypes.c_int, P, P]
    lib.epnp_host_solve.restype = None
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def select(host, w2d, q):
    w2d = np.ascontiguousarray(w2d, np.float32)
    mask = np.zeros(w2d.shape[0], np.uint8)
    n = host.epnp_host_select(_p(w2d), w2d.shape[0], ctypes.c_float(q), _p(mask))
    return n, mask.astype(bool)


def solve(host, x3d, x2d, K, mask=None):
    x3d, x2d, K = (np.ascontiguousarray(a, np.float32) for a in (x3d, x2d, K))
    pose, err = np.zeros(7, np.float32), np.zeros(3)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    host.epnp_host_solve(_p(x3d), _p(x2d), _p(K), None if m is None else _p(m), x3d.shape[0], _p(pose), _p(err))
    return pose, err


def quat_angle(q1, q2):
    """rotation angle between two [w i j k] quaternions"""
    q1, q2 = np.asarray(q1, np.float64), np.asarray(q2, np.float64)
    d = abs(np.dot(q1 / np.linalg.norm(q1), q2 / np.linalg.norm(q2)))
    return 2.0 * np.arccos(min(d, 1.0))


def mean_reproj(pose, x3d, x2d, K):
    """mean pixel reprojection error of pose [x y z w i j k] (fp64), the camera as EPnP reads it"""
    w, i, j, k = np.asarray(pose[3:], np.float64) / np.linalg.norm(np.asarray(pose[3:], np.float64))
    R = np.array([[w * w + i * i - j * j - k * k, 2 * (i * j - w * k), 2 * (i * k + w * j)],
                  [2 * (i * j + w * k), w * w - i * i + j * j - k * k, 2 * (j * k - w * i)],
                  [2 * (i * k - w * j), 2 * (j * k + w * i), w * w - i * i - j * j + k * k]])
    xc = np.asarray(x3d, np.float64) @ R.T + np.asarray(pose[:3], np.float64)
    K = np.asarray(K, np.float64)
    uv = np.stack((K[0, 2] + K[0, 0] * xc[:, 0] / xc[:, 2], K[1, 2] + K[1, 1] * xc[:, 1] / xc[:, 2]), -1)
    return float(np.linalg.norm(uv - np.asarray(x2d, np.float64), axis=-1).mean())


def parity(poses, g, masks=None):
    """Per object: rotation angle and relative translation error to cv2's pose.  An object outside the tolerances must
    be a near-tie: its pose reprojects as well as cv2's (relative difference <= TIE_TOL).  -> (max angle, max rel t,
    number of near-ties)"""
    ang, trel, ties = [], [], 0
    for b, pose in enumerate(np.asarray(poses, np.float64)):
        ref = g["pose"][b]
        a = quat_angle(pose[3:], ref[3:])
        t = np.linalg.norm(pose[:3] - ref[:3]) / np.linalg.norm(ref[:3])
        ang.append(a)
        trel.append(t)
        if a <= ANG_TOL and t <= T_TOL:
            continue
        m = masks[b] if masks is not None else slice(None)
        e = mean_reproj(pose, g["x3d"][b][m], g["x2d"][b][m], g["cam_mats"][b])
        assert abs(e - g["reproj"][b]) <= TIE_TOL * g["reproj"][b], (b, a, t, e, g["reproj"][b])
        ties += 1
    return max(ang), max(trel), ties


def test_selection_equals_numpy_quantile(host):
    rng = np.random.default_rng(5)
    for trial in range(600):
        N = int(rng.integers(4, 700))
        q = np.float32(rng.choice([0.0, 0.1, 0.25, 0.37, 0.5, 0.8, 0.8, 0.9, 0.99, 1.0]))
        kind = trial % 3
        if kind == 0:
            conf = rng.random(N, dtype=np.float32)
        elif kind == 1:                       # ties
            conf = (rng.integers(0, 7, N) / 8.0).astype(np.float32)
        else:                                 # neighbours one ulp apart around the threshold
            base = np.float32(rng.random())
            steps = rng.integers(-3, 4, N)
            conf = np.array([base] * N, np.float32)
            for s in range(1, 4):
                conf[steps >= s] = np.nextafter(conf[steps >= s], np.float32(np.inf))
                conf[steps <= -s] = np.nextafter(conf[steps <= -s], np.float32(-np.inf))
        # split conf into two channels whose fp32 mean is exactly conf
        w2d = np.stack((conf, conf), -1)
        ref = w2d.mean(-1) >= np.quantile(w2d.mean(-1), q)
        n, mask = select(host, w2d, q)
        assert n == ref.sum() and (mask == ref).all(), (trial, N, q)
        assert n >= host.epnp_host_min_selected(N, ctypes.c_float(q))


def test_selection_of_unequal_channels_and_nan(host):
    rng = np.random.default_rng(6)
    for _ in range(200):
        N = int(rng.integers(4, 300))
        w2d = rng.random((N, 2), dtype=np.float32) * np.float32(rng.choice([1e-3, 1.0, 1e4]))
        conf = w2d.mean(-1)
        ref = conf >= np.quantile(conf, np.float32(0.8))
        n, mask = select(host, w2d, 0.8)
        assert (mask == ref).all()
    w2d[3, 1] = np.nan
    assert select(host, w2d, 0.8)[0] == -1


def test_min_selected_is_attained_by_distinct_confidences(host):
    for N in (4, 5, 20, 40, 257, 4096):
        for q in (0.0, 0.3, 0.8, 0.95, 1.0):
            conf = np.arange(N, dtype=np.float32)
            n, _ = select(host, np.stack((conf, conf), -1), q)
            assert n == host.epnp_host_min_selected(N, ctypes.c_float(q)), (N, q)


@pytest.mark.parametrize("case", CASES)
def test_pose_matches_cv2_golden(host, case):
    g = load_golden(os.path.join("epnp", case))
    poses, masks = [], []
    for b in range(g["x3d"].shape[0]):
        n, m = select(host, g["w2d"][b], float(g["q"]))
        assert n == g["n_sel"][b]
        poses.append(solve(host, g["x3d"][b], g["x2d"][b], g["cam_mats"][b], m)[0])
        masks.append(m)
    parity(poses, g, masks)


def test_without_weights_every_point_is_used(host):
    g = load_golden(os.path.join("epnp", "cube512"))           # q = 0 keeps every point
    pose_all, _ = solve(host, g["x3d"][0], g["x2d"][0], g["cam_mats"][0], None)
    _, m = select(host, g["w2d"][0], 0.0)
    pose_q0, _ = solve(host, g["x3d"][0], g["x2d"][0], g["cam_mats"][0], m)
    assert m.all() and np.array_equal(pose_all, pose_q0)


def test_live_cross_check_against_cv2(host):
    cv2 = pytest.importorskip("cv2")
    pytest.importorskip("scipy")
    import sys
    sys.path.insert(0, ROOT)
    from oracle import make_golden_epnp as mk
    from epropnp_b200.synth import make_problem
    for seed, kw in ((101, dict(grid2d=True)), (102, dict()), (103, dict(outlier_frac=0.1))):
        N = 1024 if kw.get("grid2d") else 300
        pc = make_problem(12, N, seed=seed, **kw)
        x3d, x2d, w2d, cam = (pc[k].numpy() for k in ("x3d", "x2d", "w2d", "cam_mats"))
        pose_ref, reproj, n_sel = mk.solve_all(x3d, x2d, w2d, cam, np.float32(0.8))
        g = dict(x3d=x3d, x2d=x2d, cam_mats=cam, pose=pose_ref, reproj=reproj)
        poses, masks = [], []
        for b in range(12):
            n, m = select(host, w2d[b], 0.8)
            assert n == n_sel[b]
            poses.append(solve(host, x3d[b], x2d[b], cam[b], m)[0])
            masks.append(m)
        parity(poses, g, masks)
    del cv2


def test_golden_files_exist():
    for case in CASES:
        assert os.path.exists(os.path.join(GOLDEN_DIR, "epnp", case + ".npz")), case
