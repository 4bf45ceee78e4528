#!/usr/bin/env python
"""Golden vectors of the EPnP initialiser (epnp_epnp_init_f32 / EPnPSolver): tests/golden/epnp/<case>.npz.

Per object, the reference's 6DoF test loop (EPro-PnP-6DoF/lib/test.py:179-181, restated here) keeps the points whose
confidence reaches the q-quantile of the object's confidences and hands them to OpenCV's EPnP:

    conf = w2d.mean(-1)                        # (N,) float32
    mask = conf >= np.quantile(conf, q)
    cv2.solvePnP(x3d[mask], x2d[mask], K, None, flags=cv2.SOLVEPNP_EPNP)

Each file stores the inputs (x3d, x2d, w2d, cam_mats: float32), q, the mask count n_sel (int32), cv2's pose as
[x y z w i j k] (float64, quaternion from scipy, w >= 0) and reproj: the mean pixel reprojection error of that pose over
the kept points, in float64.  Needs OpenCV and SciPy (development machines only; the tests read the files).

    python oracle/make_golden_epnp.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))
OUT = os.path.join(ROOT, "tests", "golden", "epnp")


def keep_mask(w2d, q):
    conf = w2d.mean(-1)
    return conf >= np.quantile(conf, q)


def cv2_epnp(x3d, x2d, K):
    """-> pose [x y z w i j k] (float64), mean pixel reprojection error of that pose."""
    import cv2
    from scipy.spatial.transform import Rotation
    ok, rvec, tvec = cv2.solvePnP(x3d, x2d, K, None, flags=cv2.SOLVEPNP_EPNP)
    assert ok
    quat = Rotation.from_rotvec(rvec.ravel()).as_quat()[[3, 0, 1, 2]]
    quat = quat * (1.0 if quat[0] >= 0 else -1.0)
    R = Rotation.from_rotvec(rvec.ravel()).as_matrix()
    xc = x3d.astype(np.float64) @ R.T + tvec.ravel()
    K = K.astype(np.float64)
    uv = np.stack((K[0, 2] + K[0, 0] * xc[:, 0] / xc[:, 2], K[1, 2] + K[1, 1] * xc[:, 1] / xc[:, 2]), -1)
    err = np.linalg.norm(uv - x2d.astype(np.float64), axis=-1).mean()
    return np.concatenate((tvec.ravel(), quat)), err


def solve_all(x3d, x2d, w2d, cam, q):
    B = x3d.shape[0]
    pose, reproj, n_sel = np.zeros((B, 7)), np.zeros(B), np.zeros(B, np.int32)
    for b in range(B):
        m = keep_mask(w2d[b], q)
        n_sel[b] = m.sum()
        pose[b], reproj[b] = cv2_epnp(x3d[b][m], x2d[b][m], cam[b])
    return pose, reproj, n_sel


def problem(B, N, seed, **kw):
    from epropnp_b200.synth import make_problem
    pc = make_problem(B, N, seed=seed, **kw)
    return tuple(pc[k].numpy() for k in ("x3d", "x2d", "w2d", "cam_mats"))


def tied_weights(B, N, seed):
    """Confidences on a coarse grid (many ties), and pairs one ulp apart straddling each row's threshold."""
    rng = np.random.default_rng(seed)
    conf = (rng.integers(1, 40, size=(B, N)) / 16.0).astype(np.float32)
    for b in range(B):
        thr = np.float32(np.quantile(conf[b], np.float32(0.8)))
        j = rng.choice(N, 6, replace=False)
        conf[b, j[:2]] = thr
        conf[b, j[2:4]] = np.nextafter(thr, np.float32(np.inf))
        conf[b, j[4:]] = np.nextafter(thr, np.float32(-np.inf))
    return np.repeat(conf[..., None], 2, axis=-1)


def cases():
    # three dense objects keep the file small; the GPU suite runs the dense shape at B = 4096 on synthetic inputs
    yield "dense", problem(3, 4096, 21, grid2d=True), 0.8
    yield "cube512", problem(16, 512, 22), 0.0
    x3d, x2d, w2d, cam = problem(16, 512, 23)
    Kn = np.array([[700.0, 0.0, 300.0], [0.0, 950.0, 262.5], [0.0, 0.0, 1.0]], np.float32)
    x2d = ((x2d - cam[:, None, :2, 2]) / cam[:, None, 0:1, 0] * np.diag(Kn)[:2] + Kn[:2, 2]).astype(np.float32)
    yield "camera", (x3d, x2d, w2d, np.broadcast_to(Kn, cam.shape).copy()), 0.5
    x3d, x2d, _, cam = problem(8, 257, 24)
    yield "select", (x3d, x2d, tied_weights(8, 257, 24), cam), 0.8
    # 40 points at q = 0.8 keep 8.  Fewer do not make a parity case: with 4 or 5 points the 2n x 12 matrix M has rank
    # 8 or 10, so M^T M has a 4- or 2-dimensional null space, with 6 or 7 its smallest singular values lie close
    # together, and which basis of that subspace cv2 returns is decided by rounding
    yield "small", problem(16, 40, 25), 0.8
    yield "outliers", problem(16, 512, 26, outlier_frac=0.2), 0.8


def main():
    os.makedirs(OUT, exist_ok=True)
    for name, (x3d, x2d, w2d, cam), q in cases():
        q = np.float32(q)
        pose, reproj, n_sel = solve_all(x3d, x2d, w2d, cam, q)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), x3d=x3d, x2d=x2d, w2d=w2d, cam_mats=cam, q=q,
                            n_sel=n_sel, pose=pose, reproj=reproj)
        print(f"{name}: B={x3d.shape[0]} N={x3d.shape[1]} q={q} n_sel {n_sel.min()}..{n_sel.max()}")


if __name__ == "__main__":
    main()
