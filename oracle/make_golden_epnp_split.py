#!/usr/bin/env python
"""Golden vector of the cluster-split EPnP initialiser (epnp_epnp_init_split_f32): tests/golden/epnp/dense16k.npz, two
objects of a 128 x 128 coordinate map (N = 16,384, more than one SM holds) at q = 0.8, solved as the reference's 6DoF
test loop solves them (see make_golden_epnp.py, whose selection, cv2 call and file format this reuses).  Needs OpenCV
and SciPy (development machines only; the tests read the file).

    python oracle/make_golden_epnp_split.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_epnp import OUT, problem, solve_all  # noqa: E402


def main():
    os.makedirs(OUT, exist_ok=True)
    x3d, x2d, w2d, cam = problem(2, 16384, 27, grid2d=True)
    q = np.float32(0.8)
    pose, reproj, n_sel = solve_all(x3d, x2d, w2d, cam, q)
    np.savez_compressed(os.path.join(OUT, "dense16k.npz"), x3d=x3d, x2d=x2d, w2d=w2d, cam_mats=cam, q=q, n_sel=n_sel,
                        pose=pose, reproj=reproj)
    print(f"dense16k: B={x3d.shape[0]} N={x3d.shape[1]} q={q} n_sel {n_sel.min()}..{n_sel.max()}")


if __name__ == "__main__":
    main()
