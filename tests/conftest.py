"""Shared fixtures.  `-m "not gpu"` runs here on CPU; `-m gpu` needs an H100 and goes through the C ABI."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "epro-pnp_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the kernels are built for sm_90a only)")


def golden_names(prefix=""):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, prefix + "*.npz")))


def load_golden(name):
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return {k: g[k] for k in g.files}


def golden_bounds(g, dtype=torch.float32):
    """-> (lb, ub) as None | float | tensor, the way the reference camera holds them."""
    kind = int(g["bounds"])
    if kind == 0:
        return None, None
    if kind == 1:
        return float(g["lb"]), float(g["ub"])
    return torch.from_numpy(g["lb"]).to(dtype), torch.from_numpy(g["ub"]).to(dtype)


def err_vs(a, b):
    """max |a-b| relative to the scale of b (max |b|) -- the "rel" of BASELINE.json's 1e-4."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def err_stats(a, b):
    """Measured error of `a` against the reference `b`: scale-relative max (the "rel" of BASELINE.json), absolute max
    and absolute p50 / p99, plus the scale they are relative to."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    d = np.abs(a - b).ravel()
    scale = float(max(np.abs(b).max(), 1e-30)) if b.size else 1.0
    if d.size == 0:
        return dict(rel_max=0.0, abs_max=0.0, abs_p50=0.0, abs_p99=0.0, scale=scale, n=0)
    return dict(rel_max=float(d.max() / scale), abs_max=float(d.max()), abs_p50=float(np.percentile(d, 50)),
                abs_p99=float(np.percentile(d, 99)), scale=scale, n=int(d.size))


# Measured parity numbers of the GPU suite: every `-m gpu` parity test records what it measured (not just pass / fail);
# the session writes them to gpurun_out/parity_r2.json (EPNP_PARITY_OUT overrides), which is copied to profiles/.
_PARITY = {}


def record_parity(case, **metrics):
    _PARITY.setdefault(case, {}).update(metrics)


def pytest_sessionfinish(session, exitstatus):
    if not _PARITY:
        return
    import json
    path = os.environ.get("EPNP_PARITY_OUT", os.path.join(ROOT, "gpurun_out", "parity_r2.json"))
    os.makedirs(os.path.dirname(path), exist_ok=True)
    merged = {}
    if os.path.exists(path):
        try:
            merged = json.load(open(path))
        except Exception:
            merged = {}
    merged.update(_PARITY)
    with open(path, "w") as f:
        json.dump(merged, f, indent=1, sort_keys=True)


def assert_lm_parity(pose, cost, ref_pose, ref_cost, tol, max_flip_frac=0.5, what=""):
    """LM parity per object.  A fixed-iteration trust-region solve is path dependent: an accept/reject
    decision that sits inside fp32 noise (levenberg_marquardt.py:228) sends it to a different point of a
    flat valley with the SAME cost (SURVEY.md section 7 hard part 1).  So an object passes if its pose is within
    `tol` (relative to the pose scale) OR it is cost-equivalent to the reference (cost equal to 2e-6
    relative, the fp32 cost-evaluation noise) with the pose still within 50 * tol.  Returns the fraction
    of objects that needed the second clause (the "flip rate"), which is bounded by max_flip_frac."""
    pose, ref_pose = np.asarray(pose, np.float64), np.asarray(ref_pose, np.float64)
    scale = max(np.abs(ref_pose).max(), 1e-30)
    perr = np.abs(pose - ref_pose).max(axis=1) / scale
    tight = perr < tol
    flips = ~tight
    if cost is not None and flips.any():
        cost, ref_cost = np.asarray(cost, np.float64), np.asarray(ref_cost, np.float64)
        crel = np.abs(cost - ref_cost) / np.maximum(np.abs(ref_cost), 1e-30)
        ok = tight | ((crel < 2e-6) & (perr < 50 * tol))
    else:
        ok = tight
    assert ok.all(), f"{what}: pose err {perr}, tol {tol}"
    frac = float(flips.mean())
    assert frac <= max_flip_frac, f"{what}: {frac:.2%} of objects are cost-equivalent flips (> {max_flip_frac:.0%})"
    return frac


@pytest.fixture(scope="session")
def cuda_device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
