"""The derivative matrix of test_derivative_matrix_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulator
(tests/simt_native.py), held to the same float64 bounds, census and margins, at sizes the emulator affords.  Kept: P = 127,
128 and 129 against cost_hvp_point_kernel's pose tile and cost_hvp_pose_kernel's CTAs, S = 63 and 64 on both sides of
evaluate_jvp's pose-major switch, N = 1 and 129 against the thread loop, one block-by-block case per entry point, scalar
bounds, the all-inlier and all-outlier cases, the exact properties, and the constants the matrix mirrors read out of the
kernel source."""
import os
import re

import pytest

import simt_native
import test_derivative_matrix_gpu as dm
from test_derivative_matrix_gpu import _c
from epropnp_b200 import build

SIMT_SMS = 2            # the batch of the object-independence check: 2 x SMs + 3 = 7 objects


@pytest.fixture
def cuda_device(monkeypatch):
    return simt_native.install(monkeypatch)


CASES = [
    _c("cost", 6, 7, 127, 2, "scalar"),
    _c("cost", 4, 5, 128, 2, "tensor", zmin=True),
    _c("cost", 6, 3, 129, 2),
    _c("cost", 6, 1, 3, 3, branch="inlier"),
    _c("cost", 4, 129, 2, 2, "scalar", branch="outlier"),
    _c("cost", 4, 9, 0, 2),
    _c("cost", 6, 33, 3, 2, "tensor", zmin=True, blocks=True),
    _c("gn", 6, 129, 1, 3, "scalar", branch="inlier"),
    _c("gn", 6, 40, 1, 3, branch="outlier"),
    _c("gn", 4, 33, 1, 3, "tensor", zmin=True, blocks=True),
    _c("jvp", 6, 20, 63, 2, "scalar", want="cost"),
    _c("jvp", 6, 20, 64, 2, "scalar", want="cost"),
    _c("jvp", 4, 1, 1, 3, branch="outlier", want="all"),
    _c("jvp", 4, 129, 2, 2, branch="inlier", want="all", clip=False),
    _c("jvp", 6, 9, 0, 2, want="all"),
    _c("jvp", 6, 33, 3, 2, "tensor", zmin=True, blocks=True, want="all"),
]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_derivative_matrix(cuda_device, case):
    dm.run_case(case, cuda_device, record=False)


def test_cpu_matrix_keeps_its_boundaries():
    on = lambda entry, key: {cs[key] for cs in CASES if cs["entry"] == entry}
    assert {dm.HVP_POSE_TILE - 1, dm.HVP_POSE_TILE, dm.HVP_POSE_TILE + 1} <= on("cost", "P")
    assert {dm.JVP_POSE_MAJOR_MIN_S - 1, dm.JVP_POSE_MAJOR_MIN_S} <= on("jvp", "P")
    assert {1, dm.NT + 1} <= on("cost", "N") | on("jvp", "N") and dm.NT + 1 in on("gn", "N")
    for entry in ("cost", "gn", "jvp"):
        assert any(cs["blocks"] for cs in CASES if cs["entry"] == entry), entry
        assert {"inlier", "outlier"} <= on(entry, "branch"), entry
    assert "scalar" in {cs["bounds"] for cs in CASES}


def test_objects_are_independent(cuda_device):
    dm.check_object_independence(cuda_device, SIMT_SMS)


def test_largest_point_count(cuda_device):
    dm.check_largest_n(cuda_device)


def _constant(path, name):
    text = open(os.path.join(build.CSRC, path)).read()
    found = re.findall(rf"constexpr int {name} = (\d+);", text)
    assert len(found) == 1, (path, name, found)
    return int(found[0])


def test_the_matrix_mirrors_the_kernels_constants():
    """Retuning a tile or the pose-major switch moves a boundary: the matrix must move with it."""
    assert _constant("pnp_kernels.cu", "HVP_POSE_TILE") == dm.HVP_POSE_TILE
    assert _constant("pnp_kernels.cu", "JVP_POSE_MAJOR_MIN_S") == dm.JVP_POSE_MAJOR_MIN_S
    assert _constant("pnp_device.cuh", "NT") == dm.NT
