"""The backward matrix of test_backward_matrix_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulator
(tests/simt_native.py), held to the same per-object float64 bounds, at sizes the emulator affords.  The boundaries stay:
N = 513 (a second, partial point tile), P = 1025 (a second pose tile) and, on an emulated one-SM device
(SIMT_EMUL_SMS=1, a grid of 4 CTAs), batches whose objects share CTAs."""
import pytest

import simt_native
import test_backward_matrix_gpu as _bm

SIMT_GRID = 4           # 4 CTAs per SM on the one-SM device


@pytest.fixture
def cuda_device(monkeypatch):
    monkeypatch.setenv("SIMT_EMUL_SMS", "1")
    monkeypatch.setattr(_bm, "resident_grid", lambda dev: SIMT_GRID)
    return simt_native.install(monkeypatch)


CASES = [
    dict(id="d6_N1_P01_B1", dof=6, bounds=None, N=1, PA=0, PB=1, B=(0, 1)),
    dict(id="d6_tensor_N513_P3_2Gp3", dof=6, bounds="tensor", N=513, PA=2, PB=1, B=(2, 3), outliers=0.1,
         beyond_grid=True),
    dict(id="d6_tensor_N7_P1025_Gp1", dof=6, bounds="tensor", N=7, PA=1024, PB=1, B=(1, 1), outliers=0.1,
         many_pose_tiles=True, beyond_grid=True),
    dict(id="d4_scalar_N40_P1025_B1", dof=4, bounds="scalar", N=40, PA=1024, PB=1, B=(0, 1), many_pose_tiles=True),
    dict(id="d4_zmin_N513_P2_Gp1", dof=4, bounds=None, N=513, PA=1, PB=1, B=(1, 1), zmin=True, outliers=0.1,
         beyond_grid=True),
    dict(id="d6_zmin_tensor_N128_P8_G", dof=6, bounds="tensor", N=128, PA=8, PB=0, B=(1, 0), zmin=True),
]
PROPS = dict(id="props", dof=6, bounds="tensor", N=513, PA=2, PB=1, B=(2, 3), outliers=0.1)
GN_CASES = [c for c in _bm.GN_CASES if c["id"] in ("d6_N5_outlier", "d6_N129_bounded_outliers", "d4_N129_zmin",
                                                    "d6_N512_zmin_bounded")]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_cost_backward_matrix(cuda_device, case):
    _bm.test_cost_backward_matrix(cuda_device, case)


def test_cost_backward_exact_properties(cuda_device, monkeypatch):
    monkeypatch.setattr(_bm, "PROP_CASE", PROPS)
    _bm.test_cost_backward_exact_properties(cuda_device)


@pytest.mark.parametrize("case", GN_CASES, ids=[c["id"] for c in GN_CASES])
def test_gn_plus_backward_matrix(cuda_device, case):
    _bm.test_gn_plus_backward_matrix(cuda_device, case)


@pytest.mark.parametrize("dof", [6, 4])
def test_training_step(cuda_device, monkeypatch, dof):
    """B = 9 objects on a grid of 4 CTAs (objects 0, 4, 8 on one CTA), N = 130, M = 64, I = 4."""
    _bm.check_train_step(cuda_device, monkeypatch, dof, 9, 130, 64, 4, f"simt/train/{dof}dof")


def test_training_step_with_pose_opt_plus(cuda_device, monkeypatch):
    _bm.check_pose_opt_plus(cuda_device, monkeypatch, 6, 130, 64, 4)
