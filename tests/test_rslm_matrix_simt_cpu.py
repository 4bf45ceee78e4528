"""The RSLM matrix of test_rslm_matrix_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulators (tests/simt_native.py
for the resident rslm_kernel, tests/simt_cluster_native.py for the split chain rslm_refine_kernel -> cost_split_kernel ->
rslm_select_kernel), held to the same per-hypothesis float64 bounds, tie branches, clamp margins and census, at sizes
the emulators afford.  Kept: a second pass of the thread loop (P = 129), odd N (the last index in the padded end of the
last pair record), minimal and odd subsets, lm_iter = 0, an LM case with tied decisions, bounds and z_min, and a split
case on a cluster of three CTAs."""
import pytest

import simt_cluster_native
import simt_native
import test_rslm_matrix_gpu as _rm

_c = _rm._c

CASES = [
    _c("resident", 6, 33, 129, 3, 2, "fast", 3),
    _c("resident", 4, 33, 64, 9, 2, "lm", 3, outliers=0.1, mixed=True),
    _c("resident", 4, 64, 128, 12, 2, "lm", 3),                     # one hypothesis with a tied decision
    _c("resident", 4, 31, 64, 8, 2, "lm", 0),
    _c("resident", 6, 63, 64, 8, 2, "lm", 3, bounds="tensor", zmin=True),
    _c("resident", 4, 64, 64, 3, 2, "fast", 1, bounds="scalar"),
    _c("split", 6, 47, 64, 7, 2, "fast", 3, ctas=3),
    _c("split", 4, 50, 64, 8, 2, "lm", 3, bounds="scalar", zmin=True, ctas=3),
]


def _install(monkeypatch, case):
    return (simt_native if case["form"] == "resident" else simt_cluster_native).install(monkeypatch)


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_rslm_matrix(monkeypatch, case):
    stats = _rm.run_case(case, _install(monkeypatch, case), record="simt/rslm_matrix")
    if case["id"] == CASES[2]["id"]:
        assert stats["tied_share"] > 0.0


@pytest.mark.parametrize("idx", [0, 6])
def test_object_alone_equals_its_row(monkeypatch, idx):
    _rm.check_exact_properties(CASES[idx], _install(monkeypatch, CASES[idx]))


def test_translation_guess(monkeypatch):
    """t_out against the float64 centre-based guess at an emulator size, one nearly collinear object."""
    dev = simt_native.install(monkeypatch)
    for dof in (6, 4):
        _rm.check_translation_guess(dev, dof, (1001,), record="simt/rslm_matrix")
