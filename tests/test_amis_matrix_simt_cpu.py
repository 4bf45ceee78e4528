"""The AMIS matrix of test_amis_matrix_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulators (tests/simt_native.py
for the resident kernels, tests/simt_cluster_native.py for the cluster-split one), held to the same per-object float64
bounds and census, at sizes the emulators afford.  Both resident forms stay: the 128-thread kernel at S = 8, 127, 128
and 129 (one and two draw passes), I = 1 and I = 8, and the 512-thread kernel at N = 2050, whose 1025 point pairs do not
split into four ranges of whole multiples of four."""
import pytest

import simt_cluster_native
import simt_native
import test_amis_matrix_gpu as _am

_c = _am._c

CASES = [
    _c("resident", 6, 3, 8, 1, 3),
    _c("resident", 6, 7, 64, 8, 2, bounds="scalar"),
    _c("resident", 6, 127, 508, 4, 2, bounds="tensor"),
    _c("resident", 6, 128, 512, 4, 2, zmin=True),
    _c("resident", 6, 129, 516, 4, 2, outliers=0.1),
    _c("resident", 6, 513, 516, 4, 3, zmin=True, mixed=True),
    _c("resident", 6, 2050, 132, 4, 2, bounds="tensor"),
    _c("resident", 4, 129, 1032, 8, 2, outliers=0.1),
    _c("resident", 6, 128, 256, 4, 2, collapse=True),
    # (seed 1 draws at iteration 1 a rotation sample whose noise lies along a short axis of L_r: the draw magnifies
    # L_r's rounding a hundredfold there, and that sample's log-weight carries it past 10 x floor in either direction)
    _c("split", 6, 50, 64, 4, 2, bounds="tensor", ctas=3, seed=2),
    _c("split", 4, 37, 64, 2, 2, zmin=True, ctas=5),
]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_amis_matrix(monkeypatch, case):
    dev = (simt_native if case["form"] == "resident" else simt_cluster_native).install(monkeypatch)
    _am.run_case(case, dev, record="simt/amis_matrix")


def test_object_alone_equals_its_row(monkeypatch):
    dev = simt_native.install(monkeypatch)
    case = CASES[4]
    c = _am.build_case(case, dev)
    full = _am.run_kernel(c, case)
    one = _am.run_kernel(c, case, slice(1, 2))
    for k in ("samples", "logw", "proposals"):
        assert (one[k][0] == full[k][1]).all(), k
