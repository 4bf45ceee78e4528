"""The checks of test_lm_stacked_gpu.py on the CPU: pnp_kernels.cu under the SIMT emulator (tests/simt_native.py), at
sizes the emulator affords.  Every form of lm_stacked_kernel runs: staged with the plain loader (N = 5) and with bulk
copies (N = 64, 640), one warp from global memory (641) and eight warps (2049); S = 1, 3 and 9 (two CTAs of five
hypothesis warps, one idle) or 33 (five CTAs of seven)."""
import pytest

import simt_native
import test_lm_stacked_gpu as _st

case = _st.case
CASES = [
    case(6, 5, 3, 3, "none", "lm"),
    case(4, 5, 33, 2, "scalar", "fast"),
    case(6, 64, 9, 3, "tensor", "lm"),
    case(4, 64, 1, 3, "none", "fast", ("pose_opt",)),
    case(6, 640, 3, 2, "scalar", "fast"),
    case(4, 640, 9, 2, "tensor", "lm", ("pose_opt", "pose_opt_plus")),
    case(6, 641, 3, 2, "tensor", "lm"),
    case(4, 641, 1, 2, "none", "fast"),
    case(6, 2049, 3, 2, "scalar", "lm", ("pose_opt", "cost")),
    case(4, 2049, 3, 1, "tensor", "fast"),
]


@pytest.fixture
def dev(monkeypatch):
    return simt_native.install(monkeypatch)


@pytest.mark.parametrize("c", CASES, ids=[c["id"] for c in CASES])
def test_stacked_equals_per_start_and_flattened(dev, c):
    _st.check_case(dev, c)


@pytest.mark.parametrize("dof,mode", [(6, "lm"), (4, "fast")])
def test_solver_leading_dimensions(dev, dof, mode):
    _st.check_solver_leading_dims(dev, dof=dof, N=32, B=3, mode=mode)


def test_empty_stacks(dev):
    _st.check_empty(dev)


def test_refusals(dev):
    _st.check_refusals(dev)


def test_compile_no_graph_break(dev):
    _st.check_compile(dev)


def test_opcheck(dev):
    _st.check_opcheck(dev)
