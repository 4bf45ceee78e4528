"""The refusals of epnp_lm_solve_stacked_f32 and their precedence, with the machinery of test_capi_refusals_cpu.py: every
case with B = 2 and with B = 0, a refused call and a valid call on an empty batch or an empty stack leaving every buffer
as it was.  No case launches a kernel.  Also native.lm_solve_stacked's shape checks."""
import numpy as np
import pytest
import torch

import simt_native
import test_capi_refusals_cpu as R
from epropnp_b200 import native
from test_capi_refusals_cpu import BAD_ARG, FAST0, OK

NAME = "epnp_lm_solve_stacked_f32"
SIG = f"{R.PTS} pose_init* pose_opt! pose_cov~ cost~ pose_plus~ cost_init~ S B N params stream"
OPTIONAL_OUT = ("pose_cov", "cost", "pose_plus", "cost_init")
ONLY = lambda *keep: {k: None for k in OPTIONAL_OUT if k not in keep}

# (case, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", {"B": -1}, (BAD_ARG, None)),
    ("N=0", {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("lm_iter<0", {"p.lm_iter": -1}, (BAD_ARG, BAD_ARG)),
    ("S<0", {"S": -1}, (BAD_ARG, BAD_ARG)),
    ("S*B_over_int", {"S": 1 << 30}, (BAD_ARG, None)),
    ("lb_without_ub", {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("x3d=NULL", {"x3d": None}, (BAD_ARG, BAD_ARG)),
    ("x2d=NULL", {"x2d": None}, (BAD_ARG, BAD_ARG)),
    ("w2d=NULL", {"w2d": None}, (BAD_ARG, BAD_ARG)),
    ("cam=NULL", {"cam": None}, (BAD_ARG, BAD_ARG)),
    ("delta=NULL", {"delta": None}, (BAD_ARG, BAD_ARG)),
    ("pose_init=NULL", {"pose_init": None}, (BAD_ARG, BAD_ARG)),
    ("pose_init=NULL_S=0", {"pose_init": None, "S": 0}, (BAD_ARG, BAD_ARG)),
    ("pose_opt=NULL", {"pose_opt": None}, (BAD_ARG, BAD_ARG)),
    # fast mode with no Gauss-Newton step has no covariance, cost or cost_init to return
    ("fast_no_steps_all_outputs", FAST0, (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_cov", dict(FAST0, **ONLY("pose_cov")), (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_cost", dict(FAST0, **ONLY("cost")), (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_cost_init", dict(FAST0, **ONLY("cost_init")), (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_cost_S=0", dict(FAST0, S=0, **ONLY("cost")), (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_pose_only", dict(FAST0, **ONLY("pose_plus")), (None, OK)),
    ("unbounded", {"lb": None, "ub": None}, (None, OK)),
    ("S=0", {"S": 0}, (OK, OK)),
    ("valid", {}, (None, OK)),
]


def _ids():
    for case, changes, (rc_b, rc_0) in CASES:
        for B, rc in ((changes.get("B", 2), rc_b), (0, rc_0)):
            if rc is not None:
                yield pytest.param(changes, B, rc, id=f"{case}-B{B}")


@pytest.mark.parametrize("changes,B,expected", list(_ids()))
def test_refusal_and_its_precedence(monkeypatch, changes, B, expected):
    monkeypatch.setitem(R.SIGS, NAME, SIG)
    rc, buffers = R._call(NAME, changes, B, monkeypatch)
    assert rc == expected, (changes, B, rc)
    for arg, (a, before) in buffers.items():
        assert np.array_equal(a, before), f"{NAME} wrote {arg}"


@pytest.mark.parametrize("shape,what", [((2, 3, 7), "pose_init must be"), ((3, 7), "pose_init must be"),
                                        ((2, 2, 3, 7), "pose_init must be"), ((2, 3, 4), "pose_init must be")])
def test_native_shape_checks(monkeypatch, shape, what):
    """native.lm_solve_stacked takes (S, B, D) only: another B, a (B, D) pose, extra leading dimensions (the layer
    flattens those) and a pose of the wrong width are refused before the library is called."""
    simt_native.install(monkeypatch)
    B, N = 2, 8
    z = lambda *s: torch.zeros(s)
    prob = native.Problem(z(B, N, 3), z(B, N, 2), z(B, N, 2), torch.eye(3).expand(B, 3, 3), None, None, 1.0)
    with pytest.raises(ValueError, match=what):
        native.lm_solve_stacked(prob, z(*shape), native.default_params(6))
    with pytest.raises(ValueError, match="needs pose_init"):
        native.lm_solve_stacked(prob, None, native.default_params(6))
