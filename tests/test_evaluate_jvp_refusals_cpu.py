"""The refusals of epnp_evaluate_jvp_f32 and their precedence, with the machinery of test_capi_refusals_cpu.py: every
case with B = 2 and with B = 0, a refused call and a valid call on an empty batch leaving every buffer as it was.  No
case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK

NAME = "epnp_evaluate_jvp_f32"
TAN = "t_x3d~ t_x2d~ t_w2d~ t_delta~ t_pose~ t_cam~ t_lb~ t_ub~"
OUT = "d_res~ d_jac~ d_cost~"
SIG = f"{R.PTS} poses* {TAN} {OUT} clip_jac S B N dof z_min huber_eps stream"
NO_OUT = {k.rstrip("~"): None for k in OUT.split()}
NO_TAN = {k.rstrip("~"): None for k in TAN.split()}
NO_BOUNDS = {"lb": None, "ub": None}

# (case, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", {"B": -1}, (BAD_ARG, None)),
    ("N=0", {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("S<0", {"S": -1}, (BAD_ARG, BAD_ARG)),
    ("S*B_over_int", {"S": 1 << 30}, (BAD_ARG, None)),
    ("lb_without_ub", {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("x3d=NULL", {"x3d": None}, (BAD_ARG, BAD_ARG)),
    ("delta=NULL", {"delta": None}, (BAD_ARG, BAD_ARG)),
    ("poses=NULL", {"poses": None}, (BAD_ARG, BAD_ARG)),
    ("no_output", NO_OUT, (BAD_ARG, BAD_ARG)),
    ("no_output_S=0", dict(NO_OUT, S=0), (BAD_ARG, BAD_ARG)),
    ("t_lb_without_bounds", dict(NO_BOUNDS, t_ub=None), (BAD_ARG, BAD_ARG)),
    ("t_ub_without_bounds", dict(NO_BOUNDS, t_lb=None), (BAD_ARG, BAD_ARG)),
    ("unbounded", dict(NO_BOUNDS, t_lb=None, t_ub=None), (None, OK)),
    ("no_tangent", NO_TAN, (None, OK)),
    ("cost_only", {"d_res": None, "d_jac": None}, (None, OK)),
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
