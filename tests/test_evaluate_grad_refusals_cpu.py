"""The refusals of epnp_evaluate_backward_f32 and their precedence, with the machinery of test_capi_refusals_cpu.py:
every case with B = 2 and with B = 0, a refused call and a valid call on an empty batch leaving every buffer as it was.
No case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK

NAME = "epnp_evaluate_backward_f32"
UPS = "g_res~ g_jac~ g_cost~"
OUT = "gx3d~ gx2d~ gw2d~ gdelta~ gpose~ gcam~ glb~ gub~"
SIG = f"{R.PTS} poses* {UPS} {OUT} clip_jac S B N dof z_min huber_eps stream"
NO_UPS = {"g_res": None, "g_jac": None, "g_cost": None}
NO_OUT = {k.rstrip("~"): None for k in OUT.split()}
NO_BOUNDS = {"lb": None, "ub": None}

# (case, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", {"B": -1}, (BAD_ARG, None)),
    ("N=0", {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("S<0", {"S": -1}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("x3d=NULL", {"x3d": None}, (BAD_ARG, BAD_ARG)),
    ("delta=NULL", {"delta": None}, (BAD_ARG, BAD_ARG)),
    ("poses=NULL", {"poses": None}, (BAD_ARG, BAD_ARG)),
    ("no_upstream", NO_UPS, (BAD_ARG, BAD_ARG)),
    ("no_output", NO_OUT, (BAD_ARG, BAD_ARG)),
    ("no_upstream_no_output", dict(NO_UPS, **NO_OUT), (BAD_ARG, BAD_ARG)),
    ("grad_lb_without_bounds", dict(NO_OUT, glb=0, **NO_BOUNDS), (BAD_ARG, BAD_ARG)),
    ("grad_ub_without_bounds", dict(NO_OUT, gub=0, **NO_BOUNDS), (BAD_ARG, BAD_ARG)),
    ("no_upstream_S=0", dict(NO_UPS, S=0), (BAD_ARG, BAD_ARG)),
    ("no_output_N=0", dict(NO_OUT, N=0), (BAD_ARG, BAD_ARG)),
    ("one_upstream", {"g_res": None, "g_jac": None}, (None, OK)),
    ("pose_only", dict(NO_OUT, gpose=0), (None, OK)),
    ("cam_without_bounds", dict(NO_OUT, gcam=0, **NO_BOUNDS), (None, OK)),
    ("S=0", {"S": 0}, (OK, OK)),
    ("valid", {}, (None, OK)),
]


def _ids():
    for case, changes, (rc_b, rc_0) in CASES:
        changes = {k: v for k, v in changes.items() if v != 0 or k in ("S", "N")}     # 0: keep that buffer
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
