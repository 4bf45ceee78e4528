"""The refusals of epnp_gn_plus_hvp_f32 and their precedence, with the machinery of test_capi_refusals_cpu.py: every
case with B = 2 and with B = 0, a refused call and a valid call on an empty batch leaving every buffer as it was.  No
case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK, TOO_MANY_POINTS

NAME = "epnp_gn_plus_hvp_f32"
SIG = (f"{R.PTS} pose* gplus* t_x3d~ t_x2d~ t_w2d~ t_delta~ t_cam~ t_lb~ t_ub~ h_x3d~ h_x2d~ h_w2d~ h_delta~ h_cam~ "
       "h_lb~ h_ub~ h_grad~ B N dof z_min eps huber_eps stream")


def _split_plus(h, name, p, dof, n):
    return h.epnp_max_points_split(dof, 0, 0) + 1


def _resident_plus(h, name, p, dof, n):
    return h.epnp_max_points(dof, 0, 0) + 4


UNBOUNDED = {"lb": None, "ub": None}
# (case, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", {"B": -1}, (BAD_ARG, None)),
    ("N=0", {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("t_lb_without_bounds", dict(UNBOUNDED, h_lb=None, h_ub=None, t_ub=None), (BAD_ARG, BAD_ARG)),
    ("t_ub_without_bounds", dict(UNBOUNDED, h_lb=None, h_ub=None, t_lb=None), (BAD_ARG, BAD_ARG)),
    ("h_lb_without_bounds", dict(UNBOUNDED, t_lb=None, t_ub=None, h_ub=None), (BAD_ARG, BAD_ARG)),
    ("h_ub_without_bounds", dict(UNBOUNDED, t_lb=None, t_ub=None, h_lb=None), (BAD_ARG, BAD_ARG)),
    ("bound_tangent_without_bounds_and_no_gplus", dict(UNBOUNDED, gplus=None, h_lb=None, h_ub=None, t_ub=None),
     (BAD_ARG, BAD_ARG)),
    ("unbounded", dict(UNBOUNDED, t_lb=None, t_ub=None, h_lb=None, h_ub=None), (None, OK)),
    ("N>resident", {"N": _resident_plus}, (None, OK)),          # streams the points: no resident limit
    ("N>split", {"N": _split_plus}, (TOO_MANY_POINTS, OK)),
    ("N>split_unbounded_t_lb", dict(UNBOUNDED, N=_split_plus, h_lb=None, h_ub=None, t_ub=None), (BAD_ARG, BAD_ARG)),
    ("valid", {}, (None, OK)),
]
for _tok in SIG.split():
    if _tok[-1] in "*!":
        CASES.append((f"{_tok[:-1]}=NULL", {_tok[:-1]: None}, (BAD_ARG, BAD_ARG)))
        CASES.append((f"{_tok[:-1]}=NULL_N>split", {_tok[:-1]: None, "N": _split_plus}, (BAD_ARG, BAD_ARG)))


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
