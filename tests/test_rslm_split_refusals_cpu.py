"""The refusals of epnp_rslm_split_f32, and their precedence, with the machinery of test_capi_refusals_cpu.py: epnp_rslm_f32's
refusals, then those of epnp_evaluate_cost_split_f32; every case with B = 2 and with B = 0, a refused call and a valid
call on an empty batch leaving every buffer as it was.  No case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK, TOO_MANY_POINTS, UNSUPPORTED

NAME = "epnp_rslm_split_f32"
SIG = f"{R.PTS} inds* start* pose_best! cost_best! pose_all! cost_all! P n B N params cluster_ctas stream"

# (case, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", {"B": -1}, (BAD_ARG, None)),
    ("N=0", {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("lm_iter<0", {"p.lm_iter": -1}, (BAD_ARG, BAD_ARG)),
    ("P=0", {"P": 0}, (BAD_ARG, BAD_ARG)),
    ("n=0", {"n": 0}, (BAD_ARG, BAD_ARG)),
    ("cluster=1", {"cluster_ctas": 1}, (BAD_ARG, BAD_ARG)),
    ("cluster=9", {"cluster_ctas": 9}, (BAD_ARG, BAD_ARG)),
    ("no_cluster_fits", {"env": "0"}, (UNSUPPORTED, OK)),
    ("N>split", {"N": R._split_plus}, (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("n=0_N>split", {"n": 0, "N": R._split_plus}, (BAD_ARG, BAD_ARG)),
    ("valid", {}, (None, OK)),
]
for _tok in SIG.split():
    if _tok[-1] in "*!":
        CASES.append((f"{_tok[:-1]}=NULL", {_tok[:-1]: None}, (BAD_ARG, BAD_ARG)))


def _ids():
    for case, changes, (rc_b, rc_0) in CASES:
        for B, rc in ((changes.get("B", 2), rc_b), (0, rc_0)):
            if rc is not None:
                yield pytest.param(changes, B, rc, id=f"{case}-B{B}")


@pytest.mark.parametrize("changes,B,expected", list(_ids()))
def test_refusal_and_its_precedence(monkeypatch, changes, B, expected):
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "16")
    monkeypatch.setitem(R.SIGS, NAME, SIG)
    rc, buffers = R._call(NAME, changes, B, monkeypatch)
    assert rc == expected, (changes, B, rc)
    for arg, (a, before) in buffers.items():
        assert np.array_equal(a, before), f"{NAME} wrote {arg}"
