"""The refusals of epnp_cost_pose_backward_f32 and epnp_cost_pose_backward_split_f32, and their precedence, with the
machinery of test_capi_refusals_cpu.py: every case with B = 2 and with B = 0, a refused call and a valid call on an empty
batch leaving every buffer as it was.  No case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK, TOO_MANY_POINTS, UNSUPPORTED

RESIDENT, SPLIT = "epnp_cost_pose_backward_f32", "epnp_cost_pose_backward_split_f32"
SIGS = {
    RESIDENT: f"{R.PTS} poses* grad* grad_pose! PA B N dof z_min stream",
    SPLIT: f"{R.PTS} poses* grad* grad_pose! PA B N dof z_min cluster_ctas stream",
}
BOTH = {RESIDENT, SPLIT}


def _resident_plus(h, name, p, dof, n):
    return h.epnp_max_points(dof, 0, 0) + 4


# (case, entry points, changes, (rc with B = 2, rc with B = 0)); PA is the number of poses per object (the P argument)
CASES = [
    ("B<0", BOTH, {"B": -1}, (BAD_ARG, None)),
    ("N=0", BOTH, {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", BOTH, {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", BOTH, {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("P<0", BOTH, {"PA": -1}, (BAD_ARG, BAD_ARG)),
    ("P=0", BOTH, {"PA": 0}, (OK, OK)),
    ("cluster=1", {SPLIT}, {"cluster_ctas": 1}, (BAD_ARG, BAD_ARG)),
    ("cluster=9", {SPLIT}, {"cluster_ctas": 9}, (BAD_ARG, BAD_ARG)),
    ("no_cluster_fits", {SPLIT}, {"env": "0"}, (UNSUPPORTED, OK)),
    ("N>resident", {RESIDENT}, {"N": _resident_plus}, (TOO_MANY_POINTS, OK)),
    ("N>split", {SPLIT}, {"N": R._split_plus}, (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("P=0_N>split", {SPLIT}, {"PA": 0, "N": R._split_plus}, (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("valid", BOTH, {}, (None, OK)),
]
for _name, _sig in SIGS.items():
    for _tok in _sig.split():
        if _tok[-1] in "*!":
            CASES.append((f"{_tok[:-1]}=NULL", {_name}, {_tok[:-1]: None}, (BAD_ARG, BAD_ARG)))


def _ids():
    for case, entries, changes, (rc_b, rc_0) in CASES:
        for name in sorted(entries):
            for B, rc in ((changes.get("B", 2), rc_b), (0, rc_0)):
                if rc is not None:
                    yield pytest.param(name, changes, B, rc, id=f"{name}-{case}-B{B}")


@pytest.mark.parametrize("name,changes,B,expected", list(_ids()))
def test_refusal_and_its_precedence(monkeypatch, name, changes, B, expected):
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "16")
    for k, v in SIGS.items():
        monkeypatch.setitem(R.SIGS, k, v)
    rc, buffers = R._call(name, changes, B, monkeypatch)
    assert rc == expected, (name, changes, B, rc)
    for arg, (a, before) in buffers.items():
        assert np.array_equal(a, before), f"{name} wrote {arg}"
