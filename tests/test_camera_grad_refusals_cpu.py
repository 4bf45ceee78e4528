"""The refusals of the four camera-gradient entry points and their precedence, with the machinery of
test_capi_refusals_cpu.py: every case with B = 2 and with B = 0, a refused call and a valid call on an empty batch
leaving every buffer as it was.  No case launches a kernel."""
import numpy as np
import pytest

import test_capi_refusals_cpu as R
from test_capi_refusals_cpu import BAD_ARG, OK, TOO_MANY_POINTS, UNSUPPORTED

COST, COST_SPLIT = "epnp_cost_camera_backward_f32", "epnp_cost_camera_backward_split_f32"
GN, GN_SPLIT = "epnp_gn_plus_camera_backward_f32", "epnp_gn_plus_camera_backward_split_f32"
OUT = "gcam~ glb~ gub~"
SIGS = {
    COST: f"{R.PTS} poses_a* grad_a* PA poses_b* grad_b* PB {OUT} B N dof z_min stream",
    COST_SPLIT: f"{R.PTS} poses_a* grad_a* PA poses_b* grad_b* PB {OUT} B N dof z_min cluster_ctas stream",
    GN: f"{R.PTS} pose* gplus* {OUT} B N dof z_min eps huber_eps stream",
    GN_SPLIT: f"{R.PTS} pose* gplus* {OUT} B N dof z_min eps huber_eps cluster_ctas stream",
}
ALL = set(SIGS)
SPLIT = {COST_SPLIT, GN_SPLIT}
NO_BOUNDS = {"lb": None, "ub": None}


def _resident_plus(h, name, p, dof, n):
    return h.epnp_max_points(dof, 0, 0) + 4


# (case, entry points, changes, (rc with B = 2, rc with B = 0))
CASES = [
    ("B<0", ALL, {"B": -1}, (BAD_ARG, None)),
    ("N=0", ALL, {"N": 0}, (BAD_ARG, BAD_ARG)),
    ("dof=5", ALL, {"dof": 5}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", ALL, {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("PA<0", {COST, COST_SPLIT}, {"PA": -1}, (BAD_ARG, BAD_ARG)),
    ("no_output", ALL, {"gcam": None, "glb": None, "gub": None}, (BAD_ARG, BAD_ARG)),
    ("grad_lb_without_bounds", ALL, dict(NO_BOUNDS, gcam=None, gub=None), (BAD_ARG, BAD_ARG)),
    ("grad_ub_without_bounds", ALL, dict(NO_BOUNDS, gcam=None, glb=None), (BAD_ARG, BAD_ARG)),
    ("grad_cam_without_bounds", ALL, dict(NO_BOUNDS, glb=None, gub=None), (None, OK)),
    ("bounds_only", ALL, {"gcam": None}, (None, OK)),
    ("cluster=1", SPLIT, {"cluster_ctas": 1}, (BAD_ARG, BAD_ARG)),
    ("cluster=9", SPLIT, {"cluster_ctas": 9}, (BAD_ARG, BAD_ARG)),
    ("no_cluster_fits", SPLIT, {"env": "0"}, (UNSUPPORTED, OK)),
    ("N>resident", {COST, GN}, {"N": _resident_plus}, (TOO_MANY_POINTS, OK)),
    ("N>split", SPLIT, {"N": R._split_plus}, (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("no_output_N>split", SPLIT, {"gcam": None, "glb": None, "gub": None, "N": R._split_plus}, (BAD_ARG, BAD_ARG)),
    ("valid", ALL, {}, (None, OK)),
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
