"""The cluster-split EPnP initialiser (epnp_epnp_init_split_f32) on the CPU: pnp_kernels.cu under the cluster SIMT
emulator (tests/simt_cluster_native.py).  The cv2 goldens with forced cluster sizes (n_sel exact, poses within
test_epnp_host_cpu.parity's bounds); tied confidences straddling rank boundaries; isolation of NaN and coplanar
objects; w2d = None; the audit build (-DEPNP_SPLIT_AUDIT) checks that every rank ends with rank 0's threshold, n, sums,
control points and candidates and that rank 0 alone stores; results do not depend on the fiber schedule; the argument
checks and refusals; EPnPSolver takes the split call exactly above the resident limit."""
import ctypes
import os

import numpy as np
import pytest
import torch

import simt_cluster_native
import simt_native
from conftest import load_golden
from test_epnp_host_cpu import parity
from epropnp import autograd as ag
from epropnp_b200 import native
from epropnp_b200.synth import make_problem

AUDIT = ("-DEPNP_SPLIT_AUDIT",)


def golden(case, B=None):
    g = load_golden(os.path.join("epnp", case))
    if B is not None:
        g = {k: (v[:B] if np.ndim(v) and k != "q" else v) for k, v in g.items()}
    return g


def tensors(g):
    return tuple(torch.from_numpy(np.ascontiguousarray(g[k])) for k in ("x3d", "x2d", "w2d", "cam_mats"))


def numpy_counts(w2d, q):
    conf = np.asarray(w2d, np.float32).mean(-1)
    return [int((c >= np.quantile(c, np.float32(q))).sum()) for c in conf]


# small: N = 40, at C = 8 ranks 5..7 are empty; select: ties on the threshold, N = 257; cube512: q = 0; camera: fu != fv
@pytest.mark.parametrize("case,B", [("small", None), ("select", None), ("cube512", 4), ("camera", 3)])
@pytest.mark.parametrize("ctas", [2, 3, 8])
def test_split_matches_cv2_golden(monkeypatch, case, B, ctas):
    simt_cluster_native.install(monkeypatch)
    g = golden(case, B)
    pose, n_sel = native.epnp_init_split(*tensors(g), float(g["q"]), want_n_sel=True, cluster_ctas=ctas)
    assert n_sel.tolist() == g["n_sel"].tolist()
    conf = g["w2d"].mean(-1)
    parity(pose.numpy(), g, [c >= np.quantile(c, g["q"]) for c in conf])


def _tied_at_rank_boundaries(N, seed=3):
    """Confidences on a coarse grid, with runs of the q = 0.8 threshold value around every rank boundary of every C."""
    pc = make_problem(2, N, seed=seed)
    rng = np.random.default_rng(seed)
    conf = (rng.integers(1, 12, size=(2, N)) / 4.0).astype(np.float32)
    for b in range(2):
        thr = np.float32(np.quantile(conf[b], np.float32(0.8)))
        for C in range(2, 9):
            share = ((N + C - 1) // C + 7) // 8 * 8
            for r in range(1, C):
                conf[b, max(0, r * share - 2):min(N, r * share + 2)] = thr
    pc["w2d"] = torch.from_numpy(np.repeat(conf[..., None], 2, axis=-1))
    return pc


def test_ties_straddling_rank_boundaries(monkeypatch):
    simt_cluster_native.install(monkeypatch)
    pc = _tied_at_rank_boundaries(203)
    t = (pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"])
    want = numpy_counts(pc["w2d"].numpy(), 0.8)
    res, n_res = native.epnp_init(*t, 0.8, want_n_sel=True)
    assert n_res.tolist() == want
    for ctas in range(2, 9):
        pose, n = native.epnp_init_split(*t, 0.8, want_n_sel=True, cluster_ctas=ctas)
        assert n.tolist() == want, ctas
        assert torch.isfinite(pose).all()
        assert float((pose - res).abs().max()) < 1e-4 * float(res.abs().max()), ctas


def test_bad_objects_leave_the_others_unchanged(monkeypatch):
    simt_cluster_native.install(monkeypatch)
    x3d, x2d, w2d, cam = tensors(golden("outliers", 4))
    base, n0 = native.epnp_init_split(x3d, x2d, w2d, cam, 0.8, want_n_sel=True, cluster_ctas=3)
    x3d2, w2d2 = x3d.clone(), w2d.clone()
    x3d2[1, :, 2] = 0.0                                        # object 1: coplanar points
    w2d2[2, 400, 1] = float("nan")                             # object 2: a NaN confidence, in the last rank's range
    pose, n = native.epnp_init_split(x3d2, x2d, w2d2, cam, 0.8, want_n_sel=True, cluster_ctas=3)
    keep = [0, 3]
    assert torch.equal(pose[keep], base[keep]) and torch.equal(n[keep], n0[keep])
    assert torch.isnan(pose[2]).all() and int(n[2]) == 0
    assert int(n[1]) == int(n0[1])                             # the selection does not look at x3d


def test_no_weights_keeps_every_point(monkeypatch):
    simt_cluster_native.install(monkeypatch)
    x3d, x2d, w2d, cam = tensors(golden("cube512", 2))
    all_pts, n = native.epnp_init_split(x3d, x2d, None, cam, 0.8, want_n_sel=True, cluster_ctas=3)
    assert n.tolist() == [512, 512]
    assert torch.equal(all_pts, native.epnp_init_split(x3d, x2d, w2d, cam, 0.0, cluster_ctas=3))
    res = native.epnp_init(x3d, x2d, None, cam, 0.8)
    assert float((all_pts - res).abs().max()) < 1e-4 * float(res.abs().max())


def _points_of_rank(N, ctas):
    share = ((N + ctas - 1) // ctas + 7) // 8 * 8
    return [max(0, min(N, (r + 1) * share) - min(N, r * share)) for r in range(8)]


@pytest.mark.parametrize("case,ctas", [("small", 8), ("select", 3), ("cube512", 5)])
def test_ranks_agree_and_rank_zero_alone_stores(monkeypatch, case, ctas):
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    g = golden(case, 3)
    x3d, x2d, w2d, cam = tensors(g)
    w2d[2, 0, 0] = float("nan")                                # the NaN path: still rank 0 alone
    counts = (ctypes.c_longlong * 16)()
    for want_n_sel in (False, True):
        lib.simt_audit_reset()
        out = native.epnp_init_split(x3d, x2d, w2d, cam, float(g["q"]), want_n_sel=want_n_sel, cluster_ctas=ctas)
        lib.simt_audit_read(counts)
        stores, mismatches = list(counts)[:8], list(counts)[8:]
        assert mismatches == [0] * 8                           # threshold, n, sums, control points, candidates
        assert stores == [3 * (8 if want_n_sel else 7)] + [0] * 7, stores
    assert out[1].tolist()[:2] == g["n_sel"].tolist()[:2]
    if case == "small":
        assert _points_of_rank(40, 8)[5:] == [0, 0, 0]         # the case has empty ranks


def test_split_results_do_not_depend_on_fiber_schedule(monkeypatch):
    """Ascending, descending and random fiber orders across the whole cluster give the same bits: no rank reads another
    rank's counts or partial sums without the cluster barrier in between."""
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    t = tensors(golden("select", 2))
    try:
        lib.simt_set_schedule(0, 1)
        base = native.epnp_init_split(*t, 0.8, want_n_sel=True, cluster_ctas=3)
        for mode, seed in ((1, 1), (2, 5)):
            lib.simt_set_schedule(mode, seed)
            lib.simt_audit_reset()
            out = native.epnp_init_split(*t, 0.8, want_n_sel=True, cluster_ctas=3)
            counts = (ctypes.c_longlong * 16)()
            lib.simt_audit_read(counts)
            assert list(counts)[8:] == [0] * 8
            assert torch.equal(out[0], base[0]) and torch.equal(out[1], base[1]), mode
    finally:
        lib.simt_set_schedule(0, 1)


def test_arguments_and_refusals(monkeypatch):
    """A cluster size outside [minimum, 8] is a bad argument; a device that cannot co-schedule the cluster is refused
    before any launch; B = 0 launches nothing; the resident call's argument checks apply."""
    simt_cluster_native.install(monkeypatch)
    lib = simt_cluster_native.handle()
    x3d, x2d, w2d, cam = tensors(golden("small", 2))
    for bad in (1, 9, -1):
        with pytest.raises(native.NativeError, match="bad argument"):
            native.epnp_init_split(x3d, x2d, w2d, cam, 0.8, cluster_ctas=bad)
    with pytest.raises(native.NativeError, match="bad argument"):
        native.epnp_init_split(x3d, x2d, w2d, cam, 1.5)
    with pytest.raises(native.NativeError, match="bad argument"):        # 20 points at q = 0.9 keep at most 2
        native.epnp_init_split(x3d[:, :20], x2d[:, :20], w2d[:, :20], cam, 0.9)
    assert native.epnp_init_split(x3d[:0], x2d[:0], w2d[:0], cam[:0], 0.8).shape == (0, 7)

    def raw(B, ctas):      # pointers that would fault if anything read them: B = 0 must return before any launch
        one = ctypes.c_void_p(16)
        return lib.epnp_epnp_init_split_f32(one, one, one, one, ctypes.c_float(0.8), one, None, B, 40, ctas, None)
    assert raw(0, 0) == 0 and raw(0, 9) == -1
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "0")
    with pytest.raises(native.NativeError, match="not supported"):
        native.epnp_init_split(x3d, x2d, w2d, cam, 0.8)
    assert raw(0, 0) == 0


def test_single_cta_emulator_refuses_split_call(monkeypatch):
    """The single-CTA emulator build cannot run a cluster: the split call reports EPNP_ERR_UNSUPPORTED after its argument
    checks, as a device without cluster support does."""
    simt_native.install(monkeypatch)
    x3d, x2d, w2d, cam = tensors(golden("small", 2))
    with pytest.raises(native.NativeError, match="not supported"):
        native.epnp_init_split(x3d, x2d, w2d, cam, 0.8)
    with pytest.raises(native.NativeError, match="bad argument"):
        native.epnp_init_split(x3d, x2d, w2d, cam, 0.8, cluster_ctas=9)


@pytest.mark.parametrize("limit", [0, 10 ** 6])
def test_epnp_solver_takes_the_split_call_exactly_above_the_resident_limit(monkeypatch, limit):
    """EPnPSolver under LMSolver, with pose_init = None and with force_init_solve and a pose_init: the EPnP call and the
    cost of its pose go through the split kernels exactly when N exceeds the resident limit; the solve stays within
    1e-4 of the one started from cv2's pose."""
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epnp import EPnPSolver
    from epropnp.levenberg_marquardt import LMSolver
    simt_cluster_native.install(monkeypatch)
    calls = []
    for name in ("epnp_init", "epnp_init_split", "evaluate_cost", "evaluate_cost_split"):
        fn = getattr(native, name)
        monkeypatch.setattr(native, name, lambda *a, _fn=fn, _n=name, **k: calls.append(_n) or _fn(*a, **k))
    monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i: limit)
    g = golden("small", 4)
    x3d, x2d, w2d, cam = tensors(g)
    camera = PerspectiveCamera(cam_mats=cam, z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(x2d, w2d)
    solver = LMSolver(6, 3, init_solver=EPnPSolver(0.8))
    pose = solver(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]
    split = limit == 0
    assert calls == ["epnp_init_split" if split else "epnp_init"]
    ref = LMSolver(6, 3)(x3d, x2d, w2d, camera, cost_fun, pose_init=torch.from_numpy(g["pose"]).float(), fast_mode=True)[0]
    assert float((pose - ref).abs().max() / ref.abs().max()) < 1e-4
    calls.clear()
    solver(x3d, x2d, w2d, camera, cost_fun, pose_init=torch.from_numpy(g["pose"]).float(), force_init_solve=True,
           fast_mode=True)
    assert set(calls) == ({"epnp_init_split", "evaluate_cost_split"} if split else {"epnp_init", "evaluate_cost"})


def test_bench_configs_split_section_runs_in_toy_mode(monkeypatch, capsys):
    import importlib.util
    import json
    from conftest import ROOT
    from test_bench_dryrun_cpu import _Event
    simt_cluster_native.install(monkeypatch)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    for k in ("EPNP_BENCH_CONFIGS_TOY", "EPNP_BENCH_SPLIT"):
        monkeypatch.setenv(k, "1")
    for k in ("EPNP_BENCH_EPNP", "EPNP_BENCH_RSLM", "EPNP_BENCH_GN_PLUS", "EPNP_BENCH_MC_EPILOGUE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("EPNP_BENCH_DEVICE", "cpu")
    spec = importlib.util.spec_from_file_location("bench_configs_split", os.path.join(ROOT, "tools", "bench_configs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    monkeypatch.setattr(ag, "_resident_limit", lambda dof, m, i: 0)      # toy N: make LMSolver take the split EPnP
    mod.main()
    rows = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    ep = [r for r in rows if "EPnP" in r["config"]]
    assert len(ep) == 2 and "ms_epnp_split" in ep[0] and "ms_resident" in ep[1]
    assert all(v > 0 for r in rows for k, v in r.items() if k.startswith("ms"))
