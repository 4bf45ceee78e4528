"""epnp_init_kernel itself (radix select, compaction, fp64 block reductions, barriers) executed under the SIMT emulator
(tests/simt_native.py) at small B and N: native.epnp_init and EPnPSolver under LMSolver against the cv2 goldens, and
the EPnP section of tools/bench_configs.py at toy size."""
import json
import os

import numpy as np
import pytest
import torch

import simt_native
from conftest import ROOT, load_golden
from test_epnp_host_cpu import parity


def golden(case, B=None):
    g = load_golden(os.path.join("epnp", case))
    if B is not None:
        g = {k: (v[:B] if np.ndim(v) and k != "q" else v) for k, v in g.items()}
    return g


@pytest.mark.parametrize("case,B", [("small", None), ("select", None), ("camera", 3), ("outliers", 4), ("dense", 2)])
def test_kernel_matches_cv2_golden(monkeypatch, case, B):
    from epropnp_b200 import native
    simt_native.install(monkeypatch)
    g = golden(case, B)
    t = {k: torch.from_numpy(g[k]) for k in ("x3d", "x2d", "w2d", "cam_mats")}
    pose, n_sel = native.epnp_init(t["x3d"], t["x2d"], t["w2d"], t["cam_mats"], float(g["q"]), want_n_sel=True)
    assert n_sel.tolist() == g["n_sel"].tolist()
    conf = g["w2d"].mean(-1)
    masks = [c >= np.quantile(c, g["q"]) for c in conf]
    parity(pose.numpy(), g, masks)


def test_schedule_order_does_not_change_the_result(monkeypatch):
    import ctypes
    from epropnp_b200 import native
    simt_native.install(monkeypatch)
    g = golden("select", 2)
    t = [torch.from_numpy(g[k]) for k in ("x3d", "x2d", "w2d", "cam_mats")]
    h = simt_native.handle(())
    h.simt_set_schedule.argtypes = [ctypes.c_int, ctypes.c_ulonglong]
    runs = []
    try:
        for mode in (0, 1, 2):
            h.simt_set_schedule(mode, 7)
            runs.append(native.epnp_init(*t, float(g["q"])))
    finally:
        h.simt_set_schedule(0, 1)
    assert all(torch.equal(runs[0], r) for r in runs[1:])


def test_no_weights_nan_and_refusals(monkeypatch):
    from epropnp_b200 import native
    simt_native.install(monkeypatch)
    g = golden("cube512", 2)
    x3d, x2d, w2d, cam = (torch.from_numpy(g[k]) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    all_pts = native.epnp_init(x3d, x2d, None, cam, 0.8)         # no weights: every point, q unused
    q0 = native.epnp_init(x3d, x2d, w2d, cam, 0.0)
    assert torch.equal(all_pts, q0)
    w = w2d.clone()
    w[1, 5, 0] = float("nan")
    pose, n = native.epnp_init(x3d, x2d, w, cam, 0.8, want_n_sel=True)
    conf0 = g["w2d"][0].mean(-1)
    assert n.tolist() == [int((conf0 >= np.quantile(conf0, np.float32(0.8))).sum()), 0]
    assert torch.isnan(pose[1]).all() and torch.equal(pose[0], native.epnp_init(x3d[:1], x2d[:1], w2d[:1], cam[:1], 0.8)[0])
    assert native.epnp_init(x3d[:0], x2d[:0], w2d[:0], cam[:0], 0.8).shape == (0, 7)
    with pytest.raises(native.NativeError):
        native.epnp_init(x3d[:, :20], x2d[:, :20], w2d[:, :20], cam, 0.9)        # at most 2 points kept
    with pytest.raises(native.NativeError):
        native.epnp_init(x3d, x2d, w2d, cam, 1.5)


def test_epnp_solver_under_lmsolver(monkeypatch):
    from epropnp.camera import PerspectiveCamera
    from epropnp.cost_fun import AdaptiveHuberPnPCost
    from epropnp.epnp import EPnPSolver
    from epropnp.levenberg_marquardt import LMSolver
    simt_native.install(monkeypatch)
    g = golden("small")
    x3d, x2d, w2d, cam = (torch.from_numpy(g[k]) for k in ("x3d", "x2d", "w2d", "cam_mats"))
    camera = PerspectiveCamera(cam_mats=cam, z_min=0.01)
    cost_fun = AdaptiveHuberPnPCost(relative_delta=0.1)
    cost_fun.set_param(x2d, w2d)
    pose = LMSolver(6, 3, init_solver=EPnPSolver(0.8))(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)[0]
    ref = LMSolver(6, 3)(x3d, x2d, w2d, camera, cost_fun, pose_init=torch.from_numpy(g["pose"]).float(), fast_mode=True)[0]
    scale = ref.abs().max()
    assert float((pose - ref).abs().max() / scale) < 1e-4
    with pytest.raises(ValueError):
        LMSolver(4, 3, init_solver=EPnPSolver())(x3d, x2d, w2d, camera, cost_fun, fast_mode=True)


def test_bench_configs_epnp_section_runs_in_toy_mode(monkeypatch, capsys):
    import importlib.util
    from test_bench_dryrun_cpu import _Event
    simt_native.install(monkeypatch)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    for k in ("EPNP_BENCH_CONFIGS_TOY", "EPNP_BENCH_EPNP"):
        monkeypatch.setenv(k, "1")
    for k in ("EPNP_BENCH_RSLM", "EPNP_BENCH_GN_PLUS", "EPNP_BENCH_MC_EPILOGUE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("EPNP_BENCH_DEVICE", "cpu")
    spec = importlib.util.spec_from_file_location("bench_configs_epnp", os.path.join(ROOT, "tools", "bench_configs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.main()
    rows = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    ep = [r for r in rows if r["config"].startswith("6DoF test-time path")]
    assert ep and all("ms_epnp" in r and "ms_epnp_gn3" in r for r in ep)
    assert all(v > 0 for r in rows for k, v in r.items() if k.startswith("ms"))
