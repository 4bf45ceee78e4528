"""The host-buffer solve from a given pose or from scratch (epnp_solve_host_f32, epnp_solve_split_host_f32) on the CPU,
under the SIMT emulators (tests/simt_native.py, tests/simt_cluster_native.py).  The host call must give the composition
of device calls it replaces -- rslm_draw -> rslm -> lm_solve or lm_amis_fused, epnp_init -> ..., and their split forms --
bit for bit whatever the chunking; with pose_init it must be lm_solve or the existing fused host call; each refusal must
be the composed device calls' and come before the first copy; PushGather with an initialiser must assemble the
single-process composition."""
import contextlib
import ctypes
import socket

import numpy as np
import pytest
import torch

import simt_cluster_native
import simt_native
import test_push_gather_cpu as _pg
from epropnp_b200 import capi, native, sharded
from epropnp_b200.synth import make_problem

OK, BAD_ARG, TOO_MANY_POINTS, UNSUPPORTED = 0, -1, -2, -3


def _host_tensors_on_cpu(monkeypatch):
    # solve_host allocates its outputs pinned: there is no CUDA runtime here
    monkeypatch.setattr(torch, "empty", (lambda f: (lambda *a, pin_memory=False, **k: f(*a, **k)))(torch.empty))


def _case(B, N, dof, bounded, seed=8):
    pc = make_problem(B, N, seed=seed, dof=dof)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
    lb, ub = ((pc["x2d"].amin(1) - 3.0).contiguous(), (pc["x2d"].amax(1) + 3.0).contiguous()) if bounded else (None, None)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta)
    host = dict(x3d=pc["x3d"], x2d=pc["x2d"], w2d=pc["w2d"], cam_mats=pc["cam_mats"].contiguous(), delta=delta,
                lb=lb, ub=ub)
    return prob, host, pc


def _init(kind, dof, seed=31):
    if kind == "rslm":
        return native.rslm_spec(dof, num_points=6, num_proposals=8, num_iter=2, seed=seed)
    return native.epnp_spec(0.5)


def composition(prob, init, p, seed, obj_offset, split=False, ctas=0, pose_init=None):
    """The device calls the host solve composes, on device-resident (here: emulated) tensors."""
    dof = p.dof
    if init is None:
        pose0 = pose_init
    elif init.kind == capi.INIT_RSLM:
        inds, start = native.rslm_draw(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.num_proposals, init.num_points, dof,
                                       eps=init.rslm.eps, seed=init.seed, obj_offset=obj_offset)
        pose0 = (native.rslm_split(prob, inds, start, init.rslm, cluster_ctas=ctas) if split else
                 native.rslm(prob, inds, start, init.rslm))["pose"]
    else:
        pose0 = (native.epnp_init_split(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.conf_quantile, cluster_ctas=ctas)
                 if split else native.epnp_init(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.conf_quantile))
    if p.mc_samples == 0:
        return native.lm_solve(prob, pose0, p, want_cov=True, want_cost=True)
    if split:
        return native.lm_amis_fused_split(prob, pose0, p, seed=seed, obj_offset=obj_offset, want_cost=True,
                                          cluster_ctas=ctas)
    return native.lm_amis_fused(prob, pose0, p, seed=seed, obj_offset=obj_offset, want_cost=True)


def _keys(p):
    return ("pose_opt", "pose_cov", "cost") + (("logw", "pose_samples") if p.mc_samples else ())


def _params(dof, M):
    if M == 0:                                   # the inference flows: GN in fast mode after the initialiser
        return native.default_params(dof, lm_iter=3, fast_mode=1, mc_samples=0)
    return native.default_params(dof, lm_iter=3, mc_samples=M, mc_iter=2)


@pytest.mark.parametrize("dof,kind,bounded,M", [(6, "rslm", False, 0), (6, "rslm", True, 16), (4, "rslm", True, 0),
                                                 (4, "rslm", False, 16), (6, "epnp", True, 0), (6, "epnp", False, 16)])
def test_host_solve_is_the_device_composition(monkeypatch, dof, kind, bounded, M):
    """Every output bit for bit, for n_chunks = 0, 1, 3 and B, at a non-zero obj_offset and an uneven B."""
    simt_native.install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    B, N = 5, 40 if dof == 6 else 33
    prob, host, _ = _case(B, N, dof, bounded)
    p, init = _params(dof, M), _init(kind, dof)
    ref = composition(prob, init, p, seed=77, obj_offset=5)
    ws = torch.empty(native.solve_workspace_bytes(B, N, p, init), dtype=torch.uint8)
    for n_chunks in (0, 1, 3, B):
        res = native.solve_host(host, p, ws, init=init, n_chunks=n_chunks, seed=77, obj_offset=5)
        for k in _keys(p):
            assert torch.equal(res[k], ref[k]), (n_chunks, k)


@pytest.mark.parametrize("dof,kind,M,ctas", [(6, "rslm", 0, 2), (6, "rslm", 12, 3), (4, "rslm", 12, 2),
                                              (4, "rslm", 0, 3), (6, "epnp", 0, 3), (6, "epnp", 12, 2)])
def test_split_host_solve_is_the_split_composition(monkeypatch, dof, kind, M, ctas):
    simt_cluster_native.install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "2")
    B, N = 5, 50 if dof == 6 else 37
    prob, host, _ = _case(B, N, dof, dof == 4)
    p, init = _params(dof, M), _init(kind, dof)
    ref = composition(prob, init, p, seed=5, obj_offset=3, split=True, ctas=ctas)
    ws = torch.empty(native.solve_workspace_bytes(B, N, p, init), dtype=torch.uint8)
    for n_chunks in (0, 1, 3, B):
        res = native.solve_split_host(host, p, ws, init=init, n_chunks=n_chunks, seed=5, obj_offset=3,
                                      cluster_ctas=ctas)
        for k in _keys(p):
            assert torch.equal(res[k], ref[k]), (n_chunks, k)


def test_split_host_solve_automatic_cluster_size(monkeypatch):
    """cluster_ctas = 0: each stage takes its own automatic C, as the device calls do with 0."""
    simt_cluster_native.install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    B, N = 3, 48
    prob, host, _ = _case(B, N, 6, True, seed=12)
    p, init = _params(6, 8), _init("rslm", 6)
    ref = composition(prob, init, p, seed=1, obj_offset=0, split=True, ctas=0)
    ws = torch.empty(native.solve_workspace_bytes(B, N, p, init), dtype=torch.uint8)
    res = native.solve_split_host(host, p, ws, init=init, n_chunks=2, seed=1)
    for k in _keys(p):
        assert torch.equal(res[k], ref[k]), k


@pytest.mark.parametrize("dof,bounded", [(6, True), (4, False)])
def test_given_pose_lm_only_is_lm_solve(monkeypatch, dof, bounded):
    simt_native.install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    B, N = 5, 30
    prob, host, pc = _case(B, N, dof, bounded, seed=4)
    p = native.default_params(dof, lm_iter=4, mc_samples=0)
    ref = native.lm_solve(prob, pc["pose_init"], p, want_cov=True, want_cost=True)
    host["pose_init"] = pc["pose_init"]
    ws = torch.empty(native.solve_workspace_bytes(B, N, p), dtype=torch.uint8)
    for n_chunks in (0, 2, B):
        res = native.solve_host(host, p, ws, n_chunks=n_chunks)
        assert res["logw"] is None and res["pose_samples"] is None
        for k in ("pose_opt", "pose_cov", "cost"):
            assert torch.equal(res[k], ref[k]), (n_chunks, k)


@pytest.mark.parametrize("split", [False, True])
def test_given_pose_with_amis_is_the_fused_host_call(monkeypatch, split):
    (simt_cluster_native if split else simt_native).install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "2")
    B, N = 5, 40
    _, host, pc = _case(B, N, 6, True, seed=6)
    host["pose_init"] = pc["pose_init"]
    p = native.default_params(6, lm_iter=3, mc_samples=16, mc_iter=2)
    ws = torch.empty(native.solve_workspace_bytes(B, N, p), dtype=torch.uint8)
    assert ws.numel() == native.fused_workspace_bytes(B, N, p)
    for n_chunks in (0, 3):
        if split:
            ref = native.lm_amis_fused_split_host(host, p, ws, n_chunks=n_chunks, seed=9, obj_offset=2, cluster_ctas=3)
            res = native.solve_split_host(host, p, ws, n_chunks=n_chunks, seed=9, obj_offset=2, cluster_ctas=3)
        else:
            ref = native.lm_amis_fused_host(host, p, ws, n_chunks=n_chunks, seed=9, obj_offset=2)
            res = native.solve_host(host, p, ws, n_chunks=n_chunks, seed=9, obj_offset=2)
        for k in ("pose_opt", "pose_cov", "cost", "logw", "pose_samples"):
            assert torch.equal(res[k], ref[k]), (n_chunks, k)


def test_workspace_query():
    h = simt_native.handle()
    p = capi.EpnpParams()
    h.epnp_default_params(ctypes.byref(p), 6)
    fused = h.epnp_fused_workspace_bytes(8, 64, ctypes.byref(p))
    assert h.epnp_solve_workspace_bytes(8, 64, ctypes.byref(p), None) == fused
    assert h.epnp_solve_workspace_bytes(8, 64, ctypes.byref(p), ctypes.byref(native.epnp_spec())) == fused
    rs = capi.EpnpInit(kind=capi.INIT_RSLM, num_proposals=64, num_points=16)
    extra = h.epnp_solve_workspace_bytes(8, 64, ctypes.byref(p), ctypes.byref(rs)) - fused
    assert extra >= 64 * 8 * (16 * 4 + 7 * 4 * 2 + 4) + 8 * 4          # inds, start, pose_all, cost_all, cost_best
    for bad in (capi.EpnpInit(kind=0), capi.EpnpInit(kind=capi.INIT_RSLM, num_proposals=0, num_points=16),
                capi.EpnpInit(kind=capi.INIT_RSLM, num_proposals=64, num_points=0)):
        assert h.epnp_solve_workspace_bytes(8, 64, ctypes.byref(p), ctypes.byref(bad)) == 0
    assert h.epnp_solve_workspace_bytes(-1, 64, ctypes.byref(p), None) == 0
    assert h.epnp_solve_workspace_bytes(8, 0, ctypes.byref(p), None) == 0
    assert h.epnp_solve_workspace_bytes(8, 64, None, None) == 0
    assert ctypes.sizeof(capi.EpnpInit) == 96


# ---- refusals: (case, forms, changes, (rc with B = 2, rc with B = 0)).  Changes: "init" (rslm / epnp / None), "dof",
# "M" (mc_samples), "N", "n" / "P" / "q" of the initialiser, "spec_dof", "kind", "p.<field>", pointer arguments set to
# None or given ("pose_init": "given"), "cluster_ctas", "env", "short" (workspace one byte short).
RES, SPL = "epnp_solve_host_f32", "epnp_solve_split_host_f32"
BOTH = {RES, SPL}


def _resident(h, dof, M):
    return h.epnp_max_points(dof, M, 2 if M else 0)


REFUSALS = [
    ("valid_rslm", BOTH, {}, (None, OK)),
    ("valid_epnp", BOTH, {"init": "epnp"}, (None, OK)),
    ("valid_pose_init", BOTH, {"init": None, "pose_init": "given"}, (None, OK)),
    ("both_starts", BOTH, {"pose_init": "given"}, (BAD_ARG, BAD_ARG)),
    ("no_start", BOTH, {"init": None}, (BAD_ARG, BAD_ARG)),
    ("unknown_kind", BOTH, {"kind": 3}, (BAD_ARG, BAD_ARG)),
    ("epnp_dof4", BOTH, {"init": "epnp", "dof": 4}, (BAD_ARG, BAD_ARG)),
    ("rslm_spec_of_other_dof", BOTH, {"spec_dof": 4}, (BAD_ARG, BAD_ARG)),
    ("logw_without_amis", BOTH, {"M": 0, "logw": "given"}, (BAD_ARG, BAD_ARG)),
    ("samples_without_amis", BOTH, {"M": 0, "pose_samples": "given"}, (BAD_ARG, BAD_ARG)),
    ("amis_without_logw", BOTH, {"logw": None}, (BAD_ARG, BAD_ARG)),
    ("M<0", BOTH, {"M": -8}, (BAD_ARG, BAD_ARG)),
    ("M%I!=0", BOTH, {"M": 15}, (BAD_ARG, BAD_ARG)),
    ("lb_without_ub", BOTH, {"ub": None}, (BAD_ARG, BAD_ARG)),
    ("B<0", BOTH, {"B": -1}, (BAD_ARG, None)),
    ("conf_quantile>1", BOTH, {"init": "epnp", "q": 1.5}, (BAD_ARG, BAD_ARG)),
    ("epnp_N<4", BOTH, {"init": "epnp", "N": 3}, (BAD_ARG, BAD_ARG)),
    ("epnp_fewer_than_4_kept", BOTH, {"init": "epnp", "N": 5, "q": 0.9}, (BAD_ARG, BAD_ARG)),
    ("P=0", BOTH, {"P": 0}, (BAD_ARG, BAD_ARG)),
    ("n=0", BOTH, {"n": 0}, (BAD_ARG, BAD_ARG)),
    ("n>N", BOTH, {"n": 65}, (BAD_ARG, BAD_ARG)),
    ("rslm_lm_iter<0", BOTH, {"spec.lm_iter": -1}, (BAD_ARG, BAD_ARG)),
    ("lm_iter<0", BOTH, {"p.lm_iter": -1}, (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_amis", BOTH, {"p.fast_mode": 1, "p.lm_iter": 0}, (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_lm_cov", BOTH, {"M": 0, "p.fast_mode": 1, "p.lm_iter": 0}, (BAD_ARG, BAD_ARG)),
    ("fast_no_steps_lm_pose_only", BOTH, {"M": 0, "p.fast_mode": 1, "p.lm_iter": 0, "pose_cov": None, "cost": None},
     (None, OK)),
    # the draw kernel's shared memory: 200 indices per thread leave room for 6,400 weights
    ("draw_smem", BOTH, {"M": 0, "N": 6500, "n": 200}, (TOO_MANY_POINTS, OK)),
    ("rslm_resident", {RES}, {"M": 0, "N": lambda h, dof, M: h.epnp_max_points(dof, 0, 0) + 4}, (TOO_MANY_POINTS, OK)),
    ("epnp_resident", {RES}, {"init": "epnp", "M": 0, "N": lambda h, dof, M: h.epnp_max_points(6, 0, 0) + 4},
     (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("amis_resident", {RES}, {"init": "epnp", "N": lambda h, dof, M: _resident(h, dof, M) + 4},
     (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("split_limit", {SPL}, {"init": "epnp", "N": lambda h, dof, M: h.epnp_max_points_split(dof, M, 2) + 1},
     (TOO_MANY_POINTS, TOO_MANY_POINTS)),
    ("cluster=1", {SPL}, {"cluster_ctas": 1}, (BAD_ARG, BAD_ARG)),
    ("cluster=9", {SPL}, {"cluster_ctas": 9}, (BAD_ARG, BAD_ARG)),
    ("no_cluster_fits_rslm", {SPL}, {"env": "0"}, (UNSUPPORTED, OK)),
    ("no_cluster_fits_epnp", {SPL}, {"init": "epnp", "env": "0"}, (UNSUPPORTED, OK)),
    ("no_cluster_fits_lm_only", {SPL}, {"M": 0, "env": "0"}, (UNSUPPORTED, OK)),
    ("workspace_short", BOTH, {"short": True}, (BAD_ARG, OK)),
] + [(f"{a}=NULL", BOTH, {a: None}, (BAD_ARG, BAD_ARG))
     for a in ("x3d", "x2d", "w2d", "cam", "delta", "pose_opt", "workspace", "params")]


def _call(name, changes, B, monkeypatch):
    """-> (rc, {buffer: (array, contents before)})."""
    h = simt_cluster_native.handle() if name == SPL else simt_native.handle()
    dof = changes.get("dof", 6)
    M = changes.get("M", 8)
    p = capi.EpnpParams()
    h.epnp_default_params(ctypes.byref(p), dof)
    p.mc_samples, p.mc_iter, p.lm_iter = M, 2, 2
    for k, v in changes.items():
        if k.startswith("p."):
            setattr(p, k[2:], v)
    kind = changes.get("init", "rslm")
    init = None
    if kind == "rslm":
        init = native.rslm_spec(changes.get("spec_dof", dof), num_points=changes.get("n", 4),
                                num_proposals=changes.get("P", 4), num_iter=2)
        if "spec.lm_iter" in changes:
            init.rslm.lm_iter = changes["spec.lm_iter"]
    elif kind == "epnp":
        init = capi.EpnpInit(kind=capi.INIT_EPNP, conf_quantile=changes.get("q", 0.5))
    if init is not None and "kind" in changes:
        init.kind = changes["kind"]
    N = changes.get("N", 64)
    N = N(h, dof, M) if callable(N) else N
    if "env" in changes:
        monkeypatch.setenv("SIMT_EMUL_CLUSTERS", changes["env"])
    Bn, D = max(B, 1), 7 if dof == 6 else 4
    buffers = {}

    def buf(arg, size, default_given=True):
        given = changes.get(arg, "given" if default_given else None)
        if given is None:
            return None
        a = np.full(max(size, 1), 1234.5, dtype=np.float32)
        buffers[arg] = (a, a.copy())
        return ctypes.c_void_p(a.ctypes.data)

    pts = [buf("x3d", Bn * N * 3), buf("x2d", Bn * N * 2), buf("w2d", Bn * N * 2), buf("cam", Bn * 9),
           buf("lb", Bn * 2), buf("ub", Bn * 2), buf("delta", Bn), buf("pose_init", Bn * D, False)]
    amis = M > 0
    outs = [buf("pose_opt", Bn * D), buf("pose_cov", Bn * 36), buf("cost", Bn),
            buf("pose_samples", Bn * max(M, 1) * D, amis), buf("logw", Bn * max(M, 1), amis)]
    need = h.epnp_solve_workspace_bytes(max(B, 0), N, ctypes.byref(p), None if init is None else ctypes.byref(init))
    ws_bytes = need - 1 if changes.get("short") else need
    ws = buf("workspace", need // 4 + 64)
    params = None if changes.get("params", "given") is None else ctypes.byref(p)
    extra = (changes.get("cluster_ctas", 0),) if name == SPL else ()
    rc = getattr(h, name)(*pts, None if init is None else ctypes.byref(init), 7, 0, *outs, ws, ws_bytes, 0, B, N,
                          params, *extra, None)
    return rc, buffers


def _refusal_ids():
    for case, forms, changes, (rc_b, rc_0) in REFUSALS:
        for name in sorted(forms):
            for B, rc in ((changes.get("B", 2), rc_b), (0, rc_0)):
                if rc is not None:
                    yield pytest.param(name, changes, B, rc, id=f"{name}-{case}-B{B}")


@pytest.mark.parametrize("name,changes,B,expected", list(_refusal_ids()))
def test_refusal_comes_before_any_copy(monkeypatch, name, changes, B, expected):
    """The code each refusal returns, with B = 2 and with B = 0; a refused call, and any call on an empty batch, leaves
    every buffer it was given -- the workspace included -- as it was."""
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "16")
    rc, buffers = _call(name, changes, B, monkeypatch)
    assert rc == expected, (name, changes, B, rc)
    for arg, (a, before) in buffers.items():
        assert np.array_equal(a, before), f"{name} wrote {arg}"


@pytest.mark.parametrize("case", ["draw_smem", "rslm_resident", "epnp_resident", "amis_resident"])
def test_host_refusal_is_the_device_calls_refusal(monkeypatch, case):
    """The resident host call's code equals the first refusal of the device calls it composes, called with B = 2 on
    device (here: host) buffers."""
    simt_native.install(monkeypatch)
    changes = next(c for name, _, c, _ in REFUSALS if name == case)
    rc, _ = _call(RES, changes, 2, monkeypatch)
    h = simt_native.handle()
    dof, M = 6, changes.get("M", 8)
    N = changes["N"](h, dof, M) if callable(changes["N"]) else changes["N"]
    pc = make_problem(2, N, seed=1)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, 1.0)
    p = native.default_params(dof, lm_iter=2, mc_samples=M, mc_iter=2)
    init = (native.rslm_spec(6, num_points=changes.get("n", 4), num_proposals=4, num_iter=2)
            if changes.get("init", "rslm") == "rslm" else native.epnp_spec(0.5))
    with pytest.raises(native.NativeError) as err:
        composition(prob, init, p, seed=7, obj_offset=0, pose_init=pc["pose_init"])
    assert f"(code {rc})" in str(err.value)


# ---- PushGather with an initialiser
def test_push_from_initialiser_with_stand_in_peers(monkeypatch):
    """What PushGather.solve(init=...) runs on each rank -- initial_pose on the shard with obj_offset = lo, then the
    push call -- for two ranks in one process pushing into each other's full-batch buffers: the assembled batch is the
    single-process composition."""
    simt_native.install(monkeypatch)
    B, N, M, world = 6, 24, 8, 2
    pc = make_problem(B, N, seed=44)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
    p = native.default_params(6, lm_iter=2, mc_samples=M, mc_iter=2)
    init = _init("rslm", 6, seed=3)
    whole = composition(native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta), init, p,
                        seed=11, obj_offset=0)
    full_lw = [torch.full((B, M), float("nan")) for _ in range(world)]
    full_ps = [torch.full((B, 7), float("nan")) for _ in range(world)]
    per = B // world
    for r in range(world):
        lo, hi = r * per, (r + 1) * per
        prob = native.Problem(pc["x3d"][lo:hi], pc["x2d"][lo:hi], pc["w2d"][lo:hi], pc["cam_mats"][lo:hi], None, None,
                              delta[lo:hi])
        pose0 = native.initial_pose(prob, init, 6, obj_offset=lo)
        others = [q for q in range(world) if q != r]
        out = native.lm_amis_fused_push(prob, pose0, p, full_ps[r][lo:hi], full_lw[r][lo:hi],
                                        [full_lw[q] for q in others], [full_ps[q] for q in others], seed=11,
                                        obj_offset=lo)
        assert torch.equal(out["pose_samples"], whole["pose_samples"][lo:hi])
    for q in range(world):
        assert torch.equal(full_lw[q], whole["logw"]) and torch.equal(full_ps[q], whole["pose_opt"])


def test_push_gather_refuses_two_starts():
    pg = object.__new__(sharded.PushGather)
    pg.step, pg.depth, pg.rank, pg.per_rank = 0, 2, 0, 1
    with pytest.raises(ValueError):
        pg.solve(None, torch.zeros(1, 7), None, init=native.epnp_spec())


def _init_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.multiprocessing.set_sharing_strategy("file_system")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        capi._lib = simt_native.handle(())                       # what simt_native.install does, without pytest
        native._need_cuda = lambda t, what: None
        native.stream_ptr = lambda device=None: None
        torch.cuda.device = lambda device=None: contextlib.nullcontext()
        per, N, M, depth = 3, 20, 8, 2
        num_obj = per * world
        p = native.default_params(6, lm_iter=2, mc_samples=M, mc_iter=2)
        pg = _pg._host_push_gather_class()(num_obj, M, 7, "cpu", depth=depth, valid_for=1)
        lo, hi = rank * per, (rank + 1) * per
        ok = True
        for step, kind in enumerate(("rslm", "epnp", "rslm")):
            pc = make_problem(num_obj, N, seed=50 + step)
            delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
            init = _init(kind, 6, seed=step)
            whole = composition(native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta),
                                init, p, seed=step, obj_offset=0)
            mine = native.Problem(pc["x3d"][lo:hi], pc["x2d"][lo:hi], pc["w2d"][lo:hi], pc["cam_mats"][lo:hi], None, None,
                                  delta[lo:hi])
            out, pending = pg.solve(mine, None, p, seed=step, init=init)
            got = pending.wait()
            ok = ok and torch.equal(out["pose_samples"], whole["pose_samples"][lo:hi])
            ok = ok and torch.equal(got["logw"], whole["logw"]) and torch.equal(got["pose_opt"], whole["pose_opt"])
        dist.barrier()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_push_gather_from_initialiser_two_processes_gloo():
    """Two gloo ranks whose PushGather.solve starts from an RSLM or EPnP initialiser: every rank's assembled batch equals
    the single-process composition of the whole batch."""
    import torch.multiprocessing as mp
    simt_native.build_emulated(())                               # build once, before the workers race for it
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_init_worker, args=(r, world, port, q)) for r in range(world)]
    try:
        for pr in procs:
            pr.start()
        results = [q.get(timeout=240) for _ in range(world)]
        for pr in procs:
            pr.join(timeout=60)
    finally:
        for pr in procs:
            if pr.is_alive():
                pr.terminate()
                pr.join()
    assert sorted(results) == [(r, True) for r in range(world)]
