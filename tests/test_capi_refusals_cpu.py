"""Every C-ABI entry point's refusals, and their precedence, through ctypes on the SIMT emulator builds: resident calls
on the single-CTA emulator (tests/simt_emul), `_split` calls on the cluster emulator (tests/simt_cluster).

Each case is run twice, with B = 2 and with B = 0: which check an entry point makes before it looks at B is part of its
behaviour (some report EPNP_ERR_TOO_MANY_POINTS for an empty batch, others EPNP_OK).  A refused call, and a valid call on
an empty batch, must leave every buffer it was given as it was.  No case launches a kernel."""
import ctypes

import numpy as np
import pytest

import simt_cluster_native
import simt_native
from epropnp_b200 import capi

OK, BAD_ARG, TOO_MANY_POINTS, UNSUPPORTED = 0, -1, -2, -3
SENTINEL = 1234.5
NT = 128                    # threads per CTA of the CTA-per-object kernels (pnp_device.cuh)

# The arguments of each entry point in order.  name* a required input, name? an optional input, name! a required
# output, name~ an optional output, seed$ a required device seed; bare names are scalars (DEFAULTS), `params` an
# EpnpParams, `stream` the stream.  Every pointer is given unless a case takes it away; rslm_draw's t_init is not, so
# that x3d, x2d and cam_mats are required.
PTS = "x3d* x2d* w2d* cam* lb? ub? delta*"
SIGS = {
    "epnp_adaptive_delta_f32": "x2d* w2d* relative_delta delta! B N stream",
    "epnp_mc_epilogue_f32": "logw* pose_samples? pose_opt? cost_target? lse~ loss~ weights~ score_te~ B M dof stream",
    "epnp_mc_lse_backward_f32": "logw* lse* grad_lse* grad_logw! B M stream",
    "epnp_evaluate_cost_f32": f"{PTS} poses* cost! S B N dof z_min stream",
    "epnp_evaluate_cost_split_f32": f"{PTS} poses* cost! S B N dof z_min cluster_ctas stream",
    "epnp_evaluate_f32": f"{PTS} pose* residual~ jac~ cost~ clip_jac B N dof z_min huber_eps stream",
    "epnp_lm_solve_f32": f"{PTS} pose_init* pose_opt! pose_cov~ cost~ pose_plus~ cost_init~ B N params stream",
    "epnp_gn_plus_backward_f32": f"{PTS} pose* gplus* gx3d~ gx2d~ gw2d~ gdelta~ B N dof z_min eps huber_eps stream",
    "epnp_gn_plus_backward_split_f32":
        f"{PTS} pose* gplus* gx3d~ gx2d~ gw2d~ gdelta~ B N dof z_min eps huber_eps cluster_ctas stream",
    "epnp_rslm_f32": f"{PTS} inds* start* pose_best! cost_best! pose_all~ cost_all~ P n B N params stream",
    "epnp_rslm_draw_f32": "x3d* x2d* w2d* cam* t_init? seed obj_offset inds! start! t_out~ P n B N dof eps stream",
    "epnp_rslm_draw_seedptr_f32":
        "x3d* x2d* w2d* cam* t_init? seed$ obj_offset inds! start! t_out~ P n B N dof eps stream",
    "epnp_epnp_init_f32": "x3d* x2d* w2d? cam* conf_quantile pose! n_sel~ B N stream",
    "epnp_epnp_init_split_f32": "x3d* x2d* w2d? cam* conf_quantile pose! n_sel~ B N cluster_ctas stream",
    "epnp_amis_f32": f"{PTS} pose_opt* pose_cov* noise_n? noise_chi2? noise_rot? seed obj_offset "
                     "pose_samples! logw! proposals~ B N params stream",
    "epnp_lm_amis_fused_f32": f"{PTS} pose_init* noise_n? noise_chi2? noise_rot? seed obj_offset pose_opt! pose_cov~ "
                              "cost~ pose_plus~ cost_init~ pose_samples! logw! proposals~ B N params stream",
    "epnp_lm_amis_fused_seedptr_f32": f"{PTS} pose_init* noise_n? noise_chi2? noise_rot? seed$ obj_offset pose_opt! "
                                      "pose_cov~ cost~ pose_plus~ cost_init~ pose_samples! logw! proposals~ B N params "
                                      "stream",
    "epnp_lm_amis_fused_split_f32": f"{PTS} pose_init* noise_n? noise_chi2? noise_rot? seed obj_offset pose_opt! "
                                    "pose_cov~ cost~ pose_plus~ cost_init~ pose_samples! logw! proposals~ B N params "
                                    "cluster_ctas stream",
    "epnp_lm_amis_fused_split_seedptr_f32": f"{PTS} pose_init* noise_n? noise_chi2? noise_rot? seed$ obj_offset "
                                            "pose_opt! pose_cov~ cost~ pose_plus~ cost_init~ pose_samples! logw! "
                                            "proposals~ B N params cluster_ctas stream",
    "epnp_lm_amis_fused_push_f32": f"{PTS} pose_init* seed obj_offset pose_opt! pose_cov~ cost~ pose_samples! logw! "
                                   "peer_logw? peer_pose? n_peers B N params stream",
    "epnp_lm_amis_fused_split_push_f32": f"{PTS} pose_init* seed obj_offset pose_opt! pose_cov~ cost~ pose_samples! "
                                         "logw! peer_logw? peer_pose? n_peers B N params cluster_ctas stream",
    "epnp_cost_backward_f32": f"{PTS} poses_a* grad_a* PA poses_b* grad_b* PB gx3d~ gx2d~ gw2d~ gdelta~ B N dof z_min "
                              "stream",
    "epnp_lm_amis_fused_host_f32": f"{PTS} pose_init* seed obj_offset pose_opt! pose_cov~ cost~ pose_samples~ logw! "
                                   "workspace* workspace_bytes n_chunks B N params stream",
    "epnp_lm_amis_fused_split_host_f32": f"{PTS} pose_init* seed obj_offset pose_opt! pose_cov~ cost~ pose_samples~ "
                                         "logw! workspace* workspace_bytes n_chunks B N params cluster_ctas stream",
}
DEFAULTS = dict(relative_delta=0.05, S=1, B=2, N=64, M=8, dof=6, z_min=0.1, eps=1e-5, huber_eps=1e-10, clip_jac=0,
                P=4, n=4, seed=7, obj_offset=0, conf_quantile=0.5, n_peers=0, PA=1, PB=1, n_chunks=0, cluster_ctas=0)
POINT_BUFFERS = {"x3d", "x2d", "w2d", "gx3d", "gx2d", "gw2d"}
SAMPLE_BUFFERS = {"pose_samples", "noise_n", "noise_chi2", "noise_rot", "logw", "proposals", "lse", "grad_lse",
                  "grad_logw", "loss", "weights", "score_te", "cost_target"}
RSLM_BUFFERS = {"inds", "start", "pose_all", "cost_all"}
INT_BUFFERS = {"inds", "n_sel"}
NOT_GIVEN = {"t_init", "peer_logw", "peer_pose"}


def _spec(name):
    return [(tok.rstrip("*?!~$"), tok[-1] if tok[-1] in "*?!~$" else "") for tok in SIGS[name].split()]


def _has(name, arg):
    return any(a == arg for a, _ in _spec(name))


def _params_call(name):
    return _has(name, "params")


def _amis(name):
    return "amis" in name


def _split(name):
    return "_split" in name


def _resident_limit(h, name, p, dof, n):
    """Largest N the resident form takes (None: it streams any N)."""
    if name in ("epnp_evaluate_cost_f32", "epnp_gn_plus_backward_f32", "epnp_rslm_f32"):
        return h.epnp_max_points(dof, 0, 0)
    if name == "epnp_epnp_init_f32":
        return h.epnp_max_points(6, 0, 0)
    if name in ("epnp_amis_f32", "epnp_lm_amis_fused_f32", "epnp_lm_amis_fused_seedptr_f32",
                "epnp_lm_amis_fused_push_f32", "epnp_lm_amis_fused_host_f32"):
        return h.epnp_max_points(dof, p.mc_samples, p.mc_iter)
    if name.startswith("epnp_rslm_draw"):
        # the draw kernel's shared memory: the weights (N rounded up to 4), n indices and floats per thread, 2 KB more
        return (227 * 1024 - 2048 - n * NT * 8) // 16 * 4
    return None


def _split_limit(h, name, p, dof):
    if not _split(name):
        return None
    if name == "epnp_epnp_init_split_f32":
        return h.epnp_max_points_split(6, 0, 0)
    m, i = (p.mc_samples, p.mc_iter) if _amis(name) else (0, 0)
    limit = h.epnp_max_points_split(dof, m, i)
    assert h.epnp_split_ctas(dof, limit, m, i) > 0 and h.epnp_split_ctas(dof, limit + 1, m, i) == 0
    return limit


def _resident_plus(h, name, p, dof, n):
    limit = _resident_limit(h, name, p, dof, n)
    return None if limit is None else limit + 4


def _split_plus(h, name, p, dof, n):
    limit = _split_limit(h, name, p, dof)
    return None if limit is None else limit + 1


ALL = set(SIGS)
WITH_N = {n for n in ALL if _has(n, "N")}
PARAMS_OR_DOF = {n for n in ALL if _has(n, "dof") or _params_call(n)}
BOUNDED = {n for n in ALL if _has(n, "lb")}
AMIS = {n for n in ALL if _amis(n)}
LM = {n for n in ALL if _params_call(n) and n != "epnp_amis_f32"}
FUSED = {n for n in AMIS if n != "epnp_amis_f32"}
FAST0 = {"p.fast_mode": 1, "p.lm_iter": 0}
NOISE = {n for n in ALL if _has(n, "noise_n")}
SPLIT = {n for n in ALL if _split(n)}
PUSH = {n for n in ALL if "push" in n}
HOST = {n for n in ALL if "host" in n}
RESIDENT_LIMITED = {"epnp_evaluate_cost_f32", "epnp_gn_plus_backward_f32", "epnp_rslm_f32", "epnp_rslm_draw_f32",
                    "epnp_rslm_draw_seedptr_f32", "epnp_epnp_init_f32", "epnp_amis_f32", "epnp_lm_amis_fused_f32",
                    "epnp_lm_amis_fused_seedptr_f32", "epnp_lm_amis_fused_push_f32", "epnp_lm_amis_fused_host_f32"}

# (case, entry points, changes, (rc with B = 2, rc with B = 0), {entry point: its own pair}).  Changes: argument values,
# "p.<field>" for an EpnpParams field, "env" for the cluster emulator's environment; a callable value is computed from
# (handle, entry point, params, dof, n).  `dof` sets the params' dof for the calls that take an EpnpParams.
CASES = [
    ("B<0", ALL, {"B": -1}, (BAD_ARG, None), {}),
    ("N=0", WITH_N - {"epnp_epnp_init_f32", "epnp_epnp_init_split_f32"}, {"N": 0}, (BAD_ARG, BAD_ARG), {}),
    ("N<4", {"epnp_epnp_init_f32", "epnp_epnp_init_split_f32"}, {"N": 3}, (BAD_ARG, BAD_ARG), {}),
    ("dof=5", PARAMS_OR_DOF, {"dof": 5}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("lb_without_ub", BOUNDED, {"ub": None}, (BAD_ARG, BAD_ARG), {}),
    ("M%I!=0", AMIS, {"p.mc_samples": 510}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("I>8", AMIS, {"p.mc_iter": 16}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("acg_mle_iter<0", AMIS, {"p.acg_mle_iter": -1}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("lm_iter<0", LM, {"p.lm_iter": -1}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    # fast mode with no Gauss-Newton step has no covariance, cost or cost_init to return
    ("fast_no_steps", FUSED, FAST0, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("fast_no_steps_all_outputs", {"epnp_lm_solve_f32"}, FAST0, (BAD_ARG, BAD_ARG), {}),
    ("fast_no_steps_cov", {"epnp_lm_solve_f32"}, dict(FAST0, cost=None, pose_plus=None, cost_init=None),
     (BAD_ARG, BAD_ARG), {}),
    ("fast_no_steps_cost", {"epnp_lm_solve_f32"}, dict(FAST0, pose_cov=None, pose_plus=None, cost_init=None),
     (BAD_ARG, BAD_ARG), {}),
    ("fast_no_steps_cost_init", {"epnp_lm_solve_f32"}, dict(FAST0, pose_cov=None, cost=None, pose_plus=None),
     (BAD_ARG, BAD_ARG), {}),
    ("fast_no_steps_pose_only", {"epnp_lm_solve_f32"}, dict(FAST0, pose_cov=None, cost=None, cost_init=None),
     (None, OK), {}),
    ("noise_normal_only", NOISE, {"noise_chi2": None, "noise_rot": None}, (BAD_ARG, BAD_ARG), {}),
    ("noise_rot_missing", NOISE, {"noise_rot": None}, (BAD_ARG, BAD_ARG), {}),
    ("cluster=1", SPLIT, {"cluster_ctas": 1}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("cluster=9", SPLIT, {"cluster_ctas": 9}, (BAD_ARG, BAD_ARG), {n: (BAD_ARG, OK) for n in HOST}),
    ("no_cluster_fits", SPLIT, {"env": "0"}, (UNSUPPORTED, OK), {}),
    ("N>resident", RESIDENT_LIMITED, {"N": _resident_plus}, (TOO_MANY_POINTS, OK),
     {n: (TOO_MANY_POINTS, TOO_MANY_POINTS) for n in ("epnp_epnp_init_f32", "epnp_lm_amis_fused_f32",
                                                       "epnp_lm_amis_fused_seedptr_f32", "epnp_lm_amis_fused_push_f32")}),
    ("N>split", SPLIT, {"N": _split_plus}, (TOO_MANY_POINTS, TOO_MANY_POINTS),
     {"epnp_lm_amis_fused_split_host_f32": (TOO_MANY_POINTS, OK)}),
    ("S<0", {"epnp_evaluate_cost_f32", "epnp_evaluate_cost_split_f32"}, {"S": -1}, (BAD_ARG, BAD_ARG), {}),
    ("M=0", {"epnp_mc_epilogue_f32", "epnp_mc_lse_backward_f32"}, {"M": 0}, (BAD_ARG, BAD_ARG), {}),
    ("no_epilogue_output", {"epnp_mc_epilogue_f32"}, {"lse": None, "loss": None, "weights": None, "score_te": None},
     (BAD_ARG, BAD_ARG), {}),
    ("score_without_samples", {"epnp_mc_epilogue_f32"}, {"pose_samples": None}, (BAD_ARG, BAD_ARG), {}),
    ("score_without_pose", {"epnp_mc_epilogue_f32"}, {"pose_opt": None}, (BAD_ARG, BAD_ARG), {}),
    ("PA<0", {"epnp_cost_backward_f32"}, {"PA": -1}, (BAD_ARG, BAD_ARG), {}),
    ("P=0", {n for n in ALL if "rslm" in n}, {"P": 0}, (BAD_ARG, BAD_ARG), {}),
    ("n=0", {n for n in ALL if "rslm" in n}, {"n": 0}, (BAD_ARG, BAD_ARG), {}),
    ("n>N", {"epnp_rslm_draw_f32", "epnp_rslm_draw_seedptr_f32"}, {"n": 65}, (BAD_ARG, BAD_ARG), {}),
    ("conf_quantile>1", {"epnp_epnp_init_f32", "epnp_epnp_init_split_f32"}, {"conf_quantile": 1.5},
     (BAD_ARG, BAD_ARG), {}),
    ("peers_without_tables", PUSH, {"n_peers": 1}, (BAD_ARG, BAD_ARG), {}),
    ("n_peers>8", PUSH, {"n_peers": 9, "peer_logw": "table", "peer_pose": "table"}, (BAD_ARG, BAD_ARG), {}),
    ("n_peers<0", PUSH, {"n_peers": -1}, (BAD_ARG, BAD_ARG), {}),
    ("workspace_too_small", HOST, {"workspace_bytes": lambda ws: ws // 2}, (BAD_ARG, OK), {}),
]
for _name in SIGS:
    for _arg, _kind in _spec(_name):
        if _kind in "*!$" and _kind:
            CASES.append((f"{_arg}=NULL", {_name}, {_arg: None}, (BAD_ARG, BAD_ARG), {}))
CASES.append(("valid", ALL, {}, (None, OK), {}))


def _handle(name):
    return simt_cluster_native.handle() if _split(name) else simt_native.handle()


def _call(name, changes, B, monkeypatch):
    """-> (rc, {buffer: (array, its contents before the call)})."""
    h = _handle(name)
    p = capi.EpnpParams()
    h.epnp_default_params(ctypes.byref(p), 6)
    vals = dict(DEFAULTS, B=B)
    dof = changes.get("dof", DEFAULTS["dof"])
    p.dof = dof
    for k, v in changes.items():
        if k.startswith("p."):
            setattr(p, k[2:], v)
    for k in ("n", "P", "S", "M", "conf_quantile", "n_peers", "PA", "cluster_ctas", "dof"):
        if k in changes:
            vals[k] = changes[k]
    if "N" in changes:
        vals["N"] = changes["N"](h, name, p, dof, vals["n"]) if callable(changes["N"]) else changes["N"]
    if "B" in changes:
        vals["B"] = changes["B"]
    if "env" in changes:
        monkeypatch.setenv("SIMT_EMUL_CLUSTERS", changes["env"])
    Bn, N, M = max(vals["B"], 1), max(vals["N"], 1), max(p.mc_samples, vals["M"], 1)
    buffers, args = {}, []
    for arg, kind in _spec(name):
        if kind:
            if arg in changes and changes[arg] is None or (arg in NOT_GIVEN and changes.get(arg) != "table"):
                args.append(None)
                continue
            if arg in ("peer_logw", "peer_pose"):
                table = (ctypes.c_void_p * 16)(*[buffers["logw"][0].ctypes.data] * 16)
                buffers[arg] = (table, None)
                args.append(ctypes.cast(table, ctypes.c_void_p))
                continue
            if arg == "workspace":
                size = max(h.epnp_fused_workspace_bytes(vals["B"], vals["N"], ctypes.byref(p)) // 4, 64)
            elif arg in POINT_BUFFERS:
                size = Bn * N * 3
            elif arg in SAMPLE_BUFFERS:
                size = Bn * M * 8
            elif arg in RSLM_BUFFERS:
                size = Bn * max(vals["P"], 1) * max(vals["n"], 8)
            else:
                size = Bn * 64
            if kind == "$":
                a = np.full(4, 0x5EED, dtype=np.uint64)
            elif arg in INT_BUFFERS:
                a = np.full(size, 0x7EADBEEF, dtype=np.int32)
            else:
                a = np.full(size, SENTINEL, dtype=np.float32)
            buffers[arg] = (a, a.copy())
            args.append(ctypes.c_void_p(a.ctypes.data))
        elif arg == "params":
            args.append(ctypes.byref(p))
        elif arg == "stream":
            args.append(None)
        elif arg == "workspace_bytes":
            ws = h.epnp_fused_workspace_bytes(vals["B"], vals["N"], ctypes.byref(p))
            args.append(changes[arg](ws) if arg in changes else ws)
        else:
            args.append(vals[arg])
    rc = getattr(h, name)(*args)
    return rc, buffers


def _case_ids():
    for case, entries, changes, (rc_b, rc_0), own in CASES:
        for name in sorted(entries):
            want = own.get(name, (rc_b, rc_0))
            for B, rc in ((changes.get("B", 2), want[0]), (0, want[1])):
                if rc is not None:
                    yield pytest.param(name, changes, B, rc, id=f"{name}-{case}-B{B}")


@pytest.mark.parametrize("name,changes,B,expected", list(_case_ids()))
def test_refusal_and_its_precedence(monkeypatch, name, changes, B, expected):
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "16")
    rc, buffers = _call(name, changes, B, monkeypatch)
    assert rc == expected, (name, changes, B, rc)
    for arg, (a, before) in buffers.items():
        if before is not None and arg != "workspace":
            assert np.array_equal(a, before), f"{name} wrote {arg}"


def test_queries_refuse_what_no_call_takes():
    h = simt_native.handle()
    p = capi.EpnpParams()
    h.epnp_default_params(ctypes.byref(p), 6)
    assert h.epnp_split_ctas(5, 1024, 512, 4) == 0
    assert h.epnp_split_ctas(6, 0, 512, 4) == 0
    assert h.epnp_split_ctas(6, 1024, -1, 4) == 0
    assert h.epnp_split_ctas(6, 1024, 510, 4) == 0
    assert h.epnp_split_ctas(6, 1024, 512, 16) == 0
    assert h.epnp_split_ctas(6, 1024, 512, 4) >= 2
    assert h.epnp_max_points_split(6, 510, 4) == 0
    assert h.epnp_fused_workspace_bytes(2, 64, None) == 0
    assert h.epnp_fused_workspace_bytes(-1, 64, ctypes.byref(p)) == 0
    assert h.epnp_fused_workspace_bytes(2, 0, ctypes.byref(p)) == 0
    assert h.epnp_error_string(-99) == b"unknown error"
    assert h.epnp_last_cuda_error() == 0
    assert h.epnp_abi_version() == capi.ABI_VERSION
