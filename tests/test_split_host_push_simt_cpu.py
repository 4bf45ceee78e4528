"""The host-buffer and push forms of the cluster-split solve (epnp_lm_amis_fused_split_host_f32,
epnp_lm_amis_fused_split_push_f32 and its copy kernel, push_split_kernel) on the CPU, under the cluster SIMT emulator
(tests/simt_cluster_native.py).  The host call must give lm_amis_fused_split's results bit for bit whatever the
chunking; the push call's peers must hold exactly the local rows at the global offset and nothing else; PushGather must
take the split push above the resident limit and assemble the single-process split result; every refusal of the host
call comes before its first copy."""
import contextlib
import socket

import pytest
import torch

import simt_cluster_native
import test_push_gather_cpu as _pg
from epropnp_b200 import native, sharded
from epropnp_b200.synth import make_problem

OUT_KEYS = ("pose_opt", "pose_cov", "cost", "logw", "pose_samples")


def _host_tensors_on_cpu(monkeypatch):
    # lm_amis_fused_split_host allocates its outputs pinned: there is no CUDA runtime here
    monkeypatch.setattr(torch, "empty", (lambda f: (lambda *a, pin_memory=False, **k: f(*a, **k)))(torch.empty))


def _case(B, N, dof, bounded, seed=8):
    pc = make_problem(B, N, seed=seed, dof=dof)
    delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
    lb, ub = ((pc["x2d"].amin(1) - 3.0).contiguous(), (pc["x2d"].amax(1) + 3.0).contiguous()) if bounded else (None, None)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], lb, ub, delta)
    host = dict(x3d=pc["x3d"], x2d=pc["x2d"], w2d=pc["w2d"], cam_mats=pc["cam_mats"].contiguous(), delta=delta,
                pose_init=pc["pose_init"], lb=lb, ub=ub)
    return prob, host, pc


@pytest.mark.parametrize("dof,ctas,bounded", [(6, 2, False), (6, 3, True), (4, 2, True), (4, 3, False),
                                               (6, 2, True), (6, 3, False), (4, 2, False), (4, 3, True)])
def test_split_host_call_is_the_device_split_call(monkeypatch, dof, ctas, bounded):
    """Every output bit for bit, for n_chunks = 0 (waves of 2 co-resident clusters: chunks of 2, 2, 1), 1, 3 and B."""
    simt_cluster_native.install(monkeypatch)
    _host_tensors_on_cpu(monkeypatch)
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "2")
    B, N = 5, 50 if dof == 6 else 37
    prob, host, pc = _case(B, N, dof, bounded)
    p = native.default_params(dof, lm_iter=3, mc_samples=16, mc_iter=2)
    ref = native.lm_amis_fused_split(prob, pc["pose_init"], p, seed=77, obj_offset=5, want_cost=True, cluster_ctas=ctas)
    ws = torch.empty(native.fused_workspace_bytes(B, N, p), dtype=torch.uint8)
    for n_chunks in (0, 1, 3, B):
        res = native.lm_amis_fused_split_host(host, p, ws, n_chunks=n_chunks, seed=77, obj_offset=5, cluster_ctas=ctas)
        for k in OUT_KEYS:
            assert torch.equal(res[k], ref[k]), (n_chunks, k)
    res = native.lm_amis_fused_split_host(host, p, ws, n_chunks=3, seed=77, obj_offset=5, cluster_ctas=ctas,
                                          want_samples=False)
    assert res["pose_samples"] is None
    for k in ("pose_opt", "pose_cov", "cost", "logw"):
        assert torch.equal(res[k], ref[k]), k


def test_split_host_call_leaves_a_skipped_output_unwritten(monkeypatch):
    """An output the caller passes as NULL (pose_samples, pose_cov, cost) is neither copied nor needed."""
    simt_cluster_native.install(monkeypatch)
    B, N, M = 3, 40, 8
    prob, host, pc = _case(B, N, 6, False, seed=3)
    p = native.default_params(6, lm_iter=2, mc_samples=M, mc_iter=2)
    ref = native.lm_amis_fused_split(prob, pc["pose_init"], p, seed=2, cluster_ctas=2)
    out = dict(pose_opt=torch.full((B, 7), -7.0), pose_cov=None, cost=None, logw=torch.full((B, M), -7.0),
               pose_samples=None)
    ws = torch.empty(native.fused_workspace_bytes(B, N, p), dtype=torch.uint8)
    native.lm_amis_fused_split_host(host, p, ws, n_chunks=2, seed=2, out=out, cluster_ctas=2)
    assert torch.equal(out["pose_opt"], ref["pose_opt"]) and torch.equal(out["logw"], ref["logw"])


@pytest.mark.parametrize("dof,N,M,ctas", [(6, 50, 16, 3), (4, 37, 12, 2), (6, 48, 10, 2)])
def test_split_push_with_stand_in_peers(monkeypatch, dof, N, M, ctas):
    """Peer rows [off, off + B) equal the local rows and lm_amis_fused_split's, bit for bit; the sentinel rows around
    them are untouched.  M = 10 at off = 3 puts the logw run off 16-byte alignment (the scalar copy loop)."""
    simt_cluster_native.install(monkeypatch)
    B, off, total = 5, 3, 11
    D = 7 if dof == 6 else 4
    prob, _, pc = _case(B, N, dof, False, seed=60 + dof)
    p = native.default_params(dof, lm_iter=3, mc_samples=M, mc_iter=2)
    ref = native.lm_amis_fused_split(prob, pc["pose_init"], p, seed=7, obj_offset=off, want_cost=True, cluster_ctas=ctas)
    full_lw = [torch.full((total, M), -7.0) for _ in range(3)]
    full_ps = [torch.full((total, D), -7.0) for _ in range(3)]
    out = native.lm_amis_fused_split_push(prob, pc["pose_init"], p, full_ps[0][off:off + B], full_lw[0][off:off + B],
                                          full_lw[1:], full_ps[1:], seed=7, obj_offset=off, want_cost=True,
                                          want_cov=True, cluster_ctas=ctas)
    for k in ("pose_samples", "cost", "pose_cov"):
        assert torch.equal(out[k], ref[k]), k
    for r in range(3):
        assert torch.equal(full_lw[r][off:off + B], ref["logw"]) and torch.equal(full_ps[r][off:off + B], ref["pose_opt"])
        for t in (full_lw[r], full_ps[r]):
            assert (t[:off] == -7.0).all() and (t[off + B:] == -7.0).all()


def test_split_push_without_peers_is_the_split_call(monkeypatch):
    simt_cluster_native.install(monkeypatch)
    prob, _, pc = _case(4, 40, 6, True, seed=3)
    p = native.default_params(6, lm_iter=2, mc_samples=8, mc_iter=2)
    ref = native.lm_amis_fused_split(prob, pc["pose_init"], p, seed=9, want_cost=True, want_cost_init=False)
    out = native.lm_amis_fused_split_push(prob, pc["pose_init"], p, torch.empty(4, 7), torch.empty(4, 8), [], [],
                                          seed=9, want_cost=True, want_cov=True)
    for k in OUT_KEYS:
        assert torch.equal(out[k], ref[k]), k


def test_split_host_refusals_come_before_any_copy(monkeypatch):
    """A short workspace, a cluster size of 1 or 9, a device without co-resident clusters and too many points: each is
    refused, and the workspace and the host outputs keep their sentinels: nothing was enqueued (every copy is
    synchronous here)."""
    simt_cluster_native.install(monkeypatch)
    M, I = 16, 2
    p = native.default_params(6, lm_iter=2, mc_samples=M, mc_iter=I)

    def attempt(N, match, cluster_ctas=0, short=False, push=False):
        B = 2
        prob, host, pc = _case(B, N, 6, False, seed=4)
        out = dict(pose_opt=torch.full((B, 7), -7.0), pose_cov=torch.full((B, 6, 6), -7.0), cost=torch.full((B,), -7.0),
                   logw=torch.full((B, M), -7.0), pose_samples=torch.full((B, M, 7), -7.0))
        if push:
            with pytest.raises(native.NativeError, match=match):
                native.lm_amis_fused_split_push(prob, pc["pose_init"], p, out["pose_opt"], out["logw"], [], [],
                                                cluster_ctas=cluster_ctas)
        else:
            ws = torch.full((native.fused_workspace_bytes(B, N, p) - (1 if short else 0),), 0xAB, dtype=torch.uint8)
            with pytest.raises(native.NativeError, match=match):
                native.lm_amis_fused_split_host(host, p, ws, n_chunks=0, out=out, cluster_ctas=cluster_ctas)
            assert (ws == 0xAB).all()                             # no input was copied in
        for k, t in out.items():
            assert (t == -7.0).all(), k

    attempt(40, "bad argument", short=True)
    for bad in (1, 9):
        attempt(40, "bad argument", cluster_ctas=bad)
        attempt(40, "bad argument", cluster_ctas=bad, push=True)
    too_many = native.max_points_split(6, M, I) + 64
    attempt(too_many, "shared memory")
    attempt(too_many, "shared memory", push=True)
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "0")
    attempt(40, "not supported")
    attempt(40, "not supported", push=True)


@pytest.mark.parametrize("limit,split", [(0, True), (10 ** 6, False)])
def test_push_gather_takes_the_split_push_exactly_above_the_resident_limit(monkeypatch, limit, split):
    monkeypatch.setattr(sharded, "_resident_limit", lambda dof, m, i: limit)
    prob = type("P", (), {"N": 40})()
    p = native.default_params(6, mc_samples=8, mc_iter=2)
    want = native.lm_amis_fused_split_push if split else native.lm_amis_fused_push
    assert sharded._push_call(prob, p) is want


def _push_split_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    from epropnp_b200 import capi
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.multiprocessing.set_sharing_strategy("file_system")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        capi._lib = simt_cluster_native.handle(())               # what simt_cluster_native.install does, without pytest
        native._need_cuda = lambda t, what: None
        native.stream_ptr = lambda device=None: None
        torch.cuda.device = lambda device=None: contextlib.nullcontext()
        calls = []
        split_push = native.lm_amis_fused_split_push
        native.lm_amis_fused_split_push = lambda *a, **k: calls.append(1) or split_push(*a, **k)
        sharded._resident_limit = lambda dof, m, i: 16           # below N: the split push
        per, N, M, depth = 3, 40, 8, 3
        num_obj = per * world
        p = native.default_params(6, lm_iter=2, mc_samples=M, mc_iter=2)
        pg = _pg._host_push_gather_class()(num_obj, M, 7, "cpu", depth=depth, valid_for=2)
        lo, hi = rank * per, (rank + 1) * per
        ok, pending, expected = True, None, None
        for step in range(2 * depth + 1):                         # every slot reused twice
            pc = make_problem(num_obj, N, seed=90 + step)
            delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5)
            whole = native.lm_amis_fused_split(
                native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, delta), pc["pose_init"], p,
                seed=step, want_cov=False, want_cost_init=False)
            mine = native.Problem(pc["x3d"][lo:hi], pc["x2d"][lo:hi], pc["w2d"][lo:hi], pc["cam_mats"][lo:hi], None, None,
                                  delta[lo:hi])
            out, nxt = pg.solve(mine, pc["pose_init"][lo:hi], p, seed=step)
            ok = ok and torch.equal(out["pose_samples"], whole["pose_samples"][lo:hi])
            if pending is not None:
                got = pending.wait()
                ok = ok and torch.equal(got["logw"], expected["logw"]) and torch.equal(got["pose_opt"], expected["pose_opt"])
            pending, expected = nxt, dict(logw=whole["logw"].clone(), pose_opt=whole["pose_opt"].clone())
        got = pending.wait()
        ok = ok and torch.equal(got["logw"], expected["logw"]) and torch.equal(got["pose_opt"], expected["pose_opt"])
        ok = ok and len(calls) == 2 * depth + 1
        dist.barrier()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_push_gather_split_two_processes_gloo():
    """Two gloo ranks with the resident limit lowered below N: PushGather routes through the split push, and every
    rank's assembled full-batch buffers equal the single-process lm_amis_fused_split of the whole batch."""
    import torch.multiprocessing as mp
    simt_cluster_native.build_emulated(())                         # build once, before the workers race for it
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_push_split_worker, args=(r, world, port, q)) for r in range(world)]
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
