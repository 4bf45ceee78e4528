"""The host-buffer and push forms of the cluster-split solve on the H100, at the dense coordinate maps they exist for
(N = 16,384 = 128 x 128): epnp_lm_amis_fused_split_host_f32 must give lm_amis_fused_split's results bit for bit on the
same inputs, whatever the chunking and cluster size; epnp_lm_amis_fused_split_push_f32 must put exactly the local rows
into every peer's buffers; sharded.PushGather must assemble the single-GPU split result bit for bit across two
processes; and the refusals above the split limit (and of the resident host / push calls at N = 16,384) stay."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

OUT_KEYS = ("pose_opt", "pose_cov", "cost", "logw", "pose_samples")


def _params(dof, M=512, I=4):
    return native.default_params(dof, lm_iter=3, fast_mode=1, z_min=0.01, mc_samples=M, mc_iter=I)


def _inputs(B, N, dof, seed, dev, bounded=False):
    pc = make_problem(B, N, seed=seed, dof=dof, grid2d=round(N ** 0.5) ** 2 == N)      # a dense map where N is square
    delta = native.adaptive_delta(pc["x2d"].to(dev), pc["w2d"].to(dev), 0.1).cpu()
    lb = ub = None
    if bounded:
        lb, ub = (pc["x2d"].amin(1) - 3.0).contiguous(), (pc["x2d"].amax(1) + 3.0).contiguous()
    host = dict(x3d=pc["x3d"], x2d=pc["x2d"], w2d=pc["w2d"], cam_mats=pc["cam_mats"].contiguous(), delta=delta,
                pose_init=pc["pose_init"], lb=lb, ub=ub)
    host = {k: (v.pin_memory() if v is not None else None) for k, v in host.items()}
    d = {k: (v.to(dev) if v is not None else None) for k, v in host.items()}
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], d["lb"], d["ub"], d["delta"])
    return host, prob, d["pose_init"]


def _host_vs_device(dev, dof, N, B, ctas, chunkings, bounded=False, seed=3):
    host, prob, p0 = _inputs(B, N, dof, seed, dev, bounded)
    p = _params(dof)
    ref = native.lm_amis_fused_split(prob, p0, p, seed=11, obj_offset=7, want_cost=True, cluster_ctas=ctas)
    ws = torch.empty(native.fused_workspace_bytes(B, N, p), dtype=torch.uint8, device=dev)
    for n_chunks in chunkings:
        res = native.lm_amis_fused_split_host(host, p, ws, n_chunks=n_chunks, seed=11, obj_offset=7, cluster_ctas=ctas)
        torch.cuda.synchronize()
        for k in OUT_KEYS:
            assert torch.equal(res[k], ref[k].cpu()), (N, ctas, n_chunks, k)
    assert torch.isfinite(ref["logw"]).all()


def test_host_split_at_out_res_128_every_chunking(cuda_device):
    """Automatic C (3) at N = 16,384, B = 200: n_chunks = 0 cuts at whole waves of co-resident clusters (several chunks
    at this B), 1 and 5 equal chunks; with bounds."""
    assert native.split_ctas(6, 16384, 512, 4) == 3
    _host_vs_device(cuda_device, 6, 16384, 200, 0, (0, 1, 5), bounded=True)


@pytest.mark.parametrize("ctas", [3, 4, 5, 6, 7, 8])
def test_host_split_every_cluster_size(cuda_device, ctas):
    _host_vs_device(cuda_device, 6, 16384, 24, ctas, (0, 5), seed=ctas)


def test_host_split_4dof_and_two_ctas(cuda_device):
    _host_vs_device(cuda_device, 4, 10004, 40, 0, (0, 1, 5))
    _host_vs_device(cuda_device, 6, 4096, 40, 2, (0, 1, 5))


def test_split_push_with_stand_in_peers_at_out_res_128(cuda_device):
    dev = cuda_device
    B, off, total, N, M = 12, 5, 29, 16384, 512
    _, prob, p0 = _inputs(B, N, 6, 21, dev)
    p = _params(6)
    ref = native.lm_amis_fused_split(prob, p0, p, seed=7, obj_offset=off, want_cost=True)
    full_lw = [torch.full((total, M), -7.0, device=dev) for _ in range(4)]
    full_ps = [torch.full((total, 7), -7.0, device=dev) for _ in range(4)]
    out = native.lm_amis_fused_split_push(prob, p0, p, full_ps[0][off:off + B], full_lw[0][off:off + B], full_lw[1:],
                                          full_ps[1:], seed=7, obj_offset=off, want_cost=True, want_cov=True)
    torch.cuda.synchronize()
    for k in ("pose_samples", "cost", "pose_cov"):
        assert torch.equal(out[k], ref[k]), k
    for r in range(4):
        assert torch.equal(full_lw[r][off:off + B], ref["logw"]) and torch.equal(full_ps[r][off:off + B], ref["pose_opt"])
        for t in (full_lw[r], full_ps[r]):
            assert (t[:off] == -7.0).all() and (t[off + B:] == -7.0).all()


def test_refusals_above_the_limits(cuda_device):
    """Above max_points_split both split calls refuse ("shared memory") and the host outputs keep their sentinels; the
    resident host and push calls still refuse N = 16,384."""
    dev = cuda_device
    p = _params(6)
    M = p.mc_samples

    def sentinels(B):
        pin = dict(pin_memory=True)
        return dict(pose_opt=torch.full((B, 7), -7.0, **pin), pose_cov=torch.full((B, 6, 6), -7.0, **pin),
                    cost=torch.full((B,), -7.0, **pin), logw=torch.full((B, M), -7.0, **pin),
                    pose_samples=torch.full((B, M, 7), -7.0, **pin))

    for N, host_call, push_call in ((native.max_points_split(6, M, 4) + 64, native.lm_amis_fused_split_host,
                                     native.lm_amis_fused_split_push),
                                    (16384, native.lm_amis_fused_host, native.lm_amis_fused_push)):
        B = 2
        host, prob, p0 = _inputs(B, N, 6, 1, dev)
        ws = torch.empty(native.fused_workspace_bytes(B, N, p), dtype=torch.uint8, device=dev)
        out = sentinels(B)
        with pytest.raises(native.NativeError, match="shared memory"):
            host_call(host, p, ws, n_chunks=0, out=out)
        torch.cuda.synchronize()
        if host_call is native.lm_amis_fused_split_host:
            for k, t in out.items():
                assert (t == -7.0).all(), k
        lw, ps = torch.full((B, M), -7.0, device=dev), torch.full((B, 7), -7.0, device=dev)
        with pytest.raises(native.NativeError, match="shared memory"):
            push_call(prob, p0, p, ps, lw, [], [])
        torch.cuda.synchronize()
        assert (lw == -7.0).all() and (ps == -7.0).all()


# ------------------------------------------------------------------------------------------------
# Two-rank PushGather at N = 16,384, with the harness of tests/test_push_gather_gpu.py: one rank per GPU over NCCL, or,
# on a single-GPU box, two processes sharing cuda:0 (rendezvous over gloo, stores into the other process's IPC-mapped
# buffers).
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q, one_device):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", 0 if one_device else rank)
    torch.cuda.set_device(dev)
    if one_device:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from epropnp_b200 import sharded
        from epropnp_b200.sharded import PushGather
        per, N, M = 16, 16384, 512
        num_obj = per * world
        p = _params(6, M, 4)
        assert sharded._push_call(type("Prob", (), {"N": N})(), p) is native.lm_amis_fused_split_push
        pg = PushGather(num_obj, M, 7, dev, depth=3, valid_for=2)
        ok, pending, expected = True, None, None
        lo, hi = rank * per, (rank + 1) * per
        for step in range(5):                                   # > depth: ring slots are reused
            pc = {k: v.to(dev) for k, v in make_problem(num_obj, N, seed=500 + step, grid2d=True).items()}
            delta = native.adaptive_delta(pc["x2d"], pc["w2d"], 0.1)
            whole = native.lm_amis_fused_split(native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None,
                                                              None, delta),
                                               pc["pose_init"], p, seed=40 + step, want_cov=False, want_cost_init=False)
            mine = native.Problem(pc["x3d"][lo:hi], pc["x2d"][lo:hi], pc["w2d"][lo:hi], pc["cam_mats"][lo:hi], None, None,
                                  delta[lo:hi])
            out, nxt = pg.solve(mine, pc["pose_init"][lo:hi], p, seed=40 + step)
            ok = ok and torch.equal(out["pose_samples"], whole["pose_samples"][lo:hi])
            if pending is not None:                             # overlapped use: read batch t-1 after starting batch t
                got = pending.wait()
                torch.cuda.synchronize()
                ok = ok and torch.equal(got["logw"], expected["logw"]) and torch.equal(got["pose_opt"], expected["pose_opt"])
            pending, expected = nxt, dict(logw=whole["logw"].clone(), pose_opt=whole["pose_opt"].clone())
        got = pending.wait()
        torch.cuda.synchronize()
        ok = ok and torch.equal(got["logw"], expected["logw"]) and torch.equal(got["pose_opt"], expected["pose_opt"])
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_push_gather_at_out_res_128_assembles_the_single_gpu_split_batch(cuda_device):
    world = 2
    one_device = torch.cuda.device_count() < 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, one_device)) for r in range(world)]
    try:
        for pr in procs:
            pr.start()
        results = [q.get(timeout=300) for _ in range(world)]
        for pr in procs:
            pr.join(timeout=60)
    finally:
        for pr in procs:
            if pr.is_alive():
                pr.terminate()
            pr.join()
    assert sorted(results) == [(r, True) for r in range(world)]
