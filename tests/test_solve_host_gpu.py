"""The host-buffer solve from scratch on an H100 (epnp_solve_host_f32, epnp_solve_split_host_f32): bit for bit the
composition of device calls it replaces, on pinned host tensors, for every chunking, at the reference's two inference
shapes and on the split form; and PushGather's per-rank flow from an initialiser with stand-in peers in one process."""
import pytest
import torch

from epropnp_b200 import native
from epropnp_b200.synth import make_problem

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _setup(B, N, dof, bounded=False, grid2d=False, seed=0):
    pc = make_problem(B, N, seed=seed, dof=dof, grid2d=grid2d)
    delta = native.adaptive_delta(pc["x2d"].to(DEV), pc["w2d"].to(DEV), 0.1)
    lb = ub = None
    if bounded:
        lb, ub = (pc["x2d"].amin(1) - 3.0).contiguous(), (pc["x2d"].amax(1) + 3.0).contiguous()
    pin = lambda t: None if t is None else t.contiguous().pin_memory()
    host = dict(x3d=pin(pc["x3d"]), x2d=pin(pc["x2d"]), w2d=pin(pc["w2d"]), cam_mats=pin(pc["cam_mats"]),
                delta=pin(delta.cpu()), lb=pin(lb), ub=pin(ub))
    d = lambda t: None if t is None else t.to(DEV)
    prob = native.Problem(d(pc["x3d"]), d(pc["x2d"]), d(pc["w2d"]), d(pc["cam_mats"]), d(lb), d(ub), delta)
    return prob, host


def composition(prob, init, p, seed, obj_offset, split=False, ctas=0):
    """The device calls the host solve composes, on device tensors."""
    dof = p.dof
    if init.kind == native.capi.INIT_RSLM:
        inds, start = native.rslm_draw(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.num_proposals, init.num_points, dof,
                                       eps=init.rslm.eps, seed=init.seed, obj_offset=obj_offset)
        pose0 = (native.rslm_split(prob, inds, start, init.rslm, cluster_ctas=ctas) if split else
                 native.rslm(prob, inds, start, init.rslm))["pose"]
    else:
        pose0 = (native.epnp_init_split(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.conf_quantile, cluster_ctas=ctas)
                 if split else native.epnp_init(prob.x3d, prob.x2d, prob.w2d, prob.cam, init.conf_quantile))
    if p.mc_samples == 0:
        return native.lm_solve(prob, pose0, p, want_cov=True, want_cost=True)
    fused = native.lm_amis_fused_split if split else native.lm_amis_fused
    extra = dict(cluster_ctas=ctas) if split else {}
    return fused(prob, pose0, p, seed=seed, obj_offset=obj_offset, want_cost=True, **extra)


def _check(prob, host, init, p, chunkings, split=False, ctas=0, seed=123, obj_offset=7):
    ref = composition(prob, init, p, seed, obj_offset, split, ctas)
    ws = torch.empty(native.solve_workspace_bytes(prob.B, prob.N, p, init), dtype=torch.uint8, device=DEV)
    keys = ("pose_opt", "pose_cov", "cost") + (("logw", "pose_samples") if p.mc_samples else ())
    for n_chunks in chunkings:
        if split:
            res = native.solve_split_host(host, p, ws, init=init, n_chunks=n_chunks, seed=seed, obj_offset=obj_offset,
                                          cluster_ctas=ctas)
        else:
            res = native.solve_host(host, p, ws, init=init, n_chunks=n_chunks, seed=seed, obj_offset=obj_offset)
        torch.cuda.synchronize()
        for k in keys:
            assert torch.equal(res[k], ref[k].cpu()), (n_chunks, k)


@pytest.mark.parametrize("M", [0, 128])
def test_det_inference_shape(M):
    """EPro-PnP-Det inference: 4DoF, N = 256, RSLM (P = 64, n = 16, 3 iterations), then LM 5 in fast mode; without
    AMIS, and with AMIS 128 x 4; B odd."""
    prob, host = _setup(1023, 256, 4, bounded=True, seed=1)
    init = native.rslm_spec(4, num_points=16, num_proposals=64, num_iter=3, seed=99, fast_mode=1)
    p = native.default_params(4, lm_iter=5, fast_mode=1, mc_samples=M, mc_iter=4 if M else 0)
    _check(prob, host, init, p, (0, 1, 3, 8, 64))


@pytest.mark.parametrize("M", [0, 512])
def test_6dof_test_shape(M):
    """EPro-PnP-6DoF test loop: a dense 64 x 64 map, EPnP on the 0.8 confidence quantile, then GN(3); without AMIS, and
    with AMIS 512 x 4."""
    prob, host = _setup(63, 64 * 64, 6, grid2d=True, seed=2)
    p = native.default_params(6, lm_iter=3, fast_mode=1, mc_samples=M, mc_iter=4 if M else 0)
    _check(prob, host, native.epnp_spec(0.8), p, (0, 1, 3, 8, 63))


@pytest.mark.parametrize("kind,ctas", [("epnp", 0), ("epnp", 8), ("rslm", 0), ("rslm", 8)])
def test_split_form_at_16384_points(kind, ctas):
    prob, host = _setup(24, 16384, 6, seed=3)
    init = native.epnp_spec(0.8) if kind == "epnp" else native.rslm_spec(6, seed=5)
    p = native.default_params(6, lm_iter=5, mc_samples=512, mc_iter=4)
    _check(prob, host, init, p, (0, 1, 3, 24), split=True, ctas=ctas)


def test_given_pose_is_the_fused_host_call():
    prob, host = _setup(257, 128, 6, seed=4)
    host["pose_init"] = make_problem(257, 128, seed=4)["pose_init"].pin_memory()
    p = native.default_params(6, lm_iter=5, mc_samples=256, mc_iter=4)
    ws = torch.empty(native.solve_workspace_bytes(257, 128, p), dtype=torch.uint8, device=DEV)
    for n_chunks in (0, 8):
        ref = native.lm_amis_fused_host(host, p, ws, n_chunks=n_chunks, seed=3)
        torch.cuda.synchronize()                  # the call is asynchronous: its outputs are final only now
        ref = {k: v.clone() for k, v in ref.items() if v is not None}
        res = native.solve_host(host, p, ws, n_chunks=n_chunks, seed=3)
        torch.cuda.synchronize()
        for k in ref:
            assert torch.equal(res[k], ref[k]), (n_chunks, k)


@pytest.mark.parametrize("kind", ["rslm", "epnp"])
def test_push_from_initialiser_with_stand_in_peers(kind):
    """What PushGather.solve(init=...) runs on each rank -- initial_pose on its shard at obj_offset = lo, then the push
    call -- for two ranks in one process, each pushing into the other's full-batch buffers on the same device."""
    B, N, M, world = 192, 64, 128, 2
    prob, _ = _setup(B, N, 6, seed=6)
    init = native.epnp_spec(0.8) if kind == "epnp" else native.rslm_spec(6, seed=8)
    p = native.default_params(6, lm_iter=5, mc_samples=M, mc_iter=4)
    whole = composition(prob, init, p, seed=17, obj_offset=0)
    full_lw = [torch.full((B, M), float("nan"), device=DEV) for _ in range(world)]
    full_ps = [torch.full((B, 7), float("nan"), device=DEV) for _ in range(world)]
    per = B // world
    for r in range(world):
        lo, hi = r * per, (r + 1) * per
        mine = native.Problem(prob.x3d[lo:hi], prob.x2d[lo:hi], prob.w2d[lo:hi], prob.cam[lo:hi], None, None,
                              prob.delta[lo:hi])
        pose0 = native.initial_pose(mine, init, 6, obj_offset=lo)
        others = [q for q in range(world) if q != r]
        out = native.lm_amis_fused_push(mine, pose0, p, full_ps[r][lo:hi], full_lw[r][lo:hi],
                                        [full_lw[q] for q in others], [full_ps[q] for q in others], seed=17,
                                        obj_offset=lo)
        assert torch.equal(out["pose_samples"], whole["pose_samples"][lo:hi])
    torch.cuda.synchronize()
    for q in range(world):
        assert torch.equal(full_lw[q], whole["logw"]) and torch.equal(full_ps[q], whole["pose_opt"])
