"""The cluster-split kernels (amis_split_kernel, cost_split_kernel) on the CPU: pnp_kernels.cu under the cluster SIMT
emulator, which runs a thread-block cluster as its CTAs' fibers under one scheduler (tests/simt_cluster/cuda_runtime.h,
built by tests/simt_cluster_native.py).  Small
point sets with forced cluster sizes -- odd N, a short last rank, ranks without points -- against the fp64 oracle and
the resident kernels; the audit build (-DEPNP_SPLIT_AUDIT) checks that every rank ends with rank 0's costs,
log-densities and samples, and that rank 0 alone stores outputs; results do not depend on the fiber schedule."""
import ctypes

import pytest
import torch

import simt_cluster_native
import simt_native
import test_split_gpu as _sg
from epropnp_b200 import native
from epropnp_b200.synth import make_noise, make_problem

AUDIT = ("-DEPNP_SPLIT_AUDIT",)

# (dof, N, C): N = 50 on 3 CTAs -> 24 + 24 + 2 points; 37 on 5 -> 8 x 4 + 5 (odd, padded); 48 on 5 -> 16 x 3 + two
# empty ranks (and the TMA loader, N % 4 == 0); 64 on 2 -> 32 + 32.
CASES = [(6, 50, 3), (6, 37, 5), (6, 48, 5), (6, 64, 2), (4, 37, 2), (4, 50, 3)]


@pytest.mark.parametrize("dof,N,ctas", CASES)
def test_split_amis_against_oracle_and_resident(monkeypatch, dof, N, ctas):
    dev = simt_cluster_native.install(monkeypatch)
    # (seeds whose weights do not collapse onto one sample: there the refit's Cholesky fallback is decided by rounding,
    # for the resident kernel as much as for the split one)
    _sg.check_split_against_oracle(dev, dof, 2, N, 16, 2, ctas, seed=2, against_resident=True)


@pytest.mark.parametrize("dof,N,ctas", [(6, 50, 3), (6, 48, 5), (4, 37, 2)])
def test_split_cost_against_oracle_and_resident(monkeypatch, dof, N, ctas):
    dev = simt_cluster_native.install(monkeypatch)
    _sg.check_cost_split(dev, dof, 2, N, 600, ctas, seed=N)         # 600 poses: two tiles of 512


def _audit_run(monkeypatch, dof, N, ctas, B=2, M=16, I=2):
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    pc = make_problem(B, N, seed=31, dof=dof)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None,
                          native.adaptive_delta(pc["x2d"], pc["w2d"], 0.5))
    p = native.default_params(dof, lm_iter=3, mc_samples=M, mc_iter=I)
    counts = (ctypes.c_longlong * 16)()
    lib.simt_audit_reset()
    out = native.lm_amis_fused_split(prob, pc["pose_init"], p, seed=4, want_proposals=True, cluster_ctas=ctas)
    lib.simt_audit_read(counts)
    amis = list(counts)
    lib.simt_audit_reset()
    native.evaluate_cost_split(prob, out["pose_samples"].transpose(0, 1).contiguous(), dof, 0.1, cluster_ctas=ctas)
    lib.simt_audit_read(counts)
    return amis, list(counts), out


@pytest.mark.parametrize("dof,N,ctas", [(6, 50, 3), (6, 48, 5), (4, 37, 2)])
def test_ranks_agree_and_rank0_alone_writes(monkeypatch, dof, N, ctas):
    B, M, I, D = 2, 16, 2, 7 if dof == 6 else 4
    amis, cost, out = _audit_run(monkeypatch, dof, N, ctas, B, M, I)
    stores, mismatches = amis[:8], amis[8:]
    assert mismatches == [0] * 8                                    # costs, log-densities, samples: rank 0's bits
    assert stores[0] == B * (M + M * D + I * 19) and stores[1:] == [0] * 7
    assert cost[0] == B * M and cost[1:8] == [0] * 7
    assert torch.isfinite(out["logw"]).all()


def test_split_results_do_not_depend_on_fiber_schedule(monkeypatch):
    """Ascending, descending and random fiber orders across the whole cluster give the same bits: no rank consumes
    another rank's partial costs without the cluster barrier in between."""
    simt_cluster_native.install(monkeypatch, AUDIT)
    lib = simt_cluster_native.handle(AUDIT)
    try:
        lib.simt_set_schedule(0, 1)
        _, _, base = _audit_run(monkeypatch, 6, 50, 3)
        for mode, seed in ((1, 1), (2, 5)):
            lib.simt_set_schedule(mode, seed)
            amis, _, out = _audit_run(monkeypatch, 6, 50, 3)
            assert amis[8:] == [0] * 8
            for k in ("pose_samples", "logw", "proposals"):
                assert torch.equal(out[k], base[k]), (mode, k)
    finally:
        lib.simt_set_schedule(0, 1)


def test_split_plan_and_cluster_size_arguments(monkeypatch):
    """epnp_split_ctas is >= 2 and monotone in N; the split limits are at least 6 x the resident ones; a requested cluster
    size below the minimum or above 8 is a bad argument; a device that cannot co-schedule the cluster is refused before
    any launch."""
    simt_cluster_native.install(monkeypatch)
    for dof, M, I in ((6, 512, 4), (4, 512, 4), (6, 0, 0), (6, 128, 2)):
        top = native.max_points_split(dof, M, I)
        assert top >= 6 * native.max_points(dof, M, I)
        prev = 2
        for N in list(range(1, 2000, 97)) + list(range(2000, top + 1, 1531)) + [top]:
            c = native.split_ctas(dof, N, M, I)
            assert prev <= c <= 8, (dof, M, N, c)
            prev = c
        assert native.split_ctas(dof, top + 64, M, I) == 0
    assert native.split_ctas(6, 16384, 512, 4) >= 2
    assert native.split_ctas(5, 100, 0, 0) == 0 and native.split_ctas(6, 100, 510, 4) == 0
    pc = make_problem(1, 40, seed=2)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, 1.0)
    p = native.default_params(6, lm_iter=1, mc_samples=8, mc_iter=2)
    poses = pc["pose_init"][None]
    for bad in (1, 9, -1):
        with pytest.raises(native.NativeError, match="bad argument"):
            native.lm_amis_fused_split(prob, pc["pose_init"], p, cluster_ctas=bad)
        with pytest.raises(native.NativeError, match="bad argument"):
            native.evaluate_cost_split(prob, poses, 6, 0.1, cluster_ctas=bad)
    monkeypatch.setenv("SIMT_EMUL_CLUSTERS", "0")
    with pytest.raises(native.NativeError, match="not supported"):
        native.lm_amis_fused_split(prob, pc["pose_init"], p, want_cost=True)
    with pytest.raises(native.NativeError, match="not supported"):
        native.evaluate_cost_split(prob, poses, 6, 0.1)


def test_single_cta_emulator_refuses_split_calls(monkeypatch):
    """The single-CTA emulator build (tests/simt_emul) cannot run a cluster: the split calls report EPNP_ERR_UNSUPPORTED
    (after their argument checks), as a device without cluster support does, and launch nothing."""
    simt_native.install(monkeypatch)
    pc = make_problem(2, 40, seed=2)
    prob = native.Problem(pc["x3d"], pc["x2d"], pc["w2d"], pc["cam_mats"], None, None, 1.0)
    p = native.default_params(6, lm_iter=1, mc_samples=8, mc_iter=2)
    with pytest.raises(native.NativeError, match="not supported"):
        native.lm_amis_fused_split(prob, pc["pose_init"], p)
    with pytest.raises(native.NativeError, match="not supported"):
        native.evaluate_cost_split(prob, pc["pose_init"][None], 6, 0.1)
    with pytest.raises(native.NativeError, match="bad argument"):
        native.lm_amis_fused_split(prob, pc["pose_init"], p, cluster_ctas=9)
