/* C host of the host-buffer solve from scratch (epnp_solve_host_f32): the two default inference flows of the reference
 * from correspondences in host memory.  Needs no GPU to run the checks in main() (layout of EpnpInit, workspace query,
 * argument refusals and an empty batch, all before any CUDA call); det_inference() and dof6_test_inference() show the
 * calls a deployment makes with a device (workspace from cudaMalloc, pinned host buffers for full speed).
 *
 *   gcc -std=c99 -Iinclude examples/host_solve_c.c -o host_solve_c -Lepro-pnp_b200/lib -lepropnp_b200 \
 *       -Wl,-rpath,epro-pnp_b200/lib
 */
#include <stddef.h>
#include <stdio.h>

#include "epropnp_b200.h"

/* EPro-PnP-Det inference: RSLM (P = 64, n = 16, 3 GN iterations), then LM 5 in fast mode, no AMIS.
 * pose (B, 4) = x y z yaw, cov (B, 4, 4); workspace of epnp_solve_workspace_bytes(B, N, &p, &init) bytes. */
int det_inference(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* delta,
                  uint64_t rslm_seed, float* pose, float* cov, void* workspace, size_t workspace_bytes, int B, int N,
                  void* stream) {
    EpnpParams p;
    EpnpInit init = {0};
    epnp_default_params(&p, 4);
    p.lm_iter = 5; p.fast_mode = 1; p.mc_samples = 0;
    init.kind = EPNP_INIT_RSLM; init.num_proposals = 64; init.num_points = 16; init.seed = rslm_seed;
    epnp_default_params(&init.rslm, 4);
    init.rslm.lm_iter = 3; init.rslm.fast_mode = 1;
    return epnp_solve_host_f32(x3d, x2d, w2d, cam, NULL, NULL, delta, NULL, &init, 0, 0, pose, cov, NULL, NULL, NULL,
                               workspace, workspace_bytes, 0, B, N, &p, stream);
}

/* EPro-PnP-6DoF test loop: EPnP on the points at or above the 0.8 confidence quantile, then GN(3), no AMIS. */
int dof6_test_inference(const float* x3d, const float* x2d, const float* w2d, const float* cam, const float* delta,
                        float* pose, void* workspace, size_t workspace_bytes, int B, int N, void* stream) {
    EpnpParams p;
    EpnpInit init = {0};
    epnp_default_params(&p, 6);
    p.lm_iter = 3; p.fast_mode = 1; p.mc_samples = 0;
    init.kind = EPNP_INIT_EPNP; init.conf_quantile = 0.8f;
    return epnp_solve_host_f32(x3d, x2d, w2d, cam, NULL, NULL, delta, NULL, &init, 0, 0, pose, NULL, NULL, NULL, NULL,
                               workspace, workspace_bytes, 0, B, N, &p, stream);
}

int main(void) {
    int failures = 0;
    EpnpParams p;
    EpnpInit rslm = {0}, epnp = {0}, bad = {0};
    static float in[4096], out[4096];
    float* ws = out;                             /* never dereferenced: every call below returns before any copy */

    if (sizeof(EpnpInit) != 96 || offsetof(EpnpInit, seed) != 16 || offsetof(EpnpInit, rslm) != 32) ++failures;
    epnp_default_params(&p, 6);
    p.mc_samples = 0;
    rslm.kind = EPNP_INIT_RSLM; rslm.num_proposals = 64; rslm.num_points = 16;
    epnp_default_params(&rslm.rslm, 6);
    epnp.kind = EPNP_INIT_EPNP; epnp.conf_quantile = 0.8f;

    /* workspace: the fused layout, plus the RSLM hypotheses' (P, B, .) scratch; 0 for what no call takes */
    const size_t base = epnp_solve_workspace_bytes(1024, 256, &p, NULL);
    const size_t with_rslm = epnp_solve_workspace_bytes(1024, 256, &p, &rslm);
    if (base != epnp_fused_workspace_bytes(1024, 256, &p) || epnp_solve_workspace_bytes(1024, 256, &p, &epnp) != base)
        ++failures;
    if (with_rslm < base + (size_t)64 * 1024 * 16 * 4) ++failures;
    if (epnp_solve_workspace_bytes(1024, 256, &p, &bad) != 0 || epnp_solve_workspace_bytes(-1, 256, &p, NULL) != 0)
        ++failures;
    printf("workspace for B=1024 N=256: %zu bytes, %zu with RSLM (P=64, n=16)\n", base, with_rslm);

#define SOLVE(pose_init, init, logw, B, N, par) \
    epnp_solve_host_f32(in, in, in, in, NULL, NULL, in, (pose_init), (init), 0, 0, out, NULL, NULL, NULL, (logw), ws, \
                        (size_t)1 << 40, 0, (B), (N), (par), NULL)
    if (SOLVE(in, &rslm, NULL, 2, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;      /* both starts */
    if (SOLVE(NULL, NULL, NULL, 2, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;     /* neither */
    if (SOLVE(NULL, &bad, NULL, 2, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;     /* unknown kind */
    if (SOLVE(NULL, &rslm, out, 2, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;     /* logw without AMIS */
    epnp.conf_quantile = 1.5f;
    if (SOLVE(NULL, &epnp, NULL, 0, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;    /* the EPnP call's own refusal */
    epnp.conf_quantile = 0.8f;
    p.dof = 4;
    if (SOLVE(NULL, &epnp, NULL, 2, 64, &p) != EPNP_ERR_BAD_ARG) ++failures;    /* EPnP gives 6DoF poses only */
    p.dof = 6;
    if (SOLVE(NULL, &epnp, NULL, 0, 64, &p) != EPNP_OK) ++failures;             /* an empty batch: nothing to do */
    if (SOLVE(NULL, &rslm, NULL, 0, 64, &p) != EPNP_OK) ++failures;
#undef SOLVE
    printf("%s\n", failures ? "FAILED" : "ok");
    return failures;
}
