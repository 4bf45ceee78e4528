"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the EPro-PnP hot path (LM/GN solve + AMIS loop).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this file, and only as the checker / the reported CPU baseline -- never as a product path.

It restates, as plain batched torch functions (no classes, no in-place masks, noise passed in),
the algorithm of the reference files listed below.  Pinning: tests/test_oracle_cpu.py checks this
file against tests/golden/*.npz, which oracle/make_golden.py produced by running the UNMODIFIED
reference (/root/reference/epropnp) in this container -- in float64 the two agree to ~1e-9, so
the algorithm is the same; in float32 they agree to float32 rounding.  The single piece that is
NOT pinned by reference-owned code is the multivariate Student-t (pyro-ppl, un-vendored): its
density is cross-checked against scipy.stats.multivariate_t instead ("parity unpinned" for pyro).

Reference map (file:line under /root/reference/epropnp/):
    quat_to_rotmat / yaw_to_rotmat        common.py:22-64
    project, jacobian, clip mask           camera.py:10-30, 64-143
    quat_tangent_map                       camera.py:145-165
    huber cost / robust rescale            cost_fun.py:8-20, 33-89
    adaptive_delta                         cost_fun.py:123-126
    evaluate                               common.py:67-100
    lm_solve (LM + GN fast mode)           levenberg_marquardt.py:80-241
    gn_step / pose_add                     levenberg_marquardt.py:243-265
    normalize / denormalize                common.py:103-136
    center_based_init / rslm_solve / select_start   levenberg_marquardt.py:283-353, 115-130
    robust_cholesky                        epropnp.py:16-33
    amis_6dof (initial fit, mixture, refit) epropnp.py:87-196, 282-342
    amis_4dof (von Mises / uniform yaw)     epropnp.py:199-260; distributions.py:55-79; torch VonMises
    acg_logpdf / acg sample                distributions.py:32-52
    mvt_logpdf / mvt sample                pyro.distributions.MultivariateStudentT (see pyro_shim)
"""
import math
from dataclasses import dataclass
from typing import Union

import torch

Bound = Union[None, float, torch.Tensor]


@dataclass
class Camera:
    cam_mats: torch.Tensor            # (B, 3, 3)
    z_min: float = 0.1
    lb: Bound = None                  # None | float | (B, 2)
    ub: Bound = None


@dataclass
class LMParams:
    num_iter: int = 10
    min_lm_diagonal: float = 1e-6
    max_lm_diagonal: float = 1e32
    min_relative_decrease: float = 1e-3
    initial_trust_region_radius: float = 30.0
    max_trust_region_radius: float = 1e16
    eps: float = 1e-5


# ----------------------------------------------------------------------------- rotations
def quat_to_rotmat(q):
    w, x, y, z = q.unbind(-1)
    ww, xx, yy, zz = w * w, x * x, y * y, z * z
    r = torch.stack((
        ww + xx - yy - zz, 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), ww - xx + yy - zz, 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), ww - xx - yy + zz), dim=-1)
    return r.reshape(q.shape[:-1] + (3, 3))


def yaw_to_rotmat(yaw):
    c, s = torch.cos(yaw), torch.sin(yaw)
    o, z = torch.ones_like(yaw), torch.zeros_like(yaw)
    return torch.stack((c, z, s, z, o, z, -s, z, c), dim=-1).reshape(yaw.shape + (3, 3))


def pose_rotmat(pose):
    return yaw_to_rotmat(pose[..., 3]) if pose.shape[-1] == 4 else quat_to_rotmat(pose[..., 3:])


def quat_tangent_map(q):
    """(..., 4) -> (..., 4, 3): dq = T(q) d, the local rotation increment embedded in R^4."""
    w, x, y, z = q.unbind(-1)
    t = torch.stack((x, y, z, -w, -z, y, z, -w, -x, -y, x, -w), dim=-1)
    return t.reshape(q.shape[:-1] + (4, 3))


def pose_add(pose, step):
    if pose.shape[-1] == 4:
        return pose + step
    q = pose[..., 3:]
    qn = q + (quat_tangent_map(q) @ step[..., 3:, None]).squeeze(-1)
    qn = qn / qn.norm(dim=-1, keepdim=True).clamp(min=1e-12)
    return torch.cat((pose[..., :3] + step[..., :3], qn), dim=-1)


# ----------------------------------------------------------------------------- per-point math
def _bound(b, like):
    if b is None:
        return None
    if torch.is_tensor(b):
        return b.to(like.dtype).unsqueeze(-2)          # (B, 1, 2)
    return torch.as_tensor(float(b), dtype=like.dtype)


def evaluate(x3d, x2d, w2d, pose, cam: Camera, delta, want_jac=False, clip_jac=True,
             eps_huber=1e-10):
    """pose (*, B, D) broadcasts against x3d (B, N, 3).
    Returns dict(cost (*,B), residual (*,B,2N) | None, jac (*,B,2N,dof) | None)."""
    dof = 4 if pose.shape[-1] == 4 else 6
    K = cam.cam_mats
    R = pose_rotmat(pose)                                   # (*, B, 3, 3)
    if want_jac:                                            # camera.py:10-18 (rotate, translate, then K)
        x_rot = x3d @ R.transpose(-1, -2)                   # (*, B, N, 3)
        xh = (x_rot + pose[..., None, :3]) @ K.transpose(-1, -2)
    else:                                                   # camera.py:21-30 (K R and K t folded once per pose)
        xh = x3d @ (K @ R).transpose(-1, -2) + (K @ pose[..., :3, None]).squeeze(-1).unsqueeze(-2)
    z = xh[..., 2:3].clamp(min=cam.z_min)
    u = xh[..., :2] / z
    lb, ub = _bound(cam.lb, u), _bound(cam.ub, u)
    bounded = lb is not None and ub is not None
    if bounded:
        u = torch.minimum(torch.maximum(u, lb), ub)

    if not torch.is_tensor(delta):
        delta = torch.as_tensor(float(delta), dtype=x2d.dtype)
    delta = delta.to(x2d.dtype)[..., None]                  # (B, 1) or (1,)
    r = (u - x2d) * w2d
    s = r.norm(dim=-1)                                      # (*, B, N)
    half_rho = torch.where(s <= delta, 0.5 * s * s, delta * s - 0.5 * delta * delta)
    out = dict(cost=half_rho.sum(-1), residual=None, jac=None)
    if not want_jac:
        return out

    scale = (delta / s.clamp(min=eps_huber)).clamp(max=1.0).sqrt()          # sqrt(rho')
    out["residual"] = (r * scale[..., None]).flatten(-2)
    # d u / d x_cam  (2x3), using the first two rows of K only (camera.py:137-140)
    Kb = K[..., None, :, :]                                 # (B, 1, 3, 3)
    j_xy = Kb[..., :2, :2] / z[..., None]
    j_z = (Kb[..., :2, 2:3] - u[..., None]) / z[..., None]
    j3 = torch.cat((j_xy, j_z), dim=-1)                     # (*, B, N, 2, 3)
    if dof == 6:
        a = 2 * x_rot
        zero = torch.zeros_like(a[..., 0])
        sk = torch.stack((zero, -a[..., 2], a[..., 1],
                          a[..., 2], zero, -a[..., 0],
                          -a[..., 1], a[..., 0], zero), dim=-1).reshape(a.shape[:-1] + (3, 3))
        j_rot = j3 @ sk
    else:
        j_rot = j3[..., 0:1] * x_rot[..., None, 2:3] - j3[..., 2:3] * x_rot[..., None, 0:1]
    jac = torch.cat((j3, j_rot), dim=-1)                    # (*, B, N, 2, dof)
    if clip_jac:
        mask = (z == cam.z_min)
        if bounded:
            mask = mask | (u == lb) | (u == ub)
        else:
            mask = mask.expand(u.shape)
        jac = jac * (~mask)[..., None].to(jac.dtype)
    jac = jac * (w2d * scale[..., None])[..., None]
    out["jac"] = jac.flatten(-3, -2)
    return out


def adaptive_delta(x2d, w2d, relative_delta):
    std = x2d.var(dim=-2, unbiased=True).sum(-1).sqrt()
    return w2d.mean(dim=(-2, -1)) * std * relative_delta


def normalize_points(x3d, pose):
    off = x3d.mean(dim=-2)
    x3d_n = x3d - off[..., None, :]
    pose_n = None
    if pose is not None:
        pose_n = pose.clone()
        pose_n[..., :3] = pose[..., :3] + (pose_rotmat(pose) @ off[..., None]).squeeze(-1)
    return off, x3d_n, pose_n


def denormalize_pose(off, pose_n):
    pose = pose_n.clone()
    pose[..., :3] = pose_n[..., :3] - (pose_rotmat(pose_n) @ off[..., None]).squeeze(-1)
    return pose


# ----------------------------------------------------------------------------- LM / GN
def _normal_eq(e):
    J, r = e["jac"], e["residual"]
    Jt = J.transpose(-1, -2)
    return Jt @ J, (Jt @ r[..., None]).squeeze(-1)


def lm_solve(x3d, x2d, w2d, cam: Camera, delta, pose_init, prm: LMParams = LMParams(),
             fast_mode=False):
    """Returns pose_opt (B,D), pose_cov (B,dof,dof), cost (B)."""
    dof = 4 if pose_init.shape[-1] == 4 else 6
    pose = pose_init.clone()
    eye = torch.eye(dof, dtype=x2d.dtype)
    ev = lambda p: evaluate(x3d, x2d, w2d, p, cam, delta, want_jac=True, clip_jac=not fast_mode)
    if fast_mode:
        for _ in range(prm.num_iter):
            e = ev(pose)
            jtj, g = _normal_eq(e)
            jtj = jtj + prm.eps * eye
            cost = e["cost"]
            pose = pose_add(pose, -torch.linalg.solve(jtj, g))
        return pose, torch.linalg.inv(jtj), cost

    cur = ev(pose)
    jtj, g = _normal_eq(cur)
    cost = cur["cost"]
    B = pose.shape[0]
    radius = x2d.new_full((B,), prm.initial_trust_region_radius)
    shrink = x2d.new_full((B,), 2.0)
    for _ in range(prm.num_iter):
        d = torch.diagonal(jtj, dim1=-2, dim2=-1)
        damp = d.clamp(min=prm.min_lm_diagonal, max=prm.max_lm_diagonal) / radius[:, None] + prm.eps
        step = -torch.linalg.solve(jtj + torch.diag_embed(damp), g)
        pose_new = pose_add(pose, step)
        new = ev(pose_new)
        model_change = -(step * ((jtj @ step[..., None]).squeeze(-1) / 2 + g)).sum(-1)
        rho = (cost - new["cost"]) / model_change
        ok = (rho >= prm.min_relative_decrease) & (model_change > 0.0)
        # accepted
        pose = torch.where(ok[:, None], pose_new, pose)
        grow = radius / (1.0 - (2.0 * rho - 1.0) ** 3).clamp(min=1.0 / 3.0)
        radius = torch.where(ok, grow, radius).clamp(max=prm.max_trust_region_radius, min=prm.eps)
        # rejected
        radius = torch.where(ok, radius, radius / shrink)
        shrink = torch.where(ok, torch.full_like(shrink, 2.0), shrink * 2.0)
        jtj_new, g_new = _normal_eq(new)
        jtj = torch.where(ok[:, None, None], jtj_new, jtj)
        g = torch.where(ok[:, None], g_new, g)
        cost = torch.where(ok, new["cost"], cost)
    return pose, torch.linalg.inv(jtj + prm.eps * eye), cost


def gn_step(x3d, x2d, w2d, cam: Camera, delta, pose, eps=1e-5):
    e = evaluate(x3d, x2d, w2d, pose, cam, delta, want_jac=True, clip_jac=True)
    jtj, g = _normal_eq(e)
    jtj = jtj + eps * torch.eye(jtj.shape[-1], dtype=jtj.dtype)
    return -torch.linalg.solve(jtj, g)


# ----------------------------------------------------------------------------- random-sample LM initialiser
def center_based_init(x2d, x3d, cam: Camera, dof, eps=1e-6):
    """Translation guess from the spread of the back-projected 2D points against the spread of the 3D points
    (levenberg_marquardt.py:283-298)."""
    homo = torch.cat((x2d, torch.ones_like(x2d[..., :1])), dim=-1)
    rays = torch.linalg.solve(cam.cam_mats, homo.transpose(-1, -2)).transpose(-1, -2)
    rays = rays[..., :2] / rays[..., 2:].clamp(min=eps)
    r_std, r_mean = rays.std(dim=-2), rays.mean(dim=-2)
    o_std = x3d.std(dim=-2)
    if dof == 4:
        depth = o_std[..., 1] / r_std[..., 1].clamp(min=eps)
    else:
        depth = math.sqrt(2 / 3) * o_std.norm(dim=-1) / r_std.norm(dim=-1).clamp(min=eps)
    return torch.cat((r_mean, torch.ones_like(r_mean[..., :1])), dim=-1) * depth[..., None]


def rslm_solve(x3d, x2d, w2d, cam: Camera, delta, inds, start, prm: LMParams = LMParams(num_iter=3), fast_mode=False):
    """RSLMSolver.solve (levenberg_marquardt.py:300-353) with the random draws passed in: `inds` (P, B, n) are the
    sampled correspondences of every hypothesis, `start` (P, B, D) the starting poses.  Every hypothesis is an
    LM / GN solve of its n-point mini-problem, scored on the full set; the cheapest wins per object.
    Returns dict(hyp_pose (P,B,D), hyp_cost (P,B), pose (B,D), cost (B), winner (B))."""
    P, B, n = inds.shape
    idx = inds.long()[..., None]                                              # (P, B, n, 1)
    gather = lambda t: torch.gather(t[None].expand(P, *t.shape), 2, idx.expand(P, B, n, t.shape[-1])).reshape(P * B, n, -1)
    rep = lambda t: t if not torch.is_tensor(t) or t.dim() == 0 else t[None].expand(P, *t.shape).reshape(P * B, *t.shape[1:])
    cam_p = Camera(rep(cam.cam_mats), cam.z_min, rep(cam.lb), rep(cam.ub))
    pose, _, _ = lm_solve(gather(x3d), gather(x2d), gather(w2d), cam_p, rep(delta), start.reshape(P * B, -1), prm,
                          fast_mode=fast_mode)
    pose = pose.reshape(P, B, -1)
    cost = evaluate(x3d, x2d, w2d, pose, cam, delta)["cost"]                 # (P, B)
    min_cost, winner = cost.min(dim=0)
    return dict(hyp_pose=pose, hyp_cost=cost, pose=pose[winner, torch.arange(B)], cost=min_cost, winner=winner)


def select_start(pose_init, cost_init, pose_rs, cost_rs):
    """force_init_solve (levenberg_marquardt.py:120-128): keep pose_init where it is strictly cheaper."""
    return torch.where((cost_init < cost_rs)[:, None], pose_init, pose_rs)


# ----------------------------------------------------------------------------- small linear algebra
def robust_cholesky(mat, default_diag=None):
    """Batched lower Cholesky; a matrix that is not positive definite gets diag(default) (or I)."""
    n = mat.shape[-1]
    flat = mat.reshape(-1, n, n)
    L, info = torch.linalg.cholesky_ex(flat)
    bad = info != 0
    if bad.any():
        dflt = torch.diag(mat.new_tensor(default_diag)) if default_diag is not None else \
            torch.eye(n, dtype=mat.dtype)
        L = torch.where(bad[:, None, None], dflt, L)
    return L.reshape(mat.shape)


def _tri_solve(L, v):
    """L (..., n, n) lower, v (..., n) -> L^-1 v, broadcasting batch dims."""
    shape = torch.broadcast_shapes(L.shape[:-2], v.shape[:-1])
    Lb = L.expand(shape + L.shape[-2:])
    vb = v.expand(shape + v.shape[-1:])
    return torch.linalg.solve_triangular(Lb, vb[..., None], upper=False).squeeze(-1)


def mvt_logpdf(x, loc, L, df=3.0):
    n = loc.shape[-1]
    y = _tri_solve(L, x - loc)
    log_norm = (L.diagonal(dim1=-2, dim2=-1).log().sum(-1) + 0.5 * n * math.log(df * math.pi)
                + math.lgamma(0.5 * df) - math.lgamma(0.5 * (df + n)))
    return -0.5 * (df + n) * torch.log1p(y.square().sum(-1) / df) - log_norm


def acg_logpdf(x, L):
    q = L.shape[-1]
    y = _tri_solve(L, x)
    area = 2 * math.pi ** (0.5 * q) / math.gamma(0.5 * q)
    return -0.5 * q * y.square().sum(-1).log() - L.diagonal(dim1=-2, dim2=-1).log().sum(-1) - math.log(area)


def mvt_draw(normal3, chi2, loc, L, df=3.0):
    y = normal3 * torch.rsqrt(chi2 / df)[..., None]
    return loc + (L @ y[..., None]).squeeze(-1)


def acg_draw(normal4, L, eps=1e-6):
    g = (L @ normal4[..., None]).squeeze(-1)
    nrm = g.norm(dim=-1, keepdim=True)
    unit = torch.zeros_like(g)
    unit[..., 0] = 1.0
    return torch.where(nrm < eps, unit, g / nrm)


# ----------------------------------------------------------------------------- AMIS (6DoF)
def amis_6dof(x3d, x2d, w2d, cam: Camera, delta, pose_opt, pose_cov, noise, mc_samples=512,
              num_iter=4, eps=1e-5, acg_mle_iter=3, acg_dispersion=1e-3, return_refit=False):
    """noise = (normal3 (I,S,B,3), chi2 (I,S,B), normal4 (I,S,B,4)).
    Returns dict(samples (M,B,7), logw (M,B), trans_mode (I,B,3), trans_tril (I,B,3,3),
    rot_tril (I,B,4,4), cost (I,S,B)).  return_refit: also refit_trans (I-1,B,3,3) and refit_rot (I-1,B,4,4), the
    matrices each refit hands to robust_cholesky (the weighted translation covariance; the dispersed ACG scatter), and
    refit_logw, per refit the log-weights ((i+1)S,B) it weighs the samples by."""
    n3, c2, n4 = noise
    I, S = num_iter, mc_samples // num_iter
    B, dt = x3d.shape[0], x3d.dtype
    eye4 = torch.eye(4, dtype=dt)
    mode = torch.zeros(I, B, 3, dtype=dt)
    Lt = torch.zeros(I, B, 3, 3, dtype=dt)
    Lr = torch.zeros(I, B, 4, 4, dtype=dt)

    refit_t, refit_r, refit_w = [], [], []

    def dispersed(c):
        return c + torch.linalg.det(c)[:, None, None] ** 0.25 * (acg_dispersion * eye4)

    # proposal 0 from the local solution and its covariance
    mode[0] = pose_opt[:, :3]
    Lt[0] = robust_cholesky(pose_cov[:, :3, :3])
    T = quat_tangent_map(pose_opt[:, 3:])
    rc = torch.linalg.inv(T @ torch.linalg.inv(pose_cov[:, 3:, 3:]) @ T.transpose(-1, -2) + eye4)
    rc = rc / rc.diagonal(dim1=-2, dim2=-1).sum(-1)[:, None, None]
    Lr[0] = robust_cholesky(dispersed(rc))

    samples = torch.zeros(I, S, B, 7, dtype=dt)
    cost = torch.zeros(I, S, B, dtype=dt)
    logp = torch.zeros(I, I, S, B, dtype=dt)          # [proposal j, sample batch k]
    logw = None
    for i in range(I):
        samples[i, ..., :3] = mvt_draw(n3[i], c2[i], mode[i], Lt[i])
        samples[i, ..., 3:] = acg_draw(n4[i], Lr[i])
        cost[i] = evaluate(x3d, x2d, w2d, samples[i], cam, delta)["cost"]
        # newest proposal on every sample so far, older proposals on the newest samples
        logp[i, :i + 1] = mvt_logpdf(samples[:i + 1, ..., :3], mode[i], Lt[i]) \
            + acg_logpdf(samples[:i + 1, ..., 3:], Lr[i])
        if i > 0:
            logp[:i, i] = mvt_logpdf(samples[i, ..., :3], mode[:i, None], Lt[:i, None]) \
                + acg_logpdf(samples[i, ..., 3:], Lr[:i, None])
        mix = torch.logsumexp(logp[:i + 1, :i + 1], dim=0) - math.log(i + 1)
        logw = -cost[:i + 1] - mix                                  # (i+1, S, B)
        if i == I - 1:
            break
        # refit the next proposal to the weighted samples
        refit_w.append(logw.reshape(-1, B))
        w = torch.softmax(refit_w[-1], dim=0)                       # (n, B)
        smp = samples[:i + 1].reshape(-1, B, 7)
        t, q = smp[..., :3], smp[..., 3:]
        mode[i + 1] = (w[..., None] * t).sum(0)
        dev = t - mode[i + 1]
        refit_t.append((w[..., None, None] * dev[..., :, None] * dev[..., None, :]).sum(0))
        Lt[i + 1] = robust_cholesky(refit_t[-1])
        qq = q[..., :, None] * q[..., None, :]
        lam = eye4.expand(B, 4, 4).clone()
        for _ in range(acg_mle_iter):
            m = (q[..., None, :] @ torch.linalg.inv(lam) @ q[..., :, None]).reshape(-1, B)
            wm = w / m.clamp(min=eps)
            wm = wm / wm.sum(0)
            lam = (wm[..., None, None] * qq).sum(0) + eps * eye4
        refit_r.append(dispersed(lam))
        Lr[i + 1] = robust_cholesky(refit_r[-1])
    out = dict(samples=samples.reshape(I * S, B, 7), logw=logw.reshape(I * S, B), trans_mode=mode,
               trans_tril=Lt, rot_tril=Lr, cost=cost)
    if return_refit:
        out.update(refit_trans=torch.stack(refit_t) if refit_t else torch.zeros(0, B, 3, 3, dtype=dt),
                   refit_rot=torch.stack(refit_r) if refit_r else torch.zeros(0, B, 4, 4, dtype=dt),
                   refit_logw=refit_w)
    return out


def monte_carlo_forward_6dof(x3d, x2d, w2d, cam: Camera, delta, pose_init, noise, mc_samples=512,
                             num_iter=4, prm: LMParams = LMParams(), fast_mode=False):
    """LM (from pose_init, no init solver) followed by AMIS -- the fused path the metric names."""
    cost_init = evaluate(x3d, x2d, w2d, pose_init, cam, delta)["cost"]
    pose_opt, pose_cov, cost = lm_solve(x3d, x2d, w2d, cam, delta, pose_init, prm, fast_mode)
    r = amis_6dof(x3d, x2d, w2d, cam, delta, pose_opt, pose_cov, noise, mc_samples, num_iter, prm.eps)
    r.update(pose_opt=pose_opt, pose_cov=pose_cov, lm_cost=cost, cost_init=cost_init)
    return r


# ----------------------------------------------------------------------------- AMIS (4DoF)
_I0_SMALL = [1.0, 3.5156229, 3.0899424, 1.2067492, 0.2659732, 0.360768e-1, 0.45813e-2]
_I0_LARGE = [0.39894228, 0.1328592e-1, 0.225319e-2, -0.157565e-2, 0.916281e-2, -0.2057706e-1, 0.2635537e-1,
             -0.1647633e-1, 0.392377e-2]


def _poly(y, coef):
    r = torch.full_like(y, coef[-1])
    for c in reversed(coef[:-1]):
        r = c + y * r
    return r


def log_bessel_i0(x):
    """log I0(x) exactly as torch.distributions.von_mises._log_modified_bessel_fn(order=0) evaluates it
    (Abramowitz-Stegun polynomials) -- this is what VonMises.log_prob, hence the reference, uses."""
    small = _poly((x / 3.75) ** 2, _I0_SMALL).log()
    large = x - 0.5 * x.log() + _poly(3.75 / x, _I0_LARGE).log()
    return torch.where(x < 3.75, small, large)


def vm_mix_logpdf(yaw, loc, kappa, uniform_mix=0.25):
    vm = kappa * torch.cos(yaw - loc) - math.log(2 * math.pi) - log_bessel_i0(kappa) + math.log(1 - uniform_mix)
    return torch.logaddexp(vm, torch.full_like(vm, math.log(uniform_mix / (2 * math.pi))))


def amis_4dof(x3d, x2d, w2d, cam: Camera, delta, pose_opt, pose_cov, noise, mc_samples=512, num_iter=4, eps=1e-5,
              return_refit=False):
    """noise = (normal3 (I,S,B,3), chi2 (I,S,B), yaw draws (I,S,B)) -- the reference draws yaw with numpy on
    the host, so the draws themselves are the injected quantity.  Returns samples (M,B,4), logw (M,B), ...
    return_refit: also refit_trans (I-1,B,3,3), the matrix each refit hands to robust_cholesky, and refit_logw, per
    refit the log-weights ((i+1)S,B) it weighs the samples by."""
    n3, c2, yaw = noise
    I, S = num_iter, mc_samples // num_iter
    B, dt = x3d.shape[0], x3d.dtype
    mode = torch.zeros(I, B, 3, dtype=dt)
    Lt = torch.zeros(I, B, 3, 3, dtype=dt)
    rmode = torch.zeros(I, B, dtype=dt)
    kappa = torch.zeros(I, B, dtype=dt)
    dd = [1.0, 1.0, 4.0]
    mode[0] = pose_opt[:, :3]
    rmode[0] = pose_opt[:, 3]
    Lt[0] = robust_cholesky(pose_cov[:, :3, :3], dd)
    kappa[0] = 0.33 / pose_cov[:, 3, 3].clamp(min=eps)
    samples = torch.zeros(I, S, B, 4, dtype=dt)
    cost = torch.zeros(I, S, B, dtype=dt)
    logp = torch.zeros(I, I, S, B, dtype=dt)
    logw = None
    refit_t, refit_w = [], []
    for i in range(I):
        samples[i, ..., :3] = mvt_draw(n3[i], c2[i], mode[i], Lt[i])
        samples[i, ..., 3] = yaw[i]
        cost[i] = evaluate(x3d, x2d, w2d, samples[i], cam, delta)["cost"]
        logp[i, :i + 1] = mvt_logpdf(samples[:i + 1, ..., :3], mode[i], Lt[i]) \
            + vm_mix_logpdf(samples[:i + 1, ..., 3], rmode[i], kappa[i])
        if i > 0:
            logp[:i, i] = mvt_logpdf(samples[i, ..., :3], mode[:i, None], Lt[:i, None]) \
                + vm_mix_logpdf(samples[i, ..., 3], rmode[:i, None], kappa[:i, None])
        mix = torch.logsumexp(logp[:i + 1, :i + 1], dim=0) - math.log(i + 1)
        logw = -cost[:i + 1] - mix
        if i == I - 1:
            break
        refit_w.append(logw.reshape(-1, B))
        w = torch.softmax(refit_w[-1], dim=0)
        smp = samples[:i + 1].reshape(-1, B, 4)
        t = smp[..., :3]
        mode[i + 1] = (w[..., None] * t).sum(0)
        dev = t - mode[i + 1]
        refit_t.append((w[..., None, None] * dev[..., :, None] * dev[..., None, :]).sum(0))
        Lt[i + 1] = robust_cholesky(refit_t[-1], dd)
        s_sum = (w * smp[..., 3].sin()).sum(0)
        c_sum = (w * smp[..., 3].cos()).sum(0)
        rmode[i + 1] = torch.atan2(s_sum, c_sum)
        r_sq = s_sum ** 2 + c_sum ** 2
        kappa[i + 1] = 0.33 * r_sq.sqrt().clamp(min=eps) * (2 - r_sq) / (1 - r_sq).clamp(min=eps)
    out = dict(samples=samples.reshape(I * S, B, 4), logw=logw.reshape(I * S, B), trans_mode=mode, trans_tril=Lt,
               rot_mode=rmode, rot_kappa=kappa, cost=cost)
    if return_refit:
        out.update(refit_trans=torch.stack(refit_t) if refit_t else torch.zeros(0, B, 3, 3, dtype=dt), refit_logw=refit_w)
    return out
