"""EProPnP6DoF / EProPnP4DoF with the reference's constructor and call signatures
(reference epropnp/epropnp.py), executing on the native sm_90a kernels.

`monte_carlo_forward` = one fused launch (epnp_lm_amis_fused_f32): the LM solve, its covariance, the
first proposal, and all AMIS iterations (draw -> cost of every sample over all points -> mixture
densities -> log-weights -> proposal refit) run per object inside one CTA with the correspondences
resident in shared memory.  The reference's materialised (S, B, N, 3) intermediates, its per-iteration
host Cholesky round trips and its ~10^3 op launches do not exist here.  Objects with more correspondences than one
SM holds (N > epnp_max_points(dof, M, I), e.g. the 16,384 of a 128 x 128 coordinate map) run the same loop on a
thread-block cluster of 2-8 CTAs (epnp_lm_amis_fused_split_f32).  The RSLM initialiser refuses those with its
shared-memory error unless it was built as RSLMSolver(..., cluster_split=True), which solves them on the cluster-split
initialiser (epnp_rslm_split_f32); without it they need pose_init with force_init_solve=False.

Layout note: the kernel writes object-major (B, M, D) / (B, M) buffers; the tuples returned below
hold (M, B, D) / (M, B) *views* of them so reference call sites (softmax(dim=0), logsumexp(dim=0),
[..., [0, 2]] ...) work unchanged.

Extra keyword-only arguments (not in the reference): `amis_noise` = (normal3 (B,M,3), chi2 (B,M),
rot (B,M,4)) injects the proposals' base noise (parity tests); `amis_seed` fixes the Philox stream: an int, or a
one-element int64 CUDA tensor the kernel reads at run time (for CUDA graphs that set the seed before each replay).
Without them a seed is drawn from torch's default CPU generator, so torch.manual_seed() governs it; while a CUDA graph
is being captured it is drawn on the device instead, so every replay samples anew (common.philox_seed).
"""
from abc import ABCMeta, abstractmethod

import torch

from .builder import PNP, build_pnp
from .common import _needs_grad, evaluate_pnp, philox_seed, pnp_normalize, pnp_denormalize
from .distributions import AngularCentralGaussian, MultivariateStudentT, VonMisesUniformMix

# The steps of the AMIS loop the reference exposes as methods of the layer (epropnp.py:65-82).  Here the loop runs inside
# one kernel; the methods exist as stand-alone torch restatements (same signatures, in-place on the buffers of
# allocate_buffer) for callers that inspect or re-use the proposals, and monte_carlo_forward refuses a subclass that
# overrides one of them -- the kernel could not honour it.
_AMIS_STEPS = ("allocate_buffer", "initial_fit", "gen_new_distr", "gen_old_distr", "estimate_params")


def cholesky_wrapper(mat, default_diag=None, force_cpu=True):
    """Batched lower Cholesky; matrices that are not positive definite fall back to diag(default_diag)
    (or the identity).  Device-side (`cholesky_ex`), no host round trip; `force_cpu` is accepted for
    signature compatibility and ignored (reference epropnp.py:16-33)."""
    n = mat.size(-1)
    L, info = torch.linalg.cholesky_ex(mat)
    bad = info != 0
    fallback = torch.diag(mat.new_tensor(default_diag)) if default_diag is not None else \
        torch.eye(n, dtype=mat.dtype, device=mat.device)
    return torch.where(bad[..., None, None], fallback, L)


class EProPnPBase(torch.nn.Module, metaclass=ABCMeta):
    """End-to-End Probabilistic Perspective-n-Points.

    Args:
        mc_samples (int): total number of Monte Carlo samples
        num_iter (int): number of AMIS iterations
        normalize (bool): centre the 3D points before solving
        eps (float)
        solver: PnP solver module (LMSolver)
    """

    def __init__(self, mc_samples=512, num_iter=4, normalize=False, eps=1e-5, solver=None):
        super(EProPnPBase, self).__init__()
        assert num_iter > 0
        assert mc_samples % num_iter == 0
        self.mc_samples = mc_samples
        self.num_iter = num_iter
        self.iter_samples = self.mc_samples // self.num_iter
        self.eps = eps
        self.normalize = normalize
        self.solver = build_pnp(solver)                  # instance, None, or a config dict

    @property
    @abstractmethod
    def dof(self):
        pass

    def _amis_params(self, camera, cost_fun, fast_mode):
        """(ints, floats) of the fused operator (ops.param_lists)."""
        return self.solver.param_lists(camera, cost_fun, fast_mode, mc_samples=int(self.mc_samples),
                                       mc_iter=int(self.num_iter), amis_eps=float(self.eps),
                                       **self._extra_native_params())

    def _extra_native_params(self):
        return {}

    @abstractmethod
    def allocate_buffer(self, *args, **kwargs):
        pass

    @abstractmethod
    def initial_fit(self, *args, **kwargs):
        pass

    @abstractmethod
    def gen_new_distr(self, *args, **kwargs):
        pass

    @abstractmethod
    def gen_old_distr(self, *args, **kwargs):
        pass

    @abstractmethod
    def estimate_params(self, *args, **kwargs):
        pass

    def _refuse_overridden_steps(self):
        stock = EProPnP6DoF if self.dof == 6 else EProPnP4DoF
        changed = [name for name in _AMIS_STEPS if getattr(type(self), name, None) is not getattr(stock, name)]
        if changed:
            raise NotImplementedError(
                f"{type(self).__name__} overrides {', '.join(changed)}: the AMIS loop runs inside one kernel "
                "(epnp_lm_amis_fused_f32) that implements these steps itself, so a custom proposal family needs its own "
                "kernel; the methods are stand-alone restatements, not hooks of monte_carlo_forward")

    @staticmethod
    def _weighted_translation_fit(pose_samples, weights):
        """Weighted mean (B, 3) and covariance (B, 3, 3) of the sampled translations; weights (cum, B) sum to 1 over dim 0."""
        trans = pose_samples[..., :3]
        mean = torch.einsum('sb,sbi->bi', weights, trans)
        dev = trans - mean
        return mean, torch.einsum('sb,sbi,sbj->bij', weights, dev, dev)

    def forward(self, *args, **kwargs):
        return self.solver(*args, **kwargs)

    def monte_carlo_forward(self, x3d, x2d, w2d, camera, cost_fun, pose_init=None, force_init_solve=True,
                            amis_noise=None, amis_seed=None, **kwargs):
        """Weighted pose samples from the pose distribution defined by {x3d, x2d, w2d}.

        Args / returns as the reference (epropnp.py:87-113):
            pose_opt (B, 4|7), cost (B) | None, pose_opt_plus (B, 4|7) | None,
            pose_samples (mc_samples, B, 4|7), pose_sample_logweights (mc_samples, B), cost_init (B) | None
        kwargs forwarded to the solver: with_pose_opt_plus, fast_mode, with_cost.
        """
        self._refuse_overridden_steps()
        with_plus = kwargs.pop("with_pose_opt_plus", False)
        fast_mode = kwargs.pop("fast_mode", False)
        with_cost = kwargs.pop("with_cost", False)
        if kwargs:
            raise TypeError(f"unexpected arguments {sorted(kwargs)}")
        delta = cost_fun.delta
        differentiable = _needs_grad(x3d, x2d, w2d, delta, pose_init, camera.cam_mats, camera.lb, camera.ub)
        if self.normalize:
            transform, x3d, pose_init = pnp_normalize(x3d, pose_init, detach_transformation=True)
        assert x3d.dim() == x2d.dim() == w2d.dim() == 3
        num_obj = x3d.size(0)
        pd = 4 if self.dof == 4 else 7
        kw = dict(dtype=x3d.dtype, device=x3d.device)

        with torch.no_grad():
            if num_obj == 0:
                pose_opt = torch.empty((0, pd), **kw)
                cost = torch.empty((0,), **kw) if with_cost else None
                pose_opt_plus = torch.empty((0, pd), **kw) if with_plus else None
                pose_samples = torch.zeros((self.mc_samples, 0, pd), **kw)
                logw = torch.zeros((self.mc_samples, 0), **kw)
                cost_init = torch.empty((0,), **kw) if pose_init is not None else None
            else:
                needs_init_solver = pose_init is None or force_init_solve
                cost_init = None
                if needs_init_solver:
                    if pose_init is not None:
                        cost_init = evaluate_pnp(x3d, x2d, w2d, pose_init, camera, cost_fun, out_cost=True)[1]
                    start = self.solver._starting_pose(x3d, x2d, w2d, camera, cost_fun, pose_init, cost_init,
                                                       force_init_solve, fast_mode)
                else:
                    start = pose_init
                seed = philox_seed(amis_seed, x3d.device)
                params = self._amis_params(camera, cost_fun, fast_mode)
                if not differentiable:
                    from .autograd import monte_carlo_autograd
                    pose_opt, cost, pose_opt_plus, samples_bm, logw_bm, ci = monte_carlo_autograd(
                        x3d, x2d, w2d, camera, cost_fun, start, None, params, amis_noise, seed, with_cost,
                        want_plus=with_plus, want_cost_init=(pose_init is not None and not needs_init_solver))
                    if cost_init is None:
                        cost_init = ci
                    pose_samples = samples_bm.transpose(0, 1)      # (M, B, D) view
                    logw = logw_bm.transpose(0, 1)                 # (M, B) view

        if num_obj == 0 and torch.is_grad_enabled():
            # an empty batch must still be part of the graph (reference epropnp.py:184-187 and its differentiable
            # cost_init / pose_opt_plus): a loss built from these outputs has a grad_fn, backward() gives zero gradients
            # instead of raising, and under DDP the heads of a rank without objects still take part in the all-reduce
            tie = x3d.sum(dim=(1, 2)) + x2d.sum(dim=(1, 2)) + w2d.sum(dim=(1, 2))             # (0,), connected
            logw = x3d.reshape(self.mc_samples, 0) + x2d.reshape(self.mc_samples, 0) + w2d.reshape(self.mc_samples, 0)
            if cost_init is not None:
                cost_init = cost_init + tie + pose_init.sum(dim=1)
            if pose_opt_plus is not None:
                pose_opt_plus = pose_opt_plus + tie[:, None]

        if num_obj > 0 and differentiable:
            # training path: forward = the same fused kernel, backward = native Monte-Carlo cost gradient
            from .autograd import monte_carlo_autograd, pose_plus_autograd
            pose_opt, cost, _, samples_bm, logw_bm, cost_init = monte_carlo_autograd(
                x3d, x2d, w2d, camera, cost_fun, start, pose_init, params, amis_noise, seed, with_cost)
            pose_samples, logw = samples_bm.transpose(0, 1), logw_bm.transpose(0, 1)
            pose_opt_plus = None
            if with_plus:
                pose_opt_plus = pose_plus_autograd(self.solver, x3d, x2d, w2d, pose_opt, camera, cost_fun)

        if self.normalize:
            pose_opt = pnp_denormalize(transform, pose_opt)
            pose_samples = pnp_denormalize(transform, pose_samples)
            if pose_opt_plus is not None:
                pose_opt_plus = pnp_denormalize(transform, pose_opt_plus)
        return pose_opt, cost, pose_opt_plus, pose_samples, logw, cost_init


@PNP.register_module()
class EProPnP4DoF(EProPnPBase):
    """4DoF pose [x, y, z, yaw]; proposals: translation ~ multivariate t (df 3), yaw ~ 0.75 von Mises +
    0.25 uniform (reference epropnp.py:199-260).  `amis_noise` = (normal3 (B,M,3), chi2 (B,M), yaw (B,M)):
    for 4DoF the third tensor holds the yaw draws themselves (the reference draws them with numpy on the
    host, distributions.py:61-72); without it the kernel samples yaw with Philox + Best-Fisher rejection."""

    dof = 4

    def allocate_buffer(self, num_obj, dtype=torch.float32, device=None):
        """-> trans_mode (I, B, 3), trans_cov_tril (I, B, 3, 3), rot_mode (I, B, 1), rot_kappa (I, B, 1)  (:209-214)."""
        new = lambda *shape: torch.empty((self.num_iter, num_obj) + shape, dtype=dtype, device=device)
        return new(3), new(3, 3), new(1), new(1)

    def initial_fit(self, pose_opt, pose_cov, camera, trans_mode, trans_cov_tril, rot_mode, rot_kappa):
        """Proposal 0 from the LM solution and its covariance (:216-220)."""
        trans_mode[0], rot_mode[0] = pose_opt[:, :3], pose_opt[:, 3:]
        trans_cov_tril[0] = cholesky_wrapper(pose_cov[:, :3, :3], [1.0, 1.0, 4.0])
        rot_kappa[0] = 0.33 / pose_cov[:, 3, 3, None].clamp(min=self.eps)

    @staticmethod
    def gen_new_distr(iter_id, trans_mode, trans_cov_tril, rot_mode, rot_kappa):
        return (MultivariateStudentT(3, trans_mode[iter_id], trans_cov_tril[iter_id]),
                VonMisesUniformMix(rot_mode[iter_id], rot_kappa[iter_id]))

    @staticmethod
    def gen_old_distr(iter_id, trans_mode, trans_cov_tril, rot_mode, rot_kappa):
        """All earlier proposals, with a broadcast axis for the samples: batch shape (iter_id, 1, B)."""
        return (MultivariateStudentT(3, trans_mode[:iter_id, None], trans_cov_tril[:iter_id, None]),
                VonMisesUniformMix(rot_mode[:iter_id, None], rot_kappa[:iter_id, None]))

    def estimate_params(self, iter_id, pose_samples, pose_sample_logweights, trans_mode, trans_cov_tril, rot_mode, rot_kappa):
        """Proposal iter_id + 1 from all samples so far (cum, B, 4) and their log-weights (cum, B) (:238-260): weighted
        translation moments; yaw mode = direction of the weighted mean resultant, concentration from its length."""
        w = torch.softmax(pose_sample_logweights, dim=0)
        trans_mode[iter_id + 1], cov = self._weighted_translation_fit(pose_samples, w)
        trans_cov_tril[iter_id + 1] = cholesky_wrapper(cov, [1.0, 1.0, 4.0])
        yaw = pose_samples[..., 3]
        s, c = (w * yaw.sin()).sum(dim=0), (w * yaw.cos()).sum(dim=0)
        rot_mode[iter_id + 1] = torch.atan2(s, c).unsqueeze(-1)
        r_sq = (s.square() + c.square()).unsqueeze(-1)
        rot_kappa[iter_id + 1] = 0.33 * r_sq.sqrt().clamp(min=self.eps) * (2 - r_sq) / (1 - r_sq).clamp(min=self.eps)


@PNP.register_module()
class EProPnP6DoF(EProPnPBase):
    """6DoF pose [x, y, z, w, i, j, k]; proposals: translation ~ multivariate t (df 3), orientation ~
    angular central Gaussian (reference epropnp.py:263-342)."""

    dof = 6

    def __init__(self, *args, acg_mle_iter=3, acg_dispersion=0.001, **kwargs):
        super(EProPnP6DoF, self).__init__(*args, **kwargs)
        self.acg_mle_iter = acg_mle_iter
        self.acg_dispersion = acg_dispersion

    def _extra_native_params(self):
        return dict(acg_mle_iter=int(self.acg_mle_iter), acg_dispersion=float(self.acg_dispersion))

    def allocate_buffer(self, num_obj, dtype=torch.float32, device=None):
        """-> trans_mode (I, B, 3), trans_cov_tril (I, B, 3, 3), rot_cov_tril (I, B, 4, 4)  (:282-286)."""
        new = lambda *shape: torch.empty((self.num_iter, num_obj) + shape, dtype=dtype, device=device)
        return new(3), new(3, 3), new(4, 4)

    def _dispersed_tril(self, rot_cov):
        """chol(C + det(C)^(1/4) * dispersion * I): keeps the ACG proposal from collapsing onto one orientation."""
        eye = torch.eye(4, dtype=rot_cov.dtype, device=rot_cov.device)
        return cholesky_wrapper(rot_cov + rot_cov.det()[:, None, None] ** 0.25 * (self.acg_dispersion * eye))

    def initial_fit(self, pose_opt, pose_cov, camera, trans_mode, trans_cov_tril, rot_cov_tril):
        """Proposal 0 from the LM solution and its covariance (:288-302): the 3-dof rotation covariance of the tangent
        space is lifted to a 4x4 scatter matrix of the quaternion, (T S^-1 T^T + I)^-1 normalised to unit trace."""
        trans_mode[0] = pose_opt[:, :3]
        trans_cov_tril[0] = cholesky_wrapper(pose_cov[:, :3, :3])
        lift = camera.get_quaternion_transfrom_mat(pose_opt[:, 3:])                       # (B, 4, 3)
        eye = torch.eye(4, dtype=pose_opt.dtype, device=pose_opt.device)
        scatter = torch.linalg.inv(lift @ torch.linalg.inv(pose_cov[:, 3:, 3:]) @ lift.transpose(-1, -2) + eye)
        scatter = scatter / scatter.diagonal(dim1=-2, dim2=-1).sum(-1)[:, None, None]
        rot_cov_tril[0] = self._dispersed_tril(scatter)

    @staticmethod
    def gen_new_distr(iter_id, trans_mode, trans_cov_tril, rot_cov_tril):
        return (MultivariateStudentT(3, trans_mode[iter_id], trans_cov_tril[iter_id]),
                AngularCentralGaussian(rot_cov_tril[iter_id]))

    @staticmethod
    def gen_old_distr(iter_id, trans_mode, trans_cov_tril, rot_cov_tril):
        """All earlier proposals, with a broadcast axis for the samples: batch shape (iter_id, 1, B)."""
        return (MultivariateStudentT(3, trans_mode[:iter_id, None], trans_cov_tril[:iter_id, None]),
                AngularCentralGaussian(rot_cov_tril[:iter_id, None]))

    def estimate_params(self, iter_id, pose_samples, pose_sample_logweights, trans_mode, trans_cov_tril, rot_cov_tril):
        """Proposal iter_id + 1 from all samples so far (cum, B, 7) and their log-weights (cum, B) (:317-342): weighted
        translation moments; orientation scatter by `acg_mle_iter` fixed-point steps of the weighted ACG maximum
        likelihood, C <- sum_s w_s q_s q_s^T / (q_s^T C^-1 q_s) with the weights renormalised (+ eps I)."""
        w = torch.softmax(pose_sample_logweights, dim=0)
        trans_mode[iter_id + 1], cov = self._weighted_translation_fit(pose_samples, w)
        trans_cov_tril[iter_id + 1] = cholesky_wrapper(cov)
        q = pose_samples[..., 3:]
        eye = torch.eye(4, dtype=q.dtype, device=q.device)
        scatter = eye.expand(q.size(1), 4, 4)
        for _ in range(self.acg_mle_iter):
            mahal = torch.einsum('sbi,bij,sbj->sb', q, torch.linalg.inv(scatter), q).clamp(min=self.eps)
            ratio = w / mahal
            ratio = ratio / ratio.sum(dim=0)
            scatter = torch.einsum('sb,sbi,sbj->bij', ratio, q, q) + eye * self.eps
        rot_cov_tril[iter_id + 1] = self._dispersed_tril(scatter)
