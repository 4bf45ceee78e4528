"""The step after `monte_carlo_forward` in every caller of the layer (SURVEY.md section 8, row f4):

    MonteCarloPoseLoss      KL-divergence pose loss  cost_target + logsumexp_m(pose_sample_logweights), NaN -> 0,
                            divided by an EMA norm factor.  One class for both reference flavours:
                            EPro-PnP-6DoF/lib/models/monte_carlo_pose_loss.py:9-35 (mean / norm_factor) and
                            EPro-PnP-Det/epropnp_det/models/losses/monte_carlo_pose_loss.py:12-66 (mmdet's
                            weighted_loss: weight, reduction, avg_factor, loss_weight; norm factor averaged over ranks)
    mc_logsumexp            (M, B) log-weights -> (B), differentiable
    mc_sample_weights       pose_sample_logweights.softmax(dim=0)               (deform_pnp_head.py:524)
    mc_score_te             Monte-Carlo translation-error score                 (deform_pnp_head.py:533-536)

The layer hands out `pose_sample_logweights` (M, B) and `pose_samples` (M, B, D) as transposed views of object-major
buffers, so each of these is ONE pass over contiguous memory in the native epilogue kernel (epnp_mc_epilogue_f32 /
epnp_mc_lse_backward_f32) instead of the reference's chain of (M, B) reductions, an advanced-index gather
`pose_samples[..., [0, 2]]` and a softmax.  The native epilogue is the default for CUDA tensors;
`EPNP_NATIVE_MC_EPILOGUE=0` selects the torch composite below instead, which is the reference's formula verbatim in
meaning (CPU tensors always take it).  Both are outside the hot path: O(M B) work next to the O(M B N) of the solve.
"""
import os

import torch
import torch.nn as nn

from epropnp_b200 import ops


def _use_native(t):
    return os.environ.get("EPNP_NATIVE_MC_EPILOGUE", "1") == "1" and t.is_cuda


def _object_major(t):
    """(M, B, ...) view -> (B, M, ...) contiguous; free when `t` is the layer's transposed view."""
    return t.transpose(0, 1).contiguous()


def mc_logsumexp(pose_sample_logweights):
    """(mc_samples, num_obj) -> (num_obj,) = logsumexp over the samples (the loss's `loss_pred`); differentiable through
    the epilogue operator's formula (epnp_mc_lse_backward_f32)."""
    if pose_sample_logweights.dim() == 2 and _use_native(pose_sample_logweights):
        lse = ops.mc_epilogue(_object_major(pose_sample_logweights), None, None, None, True, False, False, False)[0]
        return lse.to(pose_sample_logweights.dtype)
    return torch.logsumexp(pose_sample_logweights, dim=0)


def mc_sample_weights(pose_sample_logweights):
    """softmax over the samples, returned as an (mc_samples, num_obj) view like the log-weights themselves."""
    if pose_sample_logweights.dim() == 2 and _use_native(pose_sample_logweights) \
            and not (pose_sample_logweights.requires_grad or ops.forward_tangent(pose_sample_logweights)):
        w = ops.mc_epilogue(_object_major(pose_sample_logweights), None, None, None, False, False, True, False)[2]
        return w.to(pose_sample_logweights.dtype).transpose(0, 1)
    return pose_sample_logweights.softmax(dim=0)


def mc_score_te(pose_samples, pose_opt, pose_sample_logweights):
    """Monte-Carlo 'te' score (num_obj,): expectation over the weighted samples of
    clamp((-log2 ||(x, z)_sample - (x, z)_opt|| + 2.5) / 4, 0, 1)   (deform_pnp_head.py:533-536)."""
    if pose_sample_logweights.dim() == 2 and _use_native(pose_sample_logweights):
        out = ops.mc_epilogue(_object_major(pose_sample_logweights.detach()), _object_major(pose_samples.detach()),
                              pose_opt.detach(), None, False, False, False, True)
        return out[3].to(pose_samples.dtype)
    sample_dev = (pose_samples[..., [0, 2]] - pose_opt[:, [0, 2]]).norm(dim=-1)
    score = ((-sample_dev.log2() + 2.5) / 4).clamp(min=0, max=1)
    return (score * pose_sample_logweights.softmax(dim=0)).sum(dim=0)


def monte_carlo_pose_loss(pose_sample_logweights, cost_target):
    """Per-object loss (num_obj,): cost_target + logsumexp(pose_sample_logweights, dim=0), NaN entries zeroed (and
    cut out of the graph, like the reference's in-place masked assignment)."""
    loss_pose = cost_target + mc_logsumexp(pose_sample_logweights)
    return torch.where(torch.isnan(loss_pose), torch.zeros_like(loss_pose), loss_pose)


def _reduce_mean_over_ranks(t):
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return t
    t = t.clone()
    dist.all_reduce(t.div_(dist.get_world_size()), op=dist.ReduceOp.SUM)
    return t


class MonteCarloPoseLoss(nn.Module):

    def __init__(self, loss_weight=1.0, init_norm_factor=1.0, momentum=0.01, reduction='mean',
                 sync_norm_factor=False):
        """6DoF flavour: MonteCarloPoseLoss(init_norm_factor, momentum) as keywords; Det flavour adds loss_weight /
        reduction and averages the norm factor over ranks (`sync_norm_factor=True`, mmdet's reduce_mean)."""
        super(MonteCarloPoseLoss, self).__init__()
        self.reduction = reduction
        self.loss_weight = loss_weight
        self.register_buffer('norm_factor', torch.tensor(init_norm_factor, dtype=torch.float))
        self.momentum = momentum
        self.sync_norm_factor = sync_norm_factor

    def forward(self, pose_sample_logweights, cost_target, norm_factor, weight=None, avg_factor=None,
                reduction_override=None):
        """
        Args:
            pose_sample_logweights: Shape (mc_samples, num_obj)
            cost_target: Shape (num_obj, )
            norm_factor: Shape ()
        """
        if self.training:
            with torch.no_grad():
                if self.sync_norm_factor:
                    norm_factor = _reduce_mean_over_ranks(norm_factor)
                self.norm_factor.mul_(1 - self.momentum).add_(self.momentum * norm_factor)
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        loss = monte_carlo_pose_loss(pose_sample_logweights, cost_target)
        if weight is not None:
            loss = loss * weight
        if avg_factor is None:
            if reduction == 'mean':
                loss = loss.mean()
            elif reduction == 'sum':
                loss = loss.sum()
        elif reduction == 'mean':
            loss = loss.sum() / avg_factor
        elif reduction != 'none':
            raise ValueError('avg_factor can not be used with reduction="sum"')
        if self.loss_weight == 1.0:
            return loss / self.norm_factor                      # the 6DoF flavour's expression, bit for bit
        return loss * (self.loss_weight / self.norm_factor)
