"""Helpers of the reference's epropnp/common.py, re-implemented.

`evaluate_pnp` is the only hot function here and goes to the native library; the rotation helpers
and the normalisation transform are a few torch ops on (B, 3)-sized tensors (not the hot path).
"""
import torch

from epropnp_b200 import ops


def skew(x):
    """(*, 3) -> (*, 3, 3) cross-product matrices [x]_x   (reference common.py:8-19)."""
    zero = torch.zeros_like(x[..., 0])
    rows = torch.stack((zero, -x[..., 2], x[..., 1],
                        x[..., 2], zero, -x[..., 0],
                        -x[..., 1], x[..., 0], zero), dim=-1)
    return rows.reshape(x.shape[:-1] + (3, 3))


def quaternion_to_rot_mat(quaternions):
    """(*, 4) [w, i, j, k] -> (*, 3, 3)   (reference common.py:22-42)."""
    w, x, y, z = quaternions.unbind(-1)
    ww, xx, yy, zz = w * w, x * x, y * y, z * z
    m = torch.stack((ww + xx - yy - zz, 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), ww - xx + yy - zz, 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), ww - xx - yy + zz), dim=-1)
    return m.reshape(quaternions.shape[:-1] + (3, 3))


def yaw_to_rot_mat(yaw):
    """(*) rotation about the Y axis -> (*, 3, 3)   (reference common.py:45-64)."""
    c, s = torch.cos(yaw), torch.sin(yaw)
    o, z = torch.ones_like(yaw), torch.zeros_like(yaw)
    return torch.stack((c, z, s, z, o, z, -s, z, c), dim=-1).reshape(yaw.shape + (3, 3))


def _pose_rot(pose):
    return yaw_to_rot_mat(pose[..., 3]) if pose.size(-1) == 4 else quaternion_to_rot_mat(pose[..., 3:])


def _needs_grad(*tensors):
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in tensors)


def _camera_requires_grad(camera):
    """cam_mats or a tensor bound of `camera` requires grad."""
    return any(torch.is_tensor(t) and t.requires_grad for t in (camera.cam_mats, camera.lb, camera.ub))


def _store(out, value):
    """Reference semantics of the out_* arguments: a tensor is filled in place and returned."""
    if torch.is_tensor(out):
        out.view(value.shape).copy_(value)
        return out
    return value


def evaluate_pnp(x3d, x2d, w2d, pose, camera, cost_fun,
                 out_jacobian=False, out_residual=False, out_cost=False, **kwargs):
    """Projection + Huber cost (+ residual / Jacobian) of pose hypotheses (reference common.py:67-100).

    x3d (B, n, 3), x2d / w2d (B, n, 2); pose (B, D) or (*, B, D) with D = 4 | 7.
    out_*: False -> skipped (None returned), True -> returned, tensor -> filled in place.
    Returns (residual (*, B, 2n) | None, cost (*, B) | None, jacobian (*, B, 2n, dof) | None).
    """
    clip_jac = kwargs.pop("clip_jac", True)
    if kwargs:
        raise TypeError(f"unexpected arguments {sorted(kwargs)}")
    camera_grad = _needs_grad(camera.cam_mats, camera.lb, camera.ub)
    if _needs_grad(x3d, x2d, w2d, pose, getattr(cost_fun, "delta", None)) or camera_grad:
        native_grad = x3d.is_cuda and x3d.dtype == pose.dtype == torch.float32
        want_j, want_r, want_c = out_jacobian is not False, out_residual is not False, out_cost is not False
        if (want_j or want_r) and native_grad:
            # differentiable residual / Jacobian (LMSolver.gn_step under autograd, reference common.py:67-100): native
            # forward + native backward
            from .autograd import evaluate_autograd
            residual, cost, jac = evaluate_autograd(x3d, x2d, w2d, pose, camera, cost_fun, clip_jac, want_r, want_j,
                                                    want_c)
            return ((_store(out_residual, residual) if want_r else None), (_store(out_cost, cost) if want_c else None),
                    (_store(out_jacobian, jac) if want_j else None))
        if want_j or want_r or ((pose.requires_grad or camera_grad) and not native_grad):
            # the same outputs, or gradients w.r.t. the pose or the camera, of CPU / float64 tensors: the torch
            # composite of the same two methods the reference calls
            x2d_proj, jac_cam = camera.project(x3d, pose, out_jac=(out_jacobian is not False), clip_jac=clip_jac)
            residual, cost, jac = cost_fun.compute(x2d_proj, x2d, w2d, jac_cam=jac_cam, out_residual=(out_residual is not False),
                                                   out_cost=(out_cost is not False), out_jacobian=(out_jacobian is not False))
            return ((_store(out_residual, residual) if out_residual is not False else None),
                    (_store(out_cost, cost) if out_cost is not False else None),
                    (_store(out_jacobian, jac) if out_jacobian is not False else None))
        from .autograd import evaluate_cost_autograd
        cost = evaluate_cost_autograd(x3d, x2d, w2d, pose, camera, cost_fun)       # native forward + native backward
        return None, (_store(out_cost, cost) if out_cost is not False else None), None

    dof = 4 if pose.size(-1) == 4 else 6
    lead = pose.shape[:-1]
    B, n = x3d.shape[0], x3d.shape[1]
    want_j, want_r, want_c = out_jacobian is not False, out_residual is not False, out_cost is not False
    from .autograd import _problem_args
    args = _problem_args(x3d, x2d, w2d, camera, cost_fun)
    poses = pose.reshape(-1, B, pose.size(-1))
    residual = cost = jac = None
    if not want_j and not want_r:
        if want_c:
            cost = ops.evaluate_cost(*args, poses, dof, float(camera.z_min)).reshape(lead)
    else:
        # stacked hypotheses with Jacobians: every (hypothesis, object) is its own object
        r, c, j = ops.evaluate_full(*args, poses, dof, float(camera.z_min), float(getattr(cost_fun, "eps", 1e-10)),
                                    bool(clip_jac), want_r, want_j, want_c)
        residual = r.reshape(lead + (2 * n,)) if want_r else None
        cost = c.reshape(lead) if want_c else None
        jac = j.reshape(lead + (2 * n, dof)) if want_j else None
    to = lambda t: None if t is None else t.to(x3d.dtype)
    residual, cost, jac = to(residual), to(cost), to(jac)
    return (_store(out_residual, residual) if want_r else None,
            _store(out_cost, cost) if want_c else None,
            _store(out_jacobian, jac) if want_j else None)


def philox_seed(seed, device):
    """The seed of a native Philox draw (AMIS samples, RSLM subsets and starts).  A given seed is used as it is: an int,
    or a one-element int64 CUDA tensor whose value the kernel reads when it runs.  Without one, a fresh seed: eagerly an
    int from torch's default CPU generator (torch.manual_seed governs it); while the current stream is being captured
    into a CUDA graph, a tensor drawn on `device` by torch's CUDA generator, so that every replay of the graph writes a
    new seed and the kernels draw new samples -- an int would be baked into the graph."""
    if seed is not None:
        return seed if torch.is_tensor(seed) and seed.is_cuda else int(seed)
    # under torch.compile likewise: a compiled graph (and a reduce-overhead CUDA graph) replays what was traced
    if torch.compiler.is_compiling() or (torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()):
        return torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=device)
    return int(torch.randint(0, 2 ** 62, (1,)).item())


def pnp_normalize(x3d, pose=None, detach_transformation=True):
    """Centre the 3D points; returns (offset (*, 1, 3), x3d_norm, pose_norm)   (reference common.py:103-127)."""
    src = x3d.detach() if detach_transformation else x3d
    offset = src.mean(dim=-2)
    x3d_norm = x3d - offset.unsqueeze(-2)
    pose_norm = None
    if pose is not None:
        shift = (_pose_rot(pose) @ offset.unsqueeze(-1)).squeeze(-1)
        pose_norm = torch.cat((pose[..., :3] + shift, pose[..., 3:]), dim=-1)
    return offset, x3d_norm, pose_norm


def pnp_denormalize(offset, pose_norm):
    """Inverse of pnp_normalize for poses of shape (*, B, D)   (reference common.py:130-136)."""
    shift = (_pose_rot(pose_norm) @ offset.unsqueeze(-1)).squeeze(-1)
    return torch.cat((pose_norm[..., :3] - shift, pose_norm[..., 3:]), dim=-1)
