#!/usr/bin/env python
"""The reference's usage demo (demo/fit_identity.ipynb, BASELINE.json config #1) on the H100-native layer:
an MLP maps a pose to 64 2D-3D correspondences + weights, EProPnP6DoF turns them back into a pose
distribution, trained end to end with the Monte-Carlo pose loss and the derivative regularisation loss.
Same calls as the notebook's cells 7-12; only `import epropnp` resolves to this repository.

    python demo/fit_identity.py --steps 300
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "epro-pnp_b200"))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from epropnp.camera import PerspectiveCamera  # noqa: E402
from epropnp.cost_fun import AdaptiveHuberPnPCost  # noqa: E402
from epropnp.epropnp import EProPnP6DoF  # noqa: E402
from epropnp.levenberg_marquardt import LMSolver, RSLMSolver  # noqa: E402


class Model(nn.Module):
    def __init__(self, num_points=64, hidden=1024):
        super().__init__()
        self.num_points = num_points
        self.mlp = nn.Sequential(nn.Linear(7, hidden), nn.LeakyReLU(), nn.Linear(hidden, num_points * 7))
        self.log_weight_scale = nn.Parameter(torch.zeros(2))
        self.epropnp = EProPnP6DoF(
            mc_samples=512, num_iter=4,
            solver=LMSolver(dof=6, num_iter=10,
                            init_solver=RSLMSolver(dof=6, num_points=8, num_proposals=128, num_iter=5)))
        self.camera = PerspectiveCamera()
        self.cost_fun = AdaptiveHuberPnPCost(relative_delta=0.5)

    def correspondences(self, in_pose):
        x3d, x2d, w2d = self.mlp(in_pose).reshape(-1, self.num_points, 7).split([3, 2, 2], dim=-1)
        w2d = (w2d.log_softmax(dim=-2) + self.log_weight_scale).exp()
        return x3d, x2d, w2d

    def forward_train(self, in_pose, cam_mats, out_pose):
        x3d, x2d, w2d = self.correspondences(in_pose)
        self.camera.set_param(cam_mats)
        self.cost_fun.set_param(x2d.detach(), w2d)
        r = self.epropnp.monte_carlo_forward(x3d, x2d, w2d, self.camera, self.cost_fun, pose_init=out_pose,
                                             force_init_solve=True, with_pose_opt_plus=True)
        return r + (self.log_weight_scale.detach().exp().mean(),)

    @torch.no_grad()
    def forward_test(self, in_pose, cam_mats, fast_mode=False):
        x3d, x2d, w2d = self.correspondences(in_pose)
        self.camera.set_param(cam_mats)
        self.cost_fun.set_param(x2d.detach(), w2d)
        return self.epropnp(x3d, x2d, w2d, self.camera, self.cost_fun, fast_mode=fast_mode)[0]


class MonteCarloPoseLoss(nn.Module):
    def __init__(self, init_norm_factor=1.0, momentum=0.1):
        super().__init__()
        self.register_buffer("norm_factor", torch.tensor(init_norm_factor, dtype=torch.float))
        self.momentum = momentum

    def forward(self, logweights, cost_target, norm_factor):
        if self.training:
            with torch.no_grad():
                self.norm_factor.mul_(1 - self.momentum).add_(self.momentum * norm_factor)
        loss = cost_target + torch.logsumexp(logweights, dim=0)
        loss = torch.where(torch.isnan(loss), torch.zeros_like(loss), loss)
        return loss.mean() / self.norm_factor


def make_data(n, device, noise, gen):
    in_pose = torch.randn(n, 7, generator=gen).to(device)
    in_pose[:, 2] += 5
    in_pose[:, 3:] = F.normalize(in_pose[:, 3:], dim=-1)
    out_pose = in_pose + torch.randn(n, 7, generator=gen).to(device) * noise
    out_pose[:, 3:] = F.normalize(out_pose[:, 3:], dim=-1)
    return in_pose, out_pose


def pose_errors(pose, gt):
    dist_t = (pose[:, :3] - gt[:, :3]).norm(dim=-1)
    dot = (pose[:, 3:] * gt[:, 3:]).sum(-1).abs().clamp(max=1.0)
    return dist_t.mean().item(), (2 * torch.acos(dot)).mean().item()


def run(steps=300, batch_size=256, seed=0, log_every=50, verbose=True, device=None, test_size=1024):
    device = torch.device("cuda:0") if device is None else device
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed)
    in_pose, out_pose = make_data(steps * batch_size, device, 0.01, gen)
    test_in, _ = make_data(test_size, device, 0.0, gen)
    cam = torch.eye(3, device=device)
    model = Model().to(device)
    loss_fn = MonteCarloPoseLoss().to(device)
    opt = torch.optim.Adam([{"params": model.mlp.parameters()}, {"params": model.log_weight_scale, "lr": 1e-2}], lr=1e-4)
    e0 = pose_errors(model.forward_test(test_in, cam.expand(test_size, -1, -1)), test_in)
    hist = []
    if device.type == "cuda":
        torch.cuda.synchronize()
    t0 = time.time()
    for it in range(steps):
        bi, bo = in_pose[it * batch_size:(it + 1) * batch_size], out_pose[it * batch_size:(it + 1) * batch_size]
        _, _, plus, _, logw, cost_tgt, norm = model.forward_train(bi, cam.expand(batch_size, -1, -1), bo)
        loss_mc = loss_fn(logw, cost_tgt, norm)
        dist_t = (plus[:, :3] - bo[:, :3]).norm(dim=-1)
        loss_t = torch.where(dist_t < 1.0, 0.5 * dist_t.square(), dist_t - 0.5).mean()
        dot = (plus[:, 3:] * bo[:, 3:]).sum(-1)
        loss_r = ((1 - dot.square()) * 2).mean()
        loss = loss_mc + 0.1 * loss_t + 0.1 * loss_r
        opt.zero_grad()
        loss.backward()
        opt.step()
        hist.append((loss_mc.item(), loss_t.item(), loss_r.item()))
        if verbose and (it % log_every == 0 or it == steps - 1):
            print(f"step {it + 1}/{steps}: loss_mc={hist[-1][0]:.4f} loss_t={hist[-1][1]:.4f} loss_r={hist[-1][2]:.4f}", flush=True)
    if device.type == "cuda":
        torch.cuda.synchronize()
    dt = time.time() - t0
    e1 = pose_errors(model.forward_test(test_in, cam.expand(test_size, -1, -1)), test_in)
    k = max(1, steps // 10)
    first = sum(h[0] for h in hist[:k]) / k
    last = sum(h[0] for h in hist[-k:]) / k
    out = dict(steps=steps, batch=batch_size, seconds=dt, ms_per_step=1e3 * dt / steps, loss_mc_first=first,
               loss_mc_last=last, test_t_err_before=e0[0], test_r_err_before=e0[1], test_t_err_after=e1[0],
               test_r_err_after=e1[1], finite=all(math.isfinite(x) for h in hist for x in h))
    if verbose:
        print(json.dumps(out))
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--batch", type=int, default=256)
    a = ap.parse_args()
    run(a.steps, a.batch)
