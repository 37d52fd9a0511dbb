"""torch.autograd through the bundle adjuster: an optimised window as a differentiable function of its observations
and their weights (svs_ba_observation_grad, INTEGRATION.md).

    poses, psi = optimise_window(ba, pb, e_obs, e_info, num_iters)
    loss(poses, psi).backward()          # fills e_obs.grad and e_info.grad

The backward pass is the adjoint of the minimiser at the state the forward pass reached, so it is only meaningful when
that state is stationary: optimise to convergence.  Robust weights are held at their value there (Gauss-Newton), and the
pose-pose constraints, the camera and the initial state are not differentiated.  The handle keeps the window between the
two passes: nothing may be loaded into or optimised on `ba` before backward() runs.
"""
from __future__ import annotations

import dataclasses

import numpy as np
import torch


def pose_grad_to_tangent(pose_qt, g_qt):
    """dL/d(qx, qy, qz, qw, tx, ty, tz) [P,7] at pose_qt [P,7] -> dL/d delta [P,6], delta = (upsilon, omega) of the
    update T <- exp(delta) T.  To first order q' = (q_v + (q_w w + w x q_v) / 2, q_w - w . q_v / 2), t' = t + u + w x t."""
    qv, qw, t = pose_qt[:, 0:3], pose_qt[:, 3:4], pose_qt[:, 4:7]
    gv, gw, gt = g_qt[:, 0:3], g_qt[:, 3:4], g_qt[:, 4:7]
    g_omega = torch.linalg.cross(t, gt) + 0.5 * (qw * gv + torch.linalg.cross(qv, gv) - gw * qv)
    return torch.cat([gt, g_omega], dim=1)


def _as_problem(pb, e_obs, e_info):
    """pb with e_obs / e_info substituted: every array as a CUDA tensor on their device when they are CUDA tensors (the
    handle then analyses the window on the device, and a repeated structure re-sends only the numbers), else numpy."""
    if e_obs.is_cuda:
        dev = e_obs.device

        def conv(a, dt):
            if a is None or isinstance(a, torch.Tensor):
                return a if a is None else a.to(dev, dt)
            return torch.as_tensor(np.asarray(a), dtype=dt, device=dev)
        return dataclasses.replace(
            pb, pose_qt=conv(pb.pose_qt, torch.float64), fixed=conv(pb.fixed, torch.uint8), psi=conv(pb.psi, torch.float64),
            e_point=conv(pb.e_point, torch.int32), e_pose=conv(pb.e_pose, torch.int32),
            e_anchor=conv(pb.e_anchor, torch.int32), e_obs=e_obs.detach().to(torch.float64).contiguous(),
            e_info=e_info.detach().to(dev, torch.float64).contiguous(), c_i=conv(pb.c_i, torch.int32),
            c_j=conv(pb.c_j, torch.int32), c_T=conv(pb.c_T, torch.float64), c_Lambda=conv(pb.c_Lambda, torch.float64))
    return dataclasses.replace(pb, e_obs=e_obs.detach().cpu().numpy().astype(np.float64),
                               e_info=e_info.detach().cpu().numpy().astype(np.float64))


class _OptimiseWindow(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e_obs, e_info, ba, pb, num_iters, robust, huber_delta, lambda_init, grad_lambda):
        ba.set_problem(_as_problem(pb, e_obs, e_info))
        ba.optimize(num_iters, robust, huber_delta, lambda_init)
        dev = e_obs.device
        poses = torch.as_tensor(ba.poses(), dtype=torch.float64, device=dev)
        psi = torch.as_tensor(ba.points(), dtype=torch.float64, device=dev)
        ctx.ba, ctx.args = ba, (robust, huber_delta, grad_lambda)
        ctx.obs_like, ctx.info_like = (e_obs.dtype, e_obs.device), (e_info.dtype, e_info.device)
        ctx.save_for_backward(poses)
        return poses, psi

    @staticmethod
    def backward(ctx, g_poses, g_psi):
        (poses,) = ctx.saved_tensors
        robust, huber_delta, grad_lambda = ctx.args
        dev = poses.device
        g_delta = None if g_poses is None else pose_grad_to_tangent(poses, g_poses.to(torch.float64))
        if not dev.type == "cuda":   # the handle takes host arrays or CUDA tensors
            g_delta = None if g_delta is None else g_delta.numpy()
            g_psi = None if g_psi is None else g_psi.to(torch.float64).numpy()
        elif g_psi is not None:
            g_psi = g_psi.to(torch.float64)
        dobs, dinfo, rc, _ = ctx.ba.observation_grad(g_delta, g_psi, robust, huber_delta, grad_lambda)
        if rc != 0:
            raise RuntimeError(f"svs_ba_observation_grad: the reduced system is not positive definite (rc = {rc})")
        dobs, dinfo = torch.as_tensor(dobs), torch.as_tensor(dinfo)
        return (dobs.to(ctx.obs_like[1], ctx.obs_like[0]), dinfo.to(ctx.info_like[1], ctx.info_like[0]),
                None, None, None, None, None, None, None)


def optimise_window(ba, pb, e_obs, e_info, num_iters, robust=True, huber_delta=1.0, lambda_init=50.0, grad_lambda=0.0):
    """Load `pb` into the BundleAdjuster `ba` with its observations e_obs [E,3] and weights e_info [E,3] replaced by the
    given tensors, optimise it for num_iters iterations and return (pose_qt [P,7], psi [L,3]) as float64 tensors on
    their device.  The backward pass gives gradients for e_obs and e_info only, from one adjoint solve at
    (H + grad_lambda I); grad_lambda = 0 needs a fixed pose."""
    return _OptimiseWindow.apply(e_obs, e_info, ba, pb, num_iters, robust, huber_delta, lambda_init, grad_lambda)
