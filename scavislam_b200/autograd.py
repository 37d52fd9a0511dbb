"""torch.autograd through the bundle adjuster: an optimised window as a differentiable function of its observations,
their weights, its pose-pose constraints and its stereo camera (svs_ba_observation_grad, svs_ba_window_grad,
INTEGRATION.md).

    poses, psi = optimise_window(ba, pb, e_obs, e_info, num_iters)
    loss(poses, psi).backward()          # fills e_obs.grad and e_info.grad

    poses, psi = optimise_window(ba, pb, e_obs, e_info, num_iters, c_T=c_T, c_Lambda=c_Lambda, cam=cam)
    loss(poses, psi).backward()          # also fills c_T.grad, c_Lambda.grad and cam.grad

The backward pass is the adjoint of the minimiser at the state the forward pass reached, so it is only meaningful when
that state is stationary: optimise to convergence.  Robust weights are held at their value there (Gauss-Newton).  Only
the initial state (its gradient is zero at a stationary point) and the values of fixed poses are not differentiated.
The handle keeps the window between the two passes: nothing may be loaded into or optimised on `ba` before backward()
runs.

The front end's motion-only pose refinement is differentiable the same way (svs_pose_grad):

    T = track_pose(po, obs_point_id, obs_uvu, point_xyz, cam, T_init, True, 2.0, 15)
    loss(T).backward()                   # fills obs_uvu.grad, point_xyz.grad and cam.grad
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


def tangent_grad_to_pose(pose_qt, g_delta):
    """dL/d delta [C,6], delta = (upsilon, omega) of T <- exp(delta) T, at pose_qt [C,7] -> dL/d(qx, qy, qz, qw, tx, ty,
    tz) [C,7]: the counterpart of pose_grad_to_tangent.  Its contraction with any first-order change (dq, dt) equals
    g_delta's with the delta that change induces, omega = 2 vec(dq q*) and upsilon = dt - omega x t, for a unit q.  A
    change along q only rescales q, which se3_mul renormalises away, so the q part has no component along q.
    The device path does not renormalise c_T on input (the translation of T_ji T_i uses the rotation matrix of c_T's
    quaternion as given), so c_T must hold unit quaternions for the gradient to be that of the window."""
    qv, qw, t = pose_qt[:, 0:3], pose_qt[:, 3:4], pose_qt[:, 4:7]
    gu, gom = g_delta[:, 0:3], g_delta[:, 3:6]
    h = gom - torch.linalg.cross(t, gu)   # g_delta . delta = gu . dt + h . omega
    g_qv = 2.0 * (qw * h + torch.linalg.cross(h, qv))   # 2 (h, 0) q, the adjoint of omega = 2 vec(dq q*)
    g_qw = -2.0 * (h * qv).sum(dim=1, keepdim=True)
    return torch.cat([g_qv, g_qw, gu], dim=1)


def _as_problem(pb, e_obs, e_info, c_T=None, c_Lambda=None, cam=None):
    """pb with e_obs / e_info (and c_T / c_Lambda / cam where given) substituted: every array as a CUDA tensor on their
    device when they are CUDA tensors (the handle then analyses the window on the device, and a repeated structure
    re-sends only the numbers), else numpy."""
    subs = {}
    if cam is not None:
        subs["cam"] = tuple(float(x) for x in cam.detach().cpu().reshape(4))
    if c_T is not None:
        subs["c_T"] = c_T.detach().reshape(-1, 7)
    if c_Lambda is not None:
        subs["c_Lambda"] = c_Lambda.detach().reshape(-1, 36)
    pb = dataclasses.replace(pb, **subs)
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
    host = lambda a: a.detach().cpu().numpy().astype(np.float64) if isinstance(a, torch.Tensor) else a
    return dataclasses.replace(pb, e_obs=host(e_obs), e_info=host(e_info), c_T=host(pb.c_T), c_Lambda=host(pb.c_Lambda))


class _OptimiseWindow(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e_obs, e_info, c_T, c_Lambda, cam, ba, pb, num_iters, robust, huber_delta, lambda_init,
                grad_lambda):
        ba.set_problem(_as_problem(pb, e_obs, e_info, c_T, c_Lambda, cam))
        ba.optimize(num_iters, robust, huber_delta, lambda_init)
        dev = e_obs.device
        poses = torch.as_tensor(ba.poses(), dtype=torch.float64, device=dev)
        psi = torch.as_tensor(ba.points(), dtype=torch.float64, device=dev)
        ctx.ba, ctx.args = ba, (robust, huber_delta, grad_lambda)
        ctx.like = [None if a is None else (a.dtype, a.device, a.shape) for a in (e_obs, e_info, c_T, c_Lambda, cam)]
        ctx.c_T = None if c_T is None else c_T.detach().to(torch.float64).reshape(-1, 7)
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
        extra = [name for name, like in zip(("cT", "cLambda", "cam"), ctx.like[2:]) if like is not None]
        if extra:
            res, rc, _ = ctx.ba.window_grad(g_delta, g_psi, robust, huber_delta, grad_lambda,
                                            want=("obs", "info", *extra))
            fn = "svs_ba_window_grad"
        else:
            dobs, dinfo, rc, _ = ctx.ba.observation_grad(g_delta, g_psi, robust, huber_delta, grad_lambda)
            res, fn = dict(obs=dobs, info=dinfo), "svs_ba_observation_grad"
        if rc != 0:
            raise RuntimeError(f"{fn}: the reduced system is not positive definite (rc = {rc})")
        res = {k: torch.as_tensor(v) for k, v in res.items()}
        if "cT" in res:
            res["cT"] = tangent_grad_to_pose(ctx.c_T.to(res["cT"].device), res["cT"])
        grads = []
        for name, like in zip(("obs", "info", "cT", "cLambda", "cam"), ctx.like):
            grads.append(None if like is None else res[name].reshape(like[2]).to(like[1], like[0]))
        return (*grads, None, None, None, None, None, None, None)


class _TrackPose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, obs_uvu, point_xyz, cam, po, obs_point_id, T_init, robust_kernel, kernel_param, num_iter, initial_mu,
                grad_lambda):
        dev = obs_uvu.device
        host = lambda a: a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        if dev.type == "cuda":   # the track stays on the device (svs_calcFastMotionOnly_device)
            pid = torch.as_tensor(obs_point_id).to(dev, torch.int32)
            obs, xyz = obs_uvu.detach(), torch.as_tensor(point_xyz).detach().to(dev)
        else:
            pid, obs, xyz = host(obs_point_id), host(obs_uvu), host(point_xyz)
        cam_t = tuple(float(x) for x in host(cam).reshape(4))
        T, _ = po.calc_fast_motion_only(pid, obs, xyz, cam_t, host(T_init).astype(np.float64).reshape(7), robust_kernel,
                                        kernel_param, num_iter, initial_mu)
        T = torch.as_tensor(T, dtype=torch.float64, device=dev)
        ctx.po, ctx.grad_lambda = po, grad_lambda
        ctx.like = [(a.dtype, a.device, a.shape) if isinstance(a, torch.Tensor) else None for a in (obs_uvu, point_xyz, cam)]
        ctx.save_for_backward(T)
        return T

    @staticmethod
    def backward(ctx, g_T):
        (T,) = ctx.saved_tensors
        names = ("obs", "xyz", "cam")
        want = [w for w, like, need in zip(names, ctx.like, ctx.needs_input_grad[:3]) if like is not None and need]
        none = (None,) * 8
        if not want:
            return (None, None, None, *none)
        g = pose_grad_to_tangent(T[None], g_T.to(torch.float64)[None])[0].contiguous()
        res, rc, _ = ctx.po.grad(g if g.is_cuda else g.numpy(), ctx.grad_lambda, want)
        if rc != 0:
            raise RuntimeError(f"svs_pose_grad: H + lambda I is not positive definite (rc = {rc}); pass grad_lambda > 0")
        grads = []
        for w, like in zip(names, ctx.like):
            grads.append(torch.as_tensor(res[w]).reshape(like[2]).to(like[1], like[0]) if w in res else None)
        return (*grads, *none)


def track_pose(po, obs_point_id, obs_uvu, point_xyz, cam, T_init, robust_kernel=True, kernel_param=1.0, num_iter=50,
               initial_mu=-1.0, grad_lambda=0.0):
    """Refine the frame pose with the PoseOptimizer `po` (calcFastMotionOnly) on the observations obs_uvu [n,3] of the
    points point_xyz [npoints,3] (obs_point_id [n] indexes them), with cam (f, px, py, b) and the start T_init [7], and
    return the pose T [7] (qx, qy, qz, qw, tx, ty, tz) as a float64 tensor on obs_uvu's device.  CUDA tensors stay on
    the device (po must live on theirs).  backward() fills obs_uvu.grad, point_xyz.grad and cam.grad where they are
    tensors that require it (svs_pose_grad, one solve at H + grad_lambda I; grad_lambda > 0 for n <= 2).  The gradient
    is that of the root the LM converges to, so run it to convergence; T_init gets none.  The handle keeps the track
    between the two passes: nothing may be refined on `po` before backward() runs."""
    return _TrackPose.apply(obs_uvu, point_xyz, cam, po, obs_point_id, T_init, robust_kernel, kernel_param, num_iter,
                            initial_mu, grad_lambda)


def optimise_window(ba, pb, e_obs, e_info, num_iters, robust=True, huber_delta=1.0, lambda_init=50.0, grad_lambda=0.0,
                    *, c_T=None, c_Lambda=None, cam=None):
    """Load `pb` into the BundleAdjuster `ba` with its observations e_obs [E,3] and weights e_info [E,3] replaced by the
    given tensors, optimise it for num_iters iterations and return (pose_qt [P,7], psi [L,3]) as float64 tensors on
    their device.  c_T [C,7] (unit quaternions, see tangent_grad_to_pose), c_Lambda [C,36] or [C,6,6] and cam [4]
    (f, px, py, b), when given, replace pb's and receive gradients too (svs_ba_window_grad); with all three None the
    backward pass is svs_ba_observation_grad.  The gradients come from one adjoint solve at (H + grad_lambda I);
    grad_lambda = 0 needs a fixed pose."""
    return _OptimiseWindow.apply(e_obs, e_info, c_T, c_Lambda, cam, ba, pb, num_iters, robust, huber_delta, lambda_init,
                                 grad_lambda)
