"""Seeded synthetic stereo image generator for the front-end path (SURVEY.md section 8d, C3):
a textured ground plane and fronto-parallel boxes rendered to 640x480 uint8 left images with
ground-truth float32 disparity, via multi-octave value noise.  Input generation only."""
from __future__ import annotations

import numpy as np

from .synth import CAM_B, CAM_F, CAM_H, CAM_PX, CAM_PY, CAM_W


def _value_noise(u, v, seed, octaves=5):
    """Smooth multi-octave value noise at continuous texture coordinates (u, v)."""
    rng = np.random.default_rng(seed)
    out = np.zeros_like(u, dtype=np.float64)
    amp, tot = 1.0, 0.0
    for o in range(octaves):
        n = 8 << o
        lat = rng.uniform(0, 1, (n + 1, n + 1))
        x = (u * n) % n
        y = (v * n) % n
        # (u * n) % n rounds to n for u just below a multiple of 1: keep the cell index in range (fx = 1 there)
        x0 = np.minimum(np.floor(x).astype(int), n - 1); y0 = np.minimum(np.floor(y).astype(int), n - 1)
        fx = x - x0; fy = y - y0
        sx = fx * fx * (3 - 2 * fx); sy = fy * fy * (3 - 2 * fy)
        a = lat[y0, x0]; b = lat[y0, x0 + 1]; c = lat[y0 + 1, x0]; d = lat[y0 + 1, x0 + 1]
        out += amp * ((a * (1 - sx) + b * sx) * (1 - sy) + (c * (1 - sx) + d * sx) * sy)
        tot += amp
        amp *= 0.55
    return out / tot


def render_frame(t_wc, yaw, seed=77, w=CAM_W, h=CAM_H, cam=None, noise_seed=None):
    """Render the left image (uint8) and disparity (float32) seen from camera centre t_wc (x,y,z)
    with heading yaw (rotation about the y axis).  Scene: ground plane y = 1.5 m (y down) and a far
    wall z = 25 m, plus a few boxes (fronto-parallel quads) -- all textured with value noise.
    cam = (f, px, py, baseline) of the left camera; None is the default 640x480 camera of synth.
    noise_seed seeds the sensor noise; None is seed + 100."""
    f, px, py, b = (CAM_F, CAM_PX, CAM_PY, CAM_B) if cam is None else cam
    uu, vv = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    dx = (uu - px) / f; dy = (vv - py) / f; dz = np.ones_like(dx)
    c, s = np.cos(yaw), np.sin(yaw)
    # ray directions in world
    rx = c * dx + s * dz; ry = dy; rz = -s * dx + c * dz
    depth = np.full((h, w), np.inf)
    tex = np.zeros((h, w))
    # ground plane y = 1.5
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = (1.5 - t_wc[1]) / ry
    ok = (ry > 1e-6) & (lam > 0.2) & np.isfinite(lam)
    lam = np.where(ok, lam, 1.0)
    X = t_wc[0] + lam * rx; Z = t_wc[2] + lam * rz
    g = _value_noise(X / 6.0, Z / 6.0, seed)
    zc = lam  # camera-frame depth along optical axis = lam * dz(=1) in camera coords
    upd = ok & (zc < depth)
    depth[upd] = zc[upd]; tex[upd] = g[upd]
    # far wall z = 25 (world)
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = (25.0 - t_wc[2]) / rz
    ok = (rz > 1e-6) & (lam > 0.2) & np.isfinite(lam)
    lam = np.where(ok, lam, 1.0)
    X = t_wc[0] + lam * rx; Y = t_wc[1] + lam * ry
    g = _value_noise(X / 8.0 + 3.1, Y / 8.0 + 1.7, seed + 1)
    upd = ok & (lam < depth)
    depth[upd] = lam[upd]; tex[upd] = g[upd]
    # boxes: quads facing -z at depth zb, centred (xb, yb), half sizes
    rngb = np.random.default_rng(seed + 2)
    for k in range(6):
        xb = rngb.uniform(-6, 6); zb = rngb.uniform(6, 20); hw = rngb.uniform(0.5, 1.5); hh = rngb.uniform(0.5, 1.4)
        yb = 1.5 - hh
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = (zb - t_wc[2]) / rz
        okl = (rz > 1e-6) & np.isfinite(lam) & (lam > 0.2)
        lam = np.where(okl, lam, 1.0)
        X = t_wc[0] + lam * rx; Y = t_wc[1] + lam * ry
        ok = okl & (np.abs(X - xb) < hw) & (np.abs(Y - yb) < hh)
        g = _value_noise((X - xb) / 2.0 + k, (Y - yb) / 2.0 + 2 * k, seed + 3 + k, octaves=4)
        upd = ok & (lam < depth)
        depth[upd] = lam[upd]; tex[upd] = g[upd]
    img = np.clip(255.0 * (0.15 + 0.8 * tex), 0, 255)
    img[~np.isfinite(depth)] = 30
    # sensor noise, deterministic
    img = img + np.random.default_rng(seed + 100 if noise_seed is None else noise_seed).normal(0, 1.0, img.shape)
    img8 = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    disp = np.where(np.isfinite(depth), f * b / np.maximum(depth, 1e-6), 0.0).astype(np.float32)
    return img8, disp


def render_stereo_pair(t_wc, yaw, seed=77, w=CAM_W, h=CAM_H, cam=None):
    """A rectified stereo pair: the left image and its ground-truth disparity as render_frame gives them, and the right
    image seen from t_wc + b (cos yaw, 0, -sin yaw), the left camera's x axis.  The right image has its own sensor
    noise (seed + 200): with the left image's noise the same at every pixel, a matcher would be flattered."""
    f, px, py, b = (CAM_F, CAM_PX, CAM_PY, CAM_B) if cam is None else cam
    t_wc = np.asarray(t_wc, dtype=np.float64)
    left, disp = render_frame(t_wc, yaw, seed, w, h, cam)
    t_r = t_wc + b * np.array([np.cos(yaw), 0.0, -np.sin(yaw)])
    right, _ = render_frame(t_r, yaw, seed, w, h, cam, noise_seed=seed + 200)
    return left, right, disp


def _render_job(args):
    pos, yaw, seed, w, h, cam = args
    img, disp = render_frame(np.asarray(pos), yaw, seed, w, h, cam)
    return img, disp


def sequence(n_frames=8, seed=77, step=0.02, dyaw=np.deg2rad(0.2), workers=1, w=CAM_W, h=CAM_H, cam=None):
    """Frames along a gentle arc: 2 cm / 0.2 deg inter-frame motion.  `workers` > 1 renders the frames in a process
    pool (the renderer is plain numpy, about a second per 640x480 frame): same images, bit for bit.  (w, h, cam) give
    another image size and camera (f, px, py, baseline), as in render_frame."""
    poses = []
    pos = np.array([0.0, 0.0, 0.0]); yaw = 0.0
    for i in range(n_frames):
        poses.append((pos.copy(), yaw))
        pos = pos + step * np.array([np.sin(yaw), 0.0, np.cos(yaw)])
        yaw += dyaw
    if workers > 1 and n_frames > 2:
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(workers, n_frames)) as pool:
            rendered = pool.map(_render_job, [(p.tolist(), y, seed, w, h, cam) for p, y in poses])
    else:
        rendered = [render_frame(p, y, seed, w, h, cam) for p, y in poses]
    return [dict(img=im, disp=dp, pos=p, yaw=y) for (im, dp), (p, y) in zip(rendered, poses)]
