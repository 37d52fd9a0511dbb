"""The derivative svs_pose_grad computes (include/svs_b200.h), checked on the CPU: the dense reference of
pose_grad_reference.py against central differences of the root the LM converges to.

That root is F(T) = sum_i J_i^T w_i f_i = 0, not the minimiser of the robust chi2 (they differ on a track with
outliers).  It is found here by undamped iteration of the LM's normal equations, started from the oracle LM's result
and run until the step is below 1e-15: the LM itself stops up to ~3.5e-7 away, which would swamp a difference quotient.
The reference drops the derivatives of J_i (Gauss-Newton), which is exact only for vanishing residuals; with 0.3 px of
noise (and 25 px outliers) that error, not the step h, sets the tolerances below.  Each was measured on these tracks
and given a margin.
"""
import numpy as np
import pytest

import pose_grad_reference as ref
from scavislam_b200 import synth_pose as sp

# (step, which) per input: pixels, metres, and (f, px, py, b)
H_OBS, H_XYZ, H_CAM = 1e-3, 1e-5, (1e-3, 1e-3, 1e-3, 1e-6)


def _track(oracle, n, seed, robust, b, **kw):
    tr = sp.make_track(n, seed=seed, **kw)
    T_lm, _ = oracle.calc_fast_motion_only(tr["pid"], tr["obs"], tr["xyz"], tr["cam"], tr["T_init"], robust, b, 50)
    T = ref.root(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T_lm, robust, b)
    return tr, T


def _fd_errors(oracle, tr, T, robust, b, g, refs, obs_idx, pts_idx):
    """Largest |central difference - reference| per input kind, relative to that kind's largest reference entry, over
    the observations obs_idx, the points pts_idx and all four camera parameters."""
    dobs, dxyz, dcam = refs

    def loss(obs=tr["obs"], xyz=tr["xyz"], cam=tr["cam"]):
        Tp = ref.root(oracle, tr["pid"], obs, xyz, cam, T, robust, b)
        return float(g @ ref.tangent(oracle, Tp, T))

    def cd(name, arr, idx, h):
        vals = []
        for s in (1, -1):
            a = np.array(arr, np.float64)
            a[idx] += s * h
            vals.append(loss(**{name: a}))
        return (vals[0] - vals[1]) / (2 * h)

    e_obs = max(abs(cd("obs", tr["obs"], (i, k), H_OBS) - dobs[i, k]) for i in obs_idx for k in range(3))
    e_xyz = max(abs(cd("xyz", tr["xyz"], (p, k), H_XYZ) - dxyz[p, k]) for p in pts_idx for k in range(3))
    e_cam = max(abs(cd("cam", tr["cam"], k, H_CAM[k]) - dcam[k]) / abs(dcam).max() for k in range(4))
    return e_obs / np.abs(dobs).max(), e_xyz / np.abs(dxyz).max(), e_cam


def _g(seed):
    return np.random.default_rng(seed).normal(size=6)


def test_projection_derivatives(oracle):
    """dpi/dX (through R) and dpi/dcam of the reference against central differences of oracle.pose_map; and the
    vectorised map and frame Jacobian of the root solver against the oracle's."""
    tr = sp.make_track(20, seed=4)
    T, cam = tr["T_true"], tr["cam"]
    R = ref.rot(T[:4])
    m, y = ref.project(cam, T, tr["xyz"])
    Jv = ref.frame_jac(cam, y)
    for p in range(5):
        X = tr["xyz"][p]
        yp = R @ X + T[4:]
        assert np.abs(m[p] - oracle.pose_map(cam, T, X)).max() <= 1e-12 * np.abs(m[p]).max()
        assert np.abs(Jv[p] - oracle.pose_frame_jac(cam, T, X)).max() <= 1e-12 * np.abs(Jv[p]).max()
        want_X, want_c = np.zeros((3, 3)), np.zeros((3, 4))
        for k in range(3):
            d = np.zeros(3); d[k] = 1e-6
            want_X[:, k] = (oracle.pose_map(cam, T, X + d) - oracle.pose_map(cam, T, X - d)) / 2e-6
        for k in range(4):
            d = np.zeros(4); d[k] = 1e-6
            want_c[:, k] = (oracle.pose_map(cam + d, T, X) - oracle.pose_map(cam - d, T, X)) / 2e-6
        assert np.abs(ref.dpi_dy(cam, yp) @ R - want_X).max() <= 1e-7 * np.abs(want_X).max()
        assert np.abs(ref.dpi_dcam(cam, yp) - want_c).max() <= 1e-7 * np.abs(want_c).max()


def test_root_is_where_the_lm_stops(oracle):
    """The LM's result lies within its stopping distance of the root (and the root's step has converged)."""
    tr = sp.make_track(300, seed=2, outlier_frac=0.1)
    T_lm, _ = oracle.calc_fast_motion_only(tr["pid"], tr["obs"], tr["xyz"], tr["cam"], tr["T_init"], True, 2.0, 50)
    T = ref.root(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T_lm, True, 2.0)
    assert np.abs(T - T_lm).max() < 1e-6
    assert np.abs(T - ref.root(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T, True, 2.0)).max() < 1e-13


CASES = {   # name: (make_track kwargs, robust, kernel_param)
    "robust_off": (dict(n=200, seed=5), False, 1.0),
    "robust_all_inside": (dict(n=200, seed=6), True, 10.0),   # 0.3 px of noise: every residual inside b
    "outliers": (dict(n=300, seed=2, outlier_frac=0.1), True, 2.0),
    "shared_points": (dict(n=300, seed=3, shared_points=True, outlier_frac=0.1), True, 2.0),
}
# Measured (obs, xyz, cam), relative to the largest reference entry of each kind:
#   robust_off 4.2e-5, 8.0e-4, 3.1e-4; robust_all_inside 1.8e-5, 2.1e-4, 1.8e-4;
#   outliers 3.0e-4, 3.5e-3, 6.5e-4; shared_points 4.6e-5, 1.5e-3, 1.7e-3.
TOL = (1e-3, 1e-2, 5e-3)


@pytest.mark.parametrize("case", list(CASES))
def test_reference_against_central_differences(oracle, case):
    kw, robust, b = CASES[case]
    tr, T = _track(oracle, robust=robust, b=b, **kw)
    g = _g(1)
    dobs, dxyz, dcam, _ = ref.pose_grad(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T, g, 0.0, robust, b)
    rng = np.random.default_rng(7)
    obs_idx = list(rng.choice(len(tr["pid"]), 4, replace=False))
    r = np.linalg.norm(tr["obs"] - ref.project(tr["cam"], T, tr["xyz"][tr["pid"]])[0], axis=1)
    if robust and (r >= b).any():
        obs_idx += list(np.nonzero(r >= b)[0][:4])   # observations beyond the kernel's quadratic branch
    pts_idx = sorted({int(tr["pid"][i]) for i in obs_idx})[:4]
    errs = _fd_errors(oracle, tr, T, robust, b, g, (dobs, dxyz, dcam), obs_idx, pts_idx)
    assert all(e <= t for e, t in zip(errs, TOL)), errs


def test_holding_the_weight_fails_on_outliers(oracle):
    """W = w I (the reweighting held at its value) instead of d(w f)/df.  On the outlier track the observation
    gradient it gives is off by 1.8e-2 of the largest entry (measured), 18 times the tolerance the exact W passes with
    3.0e-4.  Against the exact reference on the outliers' own entries it is off by 0.21 of their largest (measured)."""
    kw, robust, b = CASES["outliers"]
    tr, T = _track(oracle, robust=robust, b=b, **kw)
    g = _g(1)
    exact = ref.pose_grad(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T, g, 0.0, robust, b)[:3]
    held = ref.pose_grad(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T, g, 0.0, robust, b, hold_w=True)[:3]
    r = np.linalg.norm(tr["obs"] - ref.project(tr["cam"], T, tr["xyz"][tr["pid"]])[0], axis=1)
    out = list(np.nonzero(r >= b)[0][:4])
    pts = sorted({int(tr["pid"][i]) for i in out})
    errs = _fd_errors(oracle, tr, T, robust, b, g, held, out, pts)
    assert errs[0] > 10 * TOL[0], errs
    own = np.abs(held[0][out] - exact[0][out]).max() / np.abs(exact[0][out]).max()
    assert own > 0.1, own
