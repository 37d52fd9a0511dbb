"""The derivative svs_ba_observation_grad computes (include/svs_b200.h), checked on the CPU: the dense reference of
ba_grad_reference.py against central differences of the oracle's own minimiser, and the quaternion chain rule of the
torch.autograd backward (scavislam_b200/autograd.py) against central differences through oracle.se3_exp / se3_mul.

The minimiser: oracle.optimize re-converged from the optimum of the unperturbed window (warm start) until it stops on
Terminate.  Its steps use g2o's H with the self-anchor term (SURVEY.md B5), which damps the anchor poses, so it converges
linearly and stops when chi2 no longer decreases in double precision, a little short of the exact minimiser.  That
stopping error, not the step h, sets the tolerances below; each was measured on these windows and given a margin.
"""
import dataclasses

import numpy as np
import pytest

import ba_grad_reference as ref
from scavislam_b200 import synth

ITERS = 3000   # upper bound: every run below stops on Terminate well before it


def _window(oracle, obs_sigma):
    """make_window(10, 200) with no pose-pose constraints, pose 0 fixed, started from the truth and converged."""
    pb = synth.make_window(10, 200, seed=7, obs_sigma=obs_sigma, outlier_frac=0)
    pb = dataclasses.replace(pb, C=0, c_i=np.zeros(0, np.int32), c_j=np.zeros(0, np.int32), c_T=np.zeros((0, 7)),
                             c_Lambda=np.zeros((0, 36)), pose_qt=pb.truth_pose_qt.copy(), psi=pb.truth_psi.copy(),
                             fixed=np.zeros(10, np.uint8))
    pb.fixed[0] = 1
    poses, psi, st = oracle.optimize(pb, ITERS, True, 1.0, 1e-5, 10)
    assert st["iterations"] < ITERS
    return dataclasses.replace(pb, pose_qt=poses, psi=psi)


def _fd_check(oracle, pb, arr, h, tol, seed):
    """Largest |central difference - reference| over 10 coordinates of `arr`, relative to the largest reference entry."""
    rng = np.random.default_rng(seed)
    g_pose = rng.normal(size=(pb.P, 6))
    g_psi = rng.normal(size=(pb.L, 3))
    dobs, dinfo = ref.observation_grad(oracle, pb, g_pose, g_psi, robust=True, delta=1.0, lam=0.0)
    want = dobs if arr == "e_obs" else dinfo
    g_pose[0] = 0   # pose 0 is fixed: its entry of g must not matter, and the loss below does not see it

    def loss(p):
        poses, psi, st = oracle.optimize(p, ITERS, True, 1.0, 1e-5, 10)
        assert st["iterations"] < ITERS
        d = np.array([oracle.se3_log(oracle.se3_mul(poses[q], oracle.se3_inv(pb.pose_qt[q]))) for q in range(pb.P)])
        return float(np.sum(g_pose * d) + np.sum(g_psi * (psi - pb.psi)))

    err = 0.0
    for e in rng.choice(pb.E, 10, replace=False):
        k = int(rng.integers(3))
        step = h * (1.0 if arr == "e_obs" else pb.e_info[e, k])   # weights: a relative step
        vals = []
        for s in (1, -1):
            a = getattr(pb, arr).copy()
            a[e, k] += s * step
            vals.append(loss(dataclasses.replace(pb, **{arr: a})))
        fd = (vals[0] - vals[1]) / (2 * step)
        err = max(err, abs(fd - want[e, k]))
    rel = err / np.abs(want).max()
    assert rel <= tol, f"{arr}: {rel:.3e} of the largest entry"
    return dobs, dinfo


def test_zero_residual_window_observations(oracle):
    """Exact observations: the Gauss-Newton derivative is the derivative of the minimiser.  h = 1e-4 px; measured
    error <= 1.4e-3 of the largest entry (the minimiser's stopping error), tolerance 5e-3."""
    pb = _window(oracle, 0.0)
    dobs, dinfo = _fd_check(oracle, pb, "e_obs", 1e-4, 5e-3, seed=1)
    assert np.abs(dinfo).max() <= 1e-9 * np.abs(dobs).max()   # the weights' gradient vanishes with the residual


def test_small_noise_window_weights(oracle):
    """obs_sigma = 1e-3 px: dL/domega is first order in the residual, and so is the Gauss-Newton error relative to it.
    The signal is small here, so the minimiser's stopping error dominates: measured 3.6e-2, 3.0e-2 and 1.3e-2 of the
    largest entry for relative weight steps h = 3e-2, 1e-1 and 3e-1.  h = 3e-1 (the minimiser is smooth in the
    weights), tolerance 4e-2: a missing rho', a wrong sign or the B5 term in H each give errors of order 1."""
    pb = _window(oracle, 1e-3)
    _fd_check(oracle, pb, "e_info", 3e-1, 4e-2, seed=2)


def test_reference_h_is_the_oracle_h_without_the_self_anchor_term(oracle):
    """The reference's H equals oracle.full_system's except on the anchor diagonals of self-anchored landmarks (B5)."""
    pb = synth.make_config("C1")
    H, _ = ref.gauss_newton(oracle, pb, True, 1.0)
    Hf, _, _ = oracle.full_system(pb, True, 1.0)
    scale = np.abs(Hf).max()
    D = H - Hf
    for p in range(pb.P):
        D[6 * p:6 * p + 6, 6 * p:6 * p + 6] = 0   # pose diagonal blocks: B5 lives there
    assert np.abs(D).max() <= 1e-12 * scale
    self_anchor = np.zeros(pb.P, bool)
    self_anchor[pb.e_pose[pb.e_pose == pb.e_anchor]] = True
    for p in np.nonzero(self_anchor)[0]:
        assert np.abs(H[6 * p:6 * p + 6, 6 * p:6 * p + 6] - Hf[6 * p:6 * p + 6, 6 * p:6 * p + 6]).max() > 1e-6 * scale


def test_pose_gradient_chain_rule(oracle):
    """autograd.pose_grad_to_tangent against central differences of L(exp(delta) T) in delta, with
    L = g . (qx, qy, qz, qw, tx, ty, tz)."""
    torch = pytest.importorskip("torch")
    from scavislam_b200.autograd import pose_grad_to_tangent
    rng = np.random.default_rng(5)
    pb = synth.make_config("C1")
    T = pb.pose_qt[:6]
    g = rng.normal(size=(6, 7))
    got = pose_grad_to_tangent(torch.as_tensor(T), torch.as_tensor(g)).numpy()
    h = 1e-6
    want = np.zeros((6, 6))
    for p in range(6):
        for k in range(6):
            d = np.zeros(6)
            d[k] = h
            tp = oracle.se3_mul(oracle.se3_exp(d), T[p])
            tm = oracle.se3_mul(oracle.se3_exp(-d), T[p])
            want[p, k] = g[p] @ (tp - tm) / (2 * h)
    assert np.abs(got - want).max() <= 1e-8 * np.abs(want).max()
