"""The derivative svs_ba_window_grad computes (include/svs_b200.h) for the pose-pose constraints and the camera, checked
on the CPU: the dense reference of ba_window_grad_reference.py against central differences of the oracle's own
minimiser, and autograd.tangent_grad_to_pose against central differences through oracle.se3_exp / se3_mul.

The minimiser is oracle.optimize re-converged from the optimum of the unperturbed window until it stops on Terminate, as
in test_ba_grad_cpu.py: its stopping error, not the step h, sets the tolerances below.  Each was measured on these
windows and given a margin.  make_window(10, 200) keeps its pose-pose constraints here (C = 46, both orders of each
pair), and pose 0 is fixed.
"""
import dataclasses

import numpy as np
import pytest

import ba_window_grad_reference as wref
from scavislam_b200 import synth

ITERS = 3000   # upper bound: every run below stops on Terminate well before it


def _window(oracle, obs_sigma, exact_constraints):
    """make_window(10, 200) with its constraints, pose 0 fixed, started from the truth and converged.
    exact_constraints: every T_ji is the true relative pose, so that with obs_sigma = 0 every residual vanishes."""
    pb = synth.make_window(10, 200, seed=7, obs_sigma=obs_sigma, outlier_frac=0)
    pb = dataclasses.replace(pb, pose_qt=pb.truth_pose_qt.copy(), psi=pb.truth_psi.copy(), fixed=np.zeros(10, np.uint8),
                             c_T=pb.c_T.copy())
    pb.fixed[0] = 1
    if exact_constraints:
        T = pb.truth_pose_qt
        for c in range(pb.C):
            pb.c_T[c] = oracle.se3_mul(T[pb.c_j[c]], oracle.se3_inv(T[pb.c_i[c]]))
    poses, psi, st = oracle.optimize(pb, ITERS, True, 1.0, 1e-5, 10)
    assert st["iterations"] < ITERS
    return dataclasses.replace(pb, pose_qt=poses, psi=psi)


def _setup(oracle, pb, seed):
    rng = np.random.default_rng(seed)
    g_pose = rng.normal(size=(pb.P, 6))
    g_psi = rng.normal(size=(pb.L, 3))
    want = wref.window_grad(oracle, pb, g_pose, g_psi, robust=True, delta=1.0, lam=0.0)
    g_pose[0] = 0   # pose 0 is fixed: its entry of g must not matter, and the loss below does not see it

    def loss(p):
        poses, psi, st = oracle.optimize(p, ITERS, True, 1.0, 1e-5, 10)
        assert st["iterations"] < ITERS
        d = np.array([oracle.se3_log(oracle.se3_mul(poses[q], oracle.se3_inv(pb.pose_qt[q]))) for q in range(pb.P)])
        return float(np.sum(g_pose * d) + np.sum(g_psi * (psi - pb.psi)))
    return rng, want, loss


def _central(loss, make, step):
    return (loss(make(step)) - loss(make(-step))) / (2 * step)


def test_constraint_measurement_on_a_zero_residual_window(oracle):
    """c_T perturbed as exp(+-h e_k) T_ji, h = 1e-4.  Measured error 4.8e-6 of the largest entry, tolerance 1e-4.
    e_c = 0 here, so X = I: the factor X of dL/d delta is checked against the reference on the GPU side, at
    non-vanishing residuals."""
    pb = _window(oracle, 0.0, True)
    rng, want, loss = _setup(oracle, pb, seed=11)
    g = want["cT"]
    err = 0.0
    for c in rng.choice(pb.C, 10, replace=False):
        k = int(rng.integers(6))

        def make(s, c=c, k=k):
            d = np.zeros(6)
            d[k] = s
            cT = pb.c_T.copy()
            cT[c] = oracle.se3_mul(oracle.se3_exp(d), pb.c_T[c])
            return dataclasses.replace(pb, c_T=cT)
        err = max(err, abs(_central(loss, make, 1e-4) - g[c, k]))
    rel = err / np.abs(g).max()
    assert rel <= 1e-4, f"c_T: {rel:.3e} of the largest entry"


def test_constraint_information_on_a_small_noise_window(oracle):
    """obs_sigma = 1e-3 px and the synthetic constraints' own measurement noise: dL/dLambda is first order in the
    constraint residual, as dL/dinfo is in the edge residual.  Lambda_ab and Lambda_ba move together by
    h sqrt(Lambda_aa Lambda_bb), h = 1e-2, which the reference gives as G_ab + G_ba (G_aa on the diagonal).
    Measured error 1.5e-3 of the largest entry, tolerance 1e-2: a wrong sign or a missing 1/2 gives errors of order
    1."""
    pb = _window(oracle, 1e-3, False)
    rng, want, loss = _setup(oracle, pb, seed=12)
    G = want["cLambda"].reshape(pb.C, 6, 6)
    assert np.array_equal(G, np.transpose(G, (0, 2, 1)))
    err = 0.0
    for n, c in enumerate(rng.choice(pb.C, 10, replace=False)):
        a, b = (n % 6, n % 6) if n < 4 else tuple(int(x) for x in rng.choice(6, 2, replace=False))
        L0 = pb.c_Lambda[c].reshape(6, 6)
        step = 1e-2 * np.sqrt(L0[a, a] * L0[b, b])

        def make(s, c=c, a=a, b=b):
            cL = pb.c_Lambda.copy().reshape(pb.C, 6, 6)
            cL[c, a, b] += s
            if a != b:
                cL[c, b, a] += s
            return dataclasses.replace(pb, c_Lambda=cL.reshape(pb.C, 36))
        w = G[c, a, b] if a == b else G[c, a, b] + G[c, b, a]
        err = max(err, abs(_central(loss, make, step) - w))
    rel = err / np.abs(G).max()
    assert rel <= 1e-2, f"c_Lambda: {rel:.3e} of the largest entry"


def test_camera_on_a_zero_residual_window(oracle):
    """Each of f, px, py (h = 1e-3 px) and b (h = 1e-6 m).  Measured error 2.5e-4 of the largest entry, tolerance
    2e-3."""
    pb = _window(oracle, 0.0, True)
    _, want, loss = _setup(oracle, pb, seed=13)
    g = want["cam"]
    err = 0.0
    for k, h in enumerate((1e-3, 1e-3, 1e-3, 1e-6)):
        def make(s, k=k):
            cam = np.array(pb.cam, np.float64)
            cam[k] += s
            return dataclasses.replace(pb, cam=cam)
        err = max(err, abs(_central(loss, make, h) - g[k]) / np.abs(g).max())
    assert err <= 2e-3, f"cam: {err:.3e} of the largest entry"


def test_tangent_gradient_chain_rule(oracle):
    """autograd.tangent_grad_to_pose: its contraction with a first-order change (dq, dt) equals g_delta's with the
    delta = log(T' T^-1) that change induces (T' with q + h dq renormalised), by central differences; dq includes a
    component along q, which changes nothing, and the q part of the result is orthogonal to q.  h = 1e-6; measured
    error <= 1.4e-11 (relative to the largest entries of the result and of the change), tolerance 1e-8."""
    torch = pytest.importorskip("torch")
    from scavislam_b200.autograd import tangent_grad_to_pose
    rng = np.random.default_rng(15)
    pb = synth.make_config("C1")
    T = pb.pose_qt[:6]
    g_delta = rng.normal(size=(6, 6))
    got = tangent_grad_to_pose(torch.as_tensor(T), torch.as_tensor(g_delta)).numpy()
    assert np.abs(np.sum(got[:, :4] * T[:, :4], axis=1)).max() <= 1e-12 * np.abs(got).max()
    h = 1e-6
    for p in range(6):
        for _ in range(3):
            dqt = rng.normal(size=7)

            def moved(s):
                q = T[p, :4] + s * dqt[:4]
                return np.concatenate([q / np.linalg.norm(q), T[p, 4:] + s * dqt[4:]])
            dp = oracle.se3_log(oracle.se3_mul(moved(h), oracle.se3_inv(T[p])))
            dm = oracle.se3_log(oracle.se3_mul(moved(-h), oracle.se3_inv(T[p])))
            want = g_delta[p] @ (dp - dm) / (2 * h)
            assert abs(got[p] @ dqt - want) <= 1e-8 * np.abs(got).max() * np.abs(dqt).max()
