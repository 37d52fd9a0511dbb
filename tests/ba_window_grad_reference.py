"""Dense reference of svs_ba_window_grad (include/svs_b200.h), built from the oracle's per-edge and pose-pose functions.

H and the edge rows come from ba_grad_reference.gauss_newton (no self-anchor term, SURVEY.md B5), and v solves
(H + lambda I) v = g over the free variables as in ba_grad_reference.observation_grad.  Then, per pose-pose constraint c
with e_c = oracle.posepose_error and (J_i, J_j) = oracle.posepose_jacobians (zero for a fixed pose):
    w_c = J_i v_i + J_j v_j,  dL/dLambda_c = -(w e^T + e w^T) / 2,  dL/d delta_c = -X^T Lambda_c w,  X = third(I, e_c)
(X is posepose_jacobians' J_i at the identity), and for the camera dL/dcam_k = sum_e (de_e/dcam_k) . dL/dz_e, with
de_e/dcam_k taken from oracle.edge_error: e is affine in each camera parameter on its own (y does not depend on the
camera), so a central difference is exact up to rounding, and a step of 1e3 makes that rounding negligible.
"""
import numpy as np

import ba_grad_reference as ref

IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


def adjoint(oracle, pb, g_pose=None, g_psi=None, robust=True, delta=1.0, lam=0.0):
    """(v [6P + 3L] over the free variables, edge list of ref.gauss_newton)."""
    P, L = pb.P, pb.L
    H, edges = ref.gauss_newton(oracle, pb, robust, delta)
    g = np.zeros(6 * P + 3 * L)
    if g_pose is not None:
        g[:6 * P] = np.asarray(g_pose, np.float64).reshape(-1)
    if g_psi is not None:
        g[6 * P:] = np.asarray(g_psi, np.float64).reshape(-1)
    has_edges = np.zeros(L, bool)
    has_edges[np.asarray(pb.e_point, np.int64)] = True
    free = np.concatenate([np.repeat(np.asarray(pb.fixed) == 0, 6), np.repeat(has_edges, 3)])
    v = np.zeros_like(g)
    A = H[np.ix_(free, free)] + lam * np.eye(int(free.sum()))
    v[free] = np.linalg.solve(A, g[free])
    return v, edges


def camera_jacobian(oracle, pb, e):
    """de_e/d(f, px, py, b) [3,4] of edge e at pb's state."""
    cam = np.asarray(pb.cam, np.float64)
    p, a, l = int(pb.e_pose[e]), int(pb.e_anchor[e]), int(pb.e_point[e])
    out = np.zeros((3, 4))
    for k in range(4):
        d = np.zeros(4)
        d[k] = 1e3
        hi = oracle.edge_error(cam + d, pb.pose_qt[p], pb.pose_qt[a], pb.psi[l], pb.e_obs[e])
        lo = oracle.edge_error(cam - d, pb.pose_qt[p], pb.pose_qt[a], pb.psi[l], pb.e_obs[e])
        out[:, k] = (hi - lo) / 2e3
    return out


def window_grad(oracle, pb, g_pose=None, g_psi=None, robust=True, delta=1.0, lam=0.0):
    """dict obs / info [E,3], cT [C,6], cLambda [C,36], cam [4] at pb's state (pose_qt, psi) for the upstream gradient
    (g_pose [P,6] in the tangent (upsilon, omega), g_psi [L,3]); None = 0."""
    v, edges = adjoint(oracle, pb, g_pose, g_psi, robust, delta, lam)
    dobs, dinfo, dcam = np.zeros((pb.E, 3)), np.zeros((pb.E, 3)), np.zeros(4)
    for e, ed in enumerate(edges):
        if ed is None:
            continue
        idx, J, err, r1, om = ed
        jv = J @ v[idx]
        dobs[e] = -r1 * om * jv
        dinfo[e] = -r1 * err * jv
        dcam += camera_jacobian(oracle, pb, e).T @ dobs[e]
    dcT, dcLam = np.zeros((pb.C, 6)), np.zeros((pb.C, 36))
    for c in range(pb.C):
        i, j = int(pb.c_i[c]), int(pb.c_j[c])
        err = oracle.posepose_error(pb.c_T[c], pb.pose_qt[i], pb.pose_qt[j])
        Ji, Jj = oracle.posepose_jacobians(pb.c_T[c], err)
        w = np.zeros(6)
        if not pb.fixed[i]:
            w += Ji @ v[6 * i:6 * i + 6]
        if not pb.fixed[j]:
            w += Jj @ v[6 * j:6 * j + 6]
        X, _ = oracle.posepose_jacobians(IDENTITY, err)
        Lam = np.asarray(pb.c_Lambda[c], np.float64).reshape(6, 6)
        dcT[c] = -X.T @ Lam @ w
        dcLam[c] = (-0.5 * (np.outer(w, err) + np.outer(err, w))).reshape(36)
    return dict(obs=dobs, info=dinfo, cT=dcT, cLambda=dcLam, cam=dcam)
