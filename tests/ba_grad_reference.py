"""Dense reference of svs_ba_observation_grad (include/svs_b200.h), built from the oracle's per-edge functions.

H is assembled from scratch, not taken from oracle.full_system, because that one reproduces g2o's self-anchor term
(SURVEY.md B5), which the gradient's H must not contain: rows of J_e from oracle.edge_jacobians with the pose and anchor
columns summed into one pose when they coincide, weights rho'_e Omega_e, the pose-pose blocks from
oracle.posepose_jacobians.  Then (H + lambda I) v = g over the free variables by np.linalg.solve, and
dL/dz_e = -rho'_e Omega_e (J_e v), dL/domega_{e,k} = -rho'_e e_{e,k} (J_e v)_k.
"""
import numpy as np


def huber_weight(e2, robust, delta):
    """rho' of g2o's RobustKernelHuber at e2 = e^T Omega e (1 when not robust)."""
    return 1.0 if (not robust or e2 <= delta * delta) else delta / np.sqrt(e2)


def gauss_newton(oracle, pb, robust=True, delta=1.0):
    """(H [n,n] without the B5 term, per-edge list of (J [3,n] sparse as (cols, block), err, rho', omega) or None)."""
    P, L = pb.P, pb.L
    n = 6 * P + 3 * L
    H = np.zeros((n, n))
    cam = np.asarray(pb.cam, np.float64)
    edges = []
    for e in range(pb.E):
        om = np.asarray(pb.e_info[e], np.float64)
        if not om.any():
            edges.append(None)
            continue
        p, a, l = int(pb.e_pose[e]), int(pb.e_anchor[e]), int(pb.e_point[e])
        Tp, Ta, psi = pb.pose_qt[p], pb.pose_qt[a], pb.psi[l]
        Jpsi, Jp, Ja = oracle.edge_jacobians(cam, Tp, Ta, psi)
        err = oracle.edge_error(cam, Tp, Ta, psi, pb.e_obs[e])
        r1 = huber_weight(float(np.sum(om * err * err)), robust, delta)
        cols = {}
        for pose, J in ((p, Jp), (a, Ja)):
            if not pb.fixed[pose]:
                cols[pose] = cols.get(pose, 0) + J
        idx = [np.arange(6 * q, 6 * q + 6) for q in cols] + [np.arange(6 * P + 3 * l, 6 * P + 3 * l + 3)]
        idx = np.concatenate(idx)
        J = np.hstack(list(cols.values()) + [Jpsi])
        H[np.ix_(idx, idx)] += J.T @ (r1 * om[:, None] * J)
        edges.append((idx, J, err, r1, om))
    for c in range(pb.C):
        i, j = int(pb.c_i[c]), int(pb.c_j[c])
        err = oracle.posepose_error(pb.c_T[c], pb.pose_qt[i], pb.pose_qt[j])
        Ji, Jj = oracle.posepose_jacobians(pb.c_T[c], err)
        Lam = np.asarray(pb.c_Lambda[c], np.float64).reshape(6, 6)
        blocks = [(q, J) for q, J in ((i, Ji), (j, Jj)) if not pb.fixed[q]]
        for qa, Ja_ in blocks:
            for qb, Jb_ in blocks:
                H[6 * qa:6 * qa + 6, 6 * qb:6 * qb + 6] += Ja_.T @ Lam @ Jb_
    return H, edges


def observation_grad(oracle, pb, g_pose=None, g_psi=None, robust=True, delta=1.0, lam=0.0):
    """(dL_dobs [E,3], dL_dinfo [E,3]) at pb's state (pose_qt, psi) for the upstream gradient (g_pose [P,6] in the
    tangent (upsilon, omega), g_psi [L,3]); None = 0."""
    P, L = pb.P, pb.L
    H, edges = gauss_newton(oracle, pb, robust, delta)
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
    dobs, dinfo = np.zeros((pb.E, 3)), np.zeros((pb.E, 3))
    for e, ed in enumerate(edges):
        if ed is None:
            continue
        idx, J, err, r1, om = ed
        jv = J @ v[idx]
        dobs[e] = -r1 * om * jv
        dinfo[e] = -r1 * err * jv
    return dobs, dinfo
