"""Dense numpy restatement of svs_pose_grad (include/svs_b200.h): the derivative of the pose calcFastMotionOnly returns,
which is the root of F(T) = sum_i J_i^T w_i f_i (the LM's right-hand side), with respect to its observations, points
and camera.  Residuals and frame Jacobians come from the oracle (oracle.pose_map, oracle.pose_frame_jac); dpi/dX and
dpi/dcam are written out here.  TEST INFRASTRUCTURE ONLY.

Also here: the root itself, found by undamped iteration of the LM's own normal equations (vectorised restatements of
the two oracle functions, which the CPU tests compare with the oracle), for the central differences the reference is
checked against.
"""
import numpy as np

EPS = 1e-10   # global.h:106


def rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def dpi_dy(cam, y):
    """d map_uvu / d y for the point y in the camera: 3 x 3."""
    f, b = cam[0], cam[3]
    return np.array([[f / y[2], 0, -f * y[0] / y[2] ** 2],
                     [0, f / y[2], -f * y[1] / y[2] ** 2],
                     [f / y[2], 0, -f * (y[0] - b) / y[2] ** 2]])


def dpi_dcam(cam, y):
    """d map_uvu / d (f, px, py, b): 3 x 4."""
    f = cam[0]
    return np.array([[y[0] / y[2], 1, 0, 0],
                     [y[1] / y[2], 0, 1, 0],
                     [(y[0] - cam[3]) / y[2], 1, 0, -f / y[2]]])


def reweighting(f, robust, b):
    """(w, W): w = sqrt(rho(r)) / r of pose_optimizer.h:224-231 and W = d(w f)/df."""
    r = max(EPS, np.linalg.norm(f))
    if not robust or r < b:
        return 1.0, np.eye(3)
    w = np.sqrt(2 * b * r - b * b) / r
    fh = f / r
    return w, w * (np.eye(3) - (r - b) / (2 * r - b) * np.outer(fh, fh))


def pose_grad(oracle, pid, obs, xyz, cam, T, g, lam=0.0, robust=True, b=1.0, hold_w=False):
    """(dL_dobs [n,3], dL_dxyz [npoints,3], dL_dcam [4], v) at the pose T for dL/d delta = g.  hold_w: W = w I (the
    reweighting held fixed), which the tests show to be wrong."""
    R, t = rot(T[:4]), T[4:]
    lin = []
    H = lam * np.eye(6)
    for i in range(len(pid)):
        X = xyz[pid[i]]
        f = obs[i] - oracle.pose_map(cam, T, X)
        J = oracle.pose_frame_jac(cam, T, X)
        w, W = reweighting(f, robust, b)
        if hold_w:
            W = w * np.eye(3)
        H += J.T @ W @ J
        lin.append((J, W, R @ X + t))
    v = np.linalg.solve(H, g)
    dobs, dxyz, dcam = np.zeros((len(pid), 3)), np.zeros((len(xyz), 3)), np.zeros(4)
    for i, (J, W, y) in enumerate(lin):
        u = W @ J @ v
        dobs[i] = -u
        dxyz[pid[i]] += R.T @ dpi_dy(cam, y).T @ u
        dcam += dpi_dcam(cam, y).T @ u
    return dobs, dxyz, dcam, v


# ---------------------------------------------------------------- the root of F, for central differences
def project(cam, T, X):
    """oracle.pose_map for every row of X [n,3] (opo_map's operation order)."""
    f, px, py, b = cam
    y = X @ rot(T[:4]).T + T[4:]
    return np.stack([f * (y[:, 0] / y[:, 2]) + px, f * (y[:, 1] / y[:, 2]) + py, (y[:, 0] - b) / y[:, 2] * f + px], 1), y


def frame_jac(cam, y):
    """oracle.pose_frame_jac for every row of y [n,3] (the point in the camera): [n,3,6]."""
    f, b = cam[0], cam[3]
    x, yy, z = y[:, 0], y[:, 1], y[:, 2]
    A = -f / z
    C, D, E = f * x / z ** 2, f * yy / z ** 2, f * (x - b) / z ** 2
    zero = np.zeros_like(x)
    return np.stack([np.stack([A, zero, C, yy * C, z * A - x * C, -yy * A], 1),
                     np.stack([zero, A, D, -z * A + yy * D, -x * D, x * A], 1),
                     np.stack([A, zero, E, yy * E, z * A - x * E, -yy * A], 1)], 1)


def root(oracle, pid, obs, xyz, cam, T, robust=True, b=1.0, max_iter=60):
    """The root of F(T) = sum_i J_i^T w_i f_i by undamped iteration of the LM's normal equations (A = sum J^T J,
    B = -sum J^T w f, T <- exp(A^-1 B) T), from T until the step is below 1e-15 or stops shrinking."""
    cam = np.asarray(cam, np.float64)
    T = np.array(T, np.float64)
    last = np.inf
    for _ in range(max_iter):
        m, y = project(cam, T, xyz[pid])
        f = obs - m
        if robust:
            r = np.maximum(EPS, np.linalg.norm(f, axis=1))
            rho = np.where(r < b, r * r, 2 * b * r - b * b)
            f = f * (np.sqrt(rho) / r)[:, None]
        J = frame_jac(cam, y)
        A = np.einsum("nki,nkj->ij", J, J)
        B = -np.einsum("nki,nk->i", J, f)
        d = np.linalg.solve(A, B)
        T = oracle.se3_mul(oracle.se3_exp(d), T)
        step = np.abs(d).max()
        if step < 1e-15 or step >= last:
            break
        last = step
    return T


def tangent(oracle, T, T0):
    """delta with T = exp(delta) T0."""
    return oracle.se3_log(oracle.se3_mul(T, oracle.se3_inv(T0)))
