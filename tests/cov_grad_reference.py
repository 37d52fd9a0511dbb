"""Long-double reference of the BA window's marginal covariances (svs_ba_covariance) and of its adjoint gradients
(svs_ba_observation_grad / svs_ba_window_grad), built on build_reference.reduced_system.

Inverse.  np.linalg has no long-double routines, so inverse_ld(S) takes the float64 inverse Z0, forms the residual
R = I - S Z0 once in long double and returns Z = Z0 + Z0 R; the residual I - S Z of the result is asserted to be at the
long-double level (a small multiple of n eps_ld max(|S| |Z|)).

Covariance, with Z = S^-1 of the reduced system at the call's lambda (a fixed pose's diagonal carries +1, its Hpl
blocks are zero, so Z restricted to the free poses is the inverse of their block):
  pose block p    Z_pp, zero for a fixed pose;
  pose pair i, j  Z_ij, zero when either pose is fixed;
  landmark l      D + D (sum_{a,b} W_a^T Z_ab W_b) D over the landmark's slots, D = (Hll + lambda I)^-1; zero for a
                  landmark without edges (whose D is 0/0 at lambda = 0).
Adjoint (reduced_system with skip_self: the gradient's H never holds the self-anchor term), for the upstream gradient
g = (g_p, g_l):
  x   = Z (g_p - sum_s W_s D g_l(s)), zero for fixed poses;   v_l = D (g_l - sum_a W_a^T x_a);
  per edge, with J = (Jpsi, Jp, Ja) from oracle.edge_jacobians (pose columns summed for a self edge, zero for a fixed
  pose), dL/dz = -rho' Omega (J v) and dL/domega = -rho' e (.) (J v), zero for a zero-weight edge;
  camera          sum_e (de_e/dcam)^T dL/dz_e with ba_window_grad_reference.camera_jacobian;
  constraint c    w = J_i x_i + J_j x_j, dL/dLambda_c = -(w e^T + e w^T) / 2, dL/d delta_c = -X^T Lambda_c w with
                  X = third(I, e_c) (ba_grad.cu's header).

Magnitude companions.  Every output block comes with the same sum taken over absolute values (|D| + |D| sum |W_a|^T
|Z_ab| |W_b| |D| for a landmark, |rho' Omega| (|Jpsi| m_v + |Jp| m_x + |Ja| m_x) for an edge, and so on down to
m_x = |Z| (|g_p| + sum |W| |D| |g_l|)).  A block of Z has no sum; its companion is the Cauchy-Schwarz bound
sqrt(Z_ii[r, r] Z_jj[c, c]) of each entry.  Bars per block against these companions keep a wrong small landmark, edge
or pose block from hiding behind a large one.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import ba_window_grad_reference as wref
import build_reference as br

LD = np.longdouble
EPS_LD = np.finfo(LD).eps
IDENTITY = wref.IDENTITY


def inverse_ld(S):
    """(Z, kappa): S^-1 in long double from the float64 inverse and one long-double residual correction, and
    kappa(S) = |S|_2 |Z|_2."""
    S = np.asarray(S, LD)
    n = len(S)
    Z0 = np.linalg.inv(S.astype(np.float64)).astype(LD)
    R = np.eye(n, dtype=LD) - S @ Z0
    Z = Z0 + Z0 @ R
    res = np.abs(np.eye(n, dtype=LD) - S @ Z).max()
    scale = (np.abs(S.astype(np.float64)) @ np.abs(Z.astype(np.float64))).max()
    assert res <= 16 * n * EPS_LD * scale, f"refined residual {float(res):.2e} of {scale:.2e}"
    kappa = float(np.linalg.norm(S.astype(np.float64), 2) * np.linalg.norm(Z.astype(np.float64), 2))
    return Z, kappa


def _zblocks(Z, P):
    return Z.reshape(P, 6, P, 6).transpose(0, 2, 1, 3)   # [i, j, 6, 6]


def slot_lists(ref, pb):
    """Per landmark the slot indices of ref.W in the device's order: the anchor's slot first, then the observers by
    ascending pose (the order in which k_ba_point_cov enumerates its a-major pairs)."""
    anchor = np.full(pb.L, -1, np.int64)
    anchor[np.asarray(pb.e_point, np.int64)] = np.asarray(pb.e_anchor, np.int64)
    cnt = np.bincount(ref.slot_l, minlength=pb.L)
    start = np.concatenate([[0], np.cumsum(cnt)])
    out = []
    for l in range(pb.L):
        s = np.arange(start[l], start[l + 1])
        out.append(np.concatenate([s[ref.slot_pose[s] == anchor[l]], s[ref.slot_pose[s] != anchor[l]]]))
    return out


# ------------------------------------------------------------------------------------------------ covariance

@dataclass
class Covariance:
    pose: np.ndarray       # [P, 6, 6]
    pose_m: np.ndarray
    pair: np.ndarray       # [n, 6, 6]  Cov(x_i, x_j) for pairs[k] = (i, j)
    pair_m: np.ndarray
    point: np.ndarray      # [L, 3, 3]
    point_m: np.ndarray
    kappa: float


def _cs(Zb, i, j):
    return np.sqrt(np.abs(np.diagonal(Zb[i, i]))[:, None] * np.abs(np.diagonal(Zb[j, j]))[None, :])


def landmark_blocks(ref, pb, Z, slots, pair_mult=None):
    """([L,3,3], companion [L,3,3]) of D + D M D.  pair_mult(l, K) -> [K, K] upper-triangular multiplicities of the
    pairs a <= b in `slots` order (None: each pair once) perturbs the sum for the sensitivity checks."""
    P, L = pb.P, pb.L
    Zb = _zblocks(Z, P)
    aZb = np.abs(Zb)
    out, outm = np.zeros((L, 3, 3), LD), np.zeros((L, 3, 3), LD)
    for l in range(L):
        if not ref.has_edges[l]:
            continue
        s = slots[l]
        K = len(s)
        W, q = ref.W[s], ref.slot_pose[s]
        Zl, aZl = Zb[q[:, None], q[None, :]], aZb[q[:, None], q[None, :]]
        C = np.einsum("aic,abij,bjd->abcd", W, Zl, W)        # C_ab = W_a^T Z_ab W_b
        Cm = np.einsum("aic,abij,bjd->abcd", np.abs(W), aZl, np.abs(W))
        if pair_mult is None:
            M, Mm = C.sum((0, 1)), Cm.sum((0, 1))
        else:
            m = np.asarray(pair_mult(l, K), LD)
            iu = np.triu(np.ones((K, K), bool), 1)
            up = (m * iu)[:, :, None, None]
            dg = np.diagonal(m)[:, None, None]
            M = (up * C).sum((0, 1)) + (up * np.swapaxes(C, 2, 3)).sum((0, 1)) + (dg * C[np.arange(K), np.arange(K)]).sum(0)
            Mm = Cm.sum((0, 1))
        D = ref.Dinv[l]
        out[l] = D + D @ M @ D
        outm[l] = np.abs(D) + np.abs(D) @ Mm @ np.abs(D)
    return out, outm


def covariance(ref, pb, pairs=(), Z=None, kappa=None):
    P = pb.P
    if Z is None:
        Z, kappa = inverse_ld(ref.S)
    Zb = _zblocks(Z, P)
    fixed = np.asarray(pb.fixed) != 0
    pose, pose_m = np.zeros((P, 6, 6), LD), np.zeros((P, 6, 6), LD)
    for p in range(P):
        if not fixed[p]:
            pose[p], pose_m[p] = Zb[p, p], _cs(Zb, p, p)
    n = len(pairs)
    pair, pair_m = np.zeros((n, 6, 6), LD), np.zeros((n, 6, 6), LD)
    for k, (i, j) in enumerate(pairs):
        if not (fixed[i] or fixed[j]):
            pair[k], pair_m[k] = Zb[i, j], _cs(Zb, i, j)
    point, point_m = landmark_blocks(ref, pb, Z, slot_lists(ref, pb))
    return Covariance(pose, pose_m, pair, pair_m, point, point_m, kappa)


# ------------------------------------------------------------------------------------------------ adjoint

@dataclass
class Gradient:
    obs: np.ndarray        # [E, 3]
    obs_m: np.ndarray
    info: np.ndarray
    info_m: np.ndarray
    cT: np.ndarray         # [C, 6]
    cT_m: np.ndarray
    cLambda: np.ndarray    # [C, 36]
    cLambda_m: np.ndarray
    cam: np.ndarray        # [4]
    cam_m: np.ndarray
    x: np.ndarray          # [P, 6] pose part of v
    v: np.ndarray          # [L, 3] landmark part of v
    kappa: float


def _edge_terms(oracle, pb, robust, delta):
    cam = np.asarray(pb.cam, np.float64)
    E = pb.E
    Jpsi, Jp, Ja, err = np.zeros((E, 3, 3)), np.zeros((E, 3, 6)), np.zeros((E, 3, 6)), np.zeros((E, 3))
    for e in range(E):
        Tp, Ta, psi = pb.pose_qt[pb.e_pose[e]], pb.pose_qt[pb.e_anchor[e]], pb.psi[pb.e_point[e]]
        Jpsi[e], Jp[e], Ja[e] = oracle.edge_jacobians(cam, Tp, Ta, psi)
        err[e] = oracle.edge_error(cam, Tp, Ta, psi, pb.e_obs[e])
    om = np.asarray(pb.e_info, np.float64).astype(LD)
    err = err.astype(LD)
    r1, _ = br._huber_w(np.sum(om * err * err, 1), robust, LD(delta))
    return Jpsi.astype(LD), Jp.astype(LD), Ja.astype(LD), err, om, r1


def adjoint(oracle, pb, g_pose=None, g_psi=None, robust=True, delta=1.0, lam=0.0, ref=None, Z=None, kappa=None,
            slot_keep=None, edge_keep=None):
    """Gradient of svs_ba_window_grad in long double.  slot_keep(l, K) -> [K] bool over the landmark's slots in the
    device's order and edge_keep(l, k) -> [k] bool over its edges in the device's order (the self edge, then the
    observers by ascending pose) perturb t_l and the per-edge
    outputs (a dropped edge reads 0) for the sensitivity checks."""
    P, L, E = pb.P, pb.L, pb.E
    if ref is None:
        ref = br.reduced_system(oracle, pb, robust, delta, lam, skip_self=True)
    if Z is None:
        Z, kappa = inverse_ld(ref.S)
    fixed = np.asarray(pb.fixed) != 0
    gp = np.zeros((P, 6), LD) if g_pose is None else np.asarray(g_pose, np.float64).reshape(P, 6).astype(LD)
    gp[fixed] = 0
    gl = np.zeros((L, 3), LD) if g_psi is None else np.asarray(g_psi, np.float64).reshape(L, 3).astype(LD)
    gl[~ref.has_edges] = 0
    D = ref.Dinv.copy()
    D[~ref.has_edges] = 0
    aD, aW = np.abs(D), np.abs(ref.W)
    # pose part
    u, um = np.einsum("lij,lj->li", D, gl), np.einsum("lij,lj->li", aD, np.abs(gl))
    b, bm = gp.copy(), np.abs(gp)
    np.add.at(b, ref.slot_pose, -np.einsum("sij,sj->si", ref.W, u[ref.slot_l]))
    np.add.at(bm, ref.slot_pose, np.einsum("sij,sj->si", aW, um[ref.slot_l]))
    x = (Z @ b.reshape(-1)).reshape(P, 6)
    xm = (np.abs(Z) @ bm.reshape(-1)).reshape(P, 6)
    x[fixed] = 0
    xm[fixed] = 0
    # landmark part
    keep = np.ones(len(ref.slot_l), bool)
    if slot_keep is not None:
        for l, s in enumerate(slot_lists(ref, pb)):
            if len(s):
                keep[s] = np.asarray(slot_keep(l, len(s)), bool)
    t, tm = np.zeros((L, 3), LD), np.zeros((L, 3), LD)
    np.add.at(t, ref.slot_l[keep], np.einsum("sij,si->sj", ref.W[keep], x[ref.slot_pose[keep]]))
    np.add.at(tm, ref.slot_l, np.einsum("sij,si->sj", aW, xm[ref.slot_pose]))
    v = np.einsum("lij,lj->li", D, gl - t)
    vm = np.einsum("lij,lj->li", aD, np.abs(gl) + tm)
    # edges
    Jpsi, Jp, Ja, err, om, r1 = _edge_terms(oracle, pb, robust, delta)
    ep, eq, ea = (np.asarray(a, np.int64) for a in (pb.e_point, pb.e_pose, pb.e_anchor))
    Jp[fixed[eq]] = 0
    Ja[fixed[ea]] = 0
    self_e = eq == ea
    Jp_, Ja_ = np.where(self_e[:, None, None], 0, Jp), np.where(self_e[:, None, None], Jp + Ja, Ja)
    jv = np.einsum("eij,ej->ei", Jpsi, v[ep]) + np.einsum("eij,ej->ei", Jp_, x[eq]) + np.einsum("eij,ej->ei", Ja_, x[ea])
    jvm = (np.einsum("eij,ej->ei", np.abs(Jpsi), vm[ep]) + np.einsum("eij,ej->ei", np.abs(Jp), xm[eq])
           + np.einsum("eij,ej->ei", np.abs(Ja), xm[ea]))
    w = r1[:, None] * om
    dobs, dobs_m = -w * jv, np.abs(w) * jvm
    dinfo, dinfo_m = -r1[:, None] * err * jv, np.abs(r1[:, None] * err) * jvm
    zero = ~np.asarray(pb.e_info, np.float64).any(1)
    if edge_keep is not None:
        for l in range(L):
            es = np.nonzero(ep == l)[0]
            if len(es):
                es = es[np.lexsort((eq[es], eq[es] != ea[es]))]   # the self edge first, then by pose
                zero[es[~np.asarray(edge_keep(l, len(es)), bool)]] = True
    for a in (dobs, dobs_m, dinfo, dinfo_m):
        a[zero] = 0
    dcam, dcam_m = np.zeros(4, LD), np.zeros(4, LD)
    for e in range(E):
        if zero[e]:
            continue
        Jc = wref.camera_jacobian(oracle, pb, e).astype(LD)
        dcam += Jc.T @ dobs[e]
        dcam_m += np.abs(Jc).T @ dobs_m[e]
    # pose-pose constraints
    C = pb.C
    dcT, dcT_m, dcL, dcL_m = (np.zeros((C, n), LD) for n in (6, 6, 36, 36))
    for c in range(C):
        i, j = int(pb.c_i[c]), int(pb.c_j[c])
        e6 = oracle.posepose_error(pb.c_T[c], pb.pose_qt[i], pb.pose_qt[j])
        Ji, Jj = (J.astype(LD) for J in oracle.posepose_jacobians(pb.c_T[c], e6))
        X = oracle.posepose_jacobians(IDENTITY, e6)[0].astype(LD)
        e6 = e6.astype(LD)
        Lm = np.asarray(pb.c_Lambda[c], np.float64).reshape(6, 6).astype(LD)
        wc, wm = np.zeros(6, LD), np.zeros(6, LD)
        for q, J in ((i, Ji), (j, Jj)):
            if not fixed[q]:
                wc += J @ x[q]
                wm += np.abs(J) @ xm[q]
        dcT[c], dcT_m[c] = -X.T @ Lm @ wc, np.abs(X).T @ np.abs(Lm) @ wm
        dcL[c] = (-0.5 * (np.outer(wc, e6) + np.outer(e6, wc))).reshape(36)
        dcL_m[c] = (0.5 * (np.outer(wm, np.abs(e6)) + np.outer(np.abs(e6), wm))).reshape(36)
    return Gradient(dobs, dobs_m, dinfo, dinfo_m, dcT, dcT_m, dcL, dcL_m, dcam, dcam_m, x, v, kappa)


# ------------------------------------------------------------------------------------------------ bars

def block_ratio(got, want, comp, axes):
    """Worst over the blocks (the leading axes) of max |got - want| / max companion over the block; a block with a zero
    companion must match exactly.  `axes`: the trailing axes that make up one block."""
    d = np.abs(np.asarray(got, LD) - np.asarray(want, LD))
    m = np.asarray(comp, LD)
    if d.size == 0:
        return 0.0
    return br._ratio(d.max(axis=axes), m.max(axis=axes))


BLOCK_BAR = 1e-10   # landmark blocks, per block against the companion
GRAD_BAR = 1e-11    # every gradient output, per block against the companion


def pose_bar(kappa):
    """Blocks of Z (pose blocks, pose pairs): 1e-10 where kappa(S) eps <= 1e-11, else 10 kappa(S) eps."""
    return max(BLOCK_BAR, 10 * kappa * np.finfo(np.float64).eps)


# ------------------------------------------------------------------------------------------------ shape windows

T = br.Track
H100_SMS = 132


def _chain(P, count=3):
    """Short tracks over every frame, so that every pose sees enough points to be determined."""
    return [T(a, (a + 1, a + 2), a % 2 == 0, count) for a in range(P - 2)]


def _with_zero_weight_edge(pb):
    """Zero the weight of the third edge of the first landmark with the most edges."""
    l = int(np.argmax(np.bincount(pb.e_point, minlength=pb.L)))
    pb.e_info = pb.e_info.copy()
    pb.e_info[np.nonzero(pb.e_point == l)[0][2]] = 0.0
    return pb


def _total(tracks):
    return sum(t.count for t in tracks)


def lanes8_window(rem):
    """k_ba_point_cov<8> / k_grad_edges<8>: slot counts K = 1 (self edge only), 2, 3 (6 pairs, fewer than the lanes),
    4 (10 pairs: the first wrap), 5, 7 and 8 (36 pairs; k = 8 with a self edge, k = 7 without), two tracks padded
    around an anchor inside their span, a zero-weight edge, unobserved landmarks, and L = rem mod 32."""
    P = 30
    tracks = [T(0, (), True, 2), T(1, (2,), True, 2), T(2, (3,), False, 2), T(3, (4, 5), True, 2), T(4, (5, 6), False, 2),
              T(5, (6, 7, 8), True, 2), T(6, (7, 8, 9), False, 2), T(7, tuple(range(8, 12)), True, 2),
              T(8, tuple(range(9, 15)), True, 2), T(9, tuple(range(10, 16)), False, 2),
              T(10, tuple(range(11, 18)), True, 2), T(11, tuple(range(12, 19)), False, 2),
              T(20, (18, 19, 21, 23), True, 2), T(24, (22, 23, 25, 27), False, 2)] + _chain(P)
    un = 3
    tracks.append(T(12, (13, 14), True, (rem - _total(tracks) - un) % 32 + 32))
    pb = br.make_tracks_window(P, tracks, seed=100 + rem, C=6, unobserved=un)
    return _with_zero_weight_edge(pb)


def check_lanes8(pb, rt, rem):
    shapes = {(rt.k[li], rt.K[li], bool(rt.self_[li])) for li in range(len(rt.order))}
    want = {(1, 1, True), (2, 2, True), (1, 2, False), (3, 3, True), (2, 3, False), (4, 4, True), (3, 4, False),
            (5, 5, True), (7, 7, True), (6, 7, False), (8, 8, True), (7, 8, False)}
    assert want <= shapes, want - shapes
    assert any(p > 0 for p in rt.npad), "no padded track"
    assert not rt.long and all(rt.k[li] == 0 for li in rt.gen), "every observed track fits 8 lanes"
    assert pb.L % 32 == rem, "L mod 32 (k_ba_point_cov<8> / k_grad_edges<8>: 32 landmarks per CTA)"
    assert (~np.asarray(pb.e_info).any(1)).sum() == 1


def warp_window(rem):
    """k_ba_point_cov<32> / k_grad_edges<32> over gen_lm (K = 9 with and without a self edge (k = 9, 8), 16, 17, 32
    with k = 32 and k = 31, landmarks without edges) and over long_lm (K = 33 with k = 32 and k = 33, 64, 65 and, for
    rem = 0, 97), ngen = nlong = rem mod 8.  Pose 6 anchors a long track and pose 40 observes another: the fixed poses
    of the lambda = 0 runs."""
    P = 100 if rem == 0 else 70
    gen = [T(0, tuple(range(1, 9)), True, 1), T(1, tuple(range(2, 10)), False, 1), T(2, tuple(range(3, 18)), True, 1),
           T(3, tuple(range(4, 20)), False, 1), T(4, tuple(range(5, 36)), True, 1), T(5, tuple(range(6, 37)), False, 1)]
    long_ = [T(6, tuple(range(7, 39)), False, 1), T(7, tuple(range(8, 40)), True, 1), T(2, tuple(range(3, 66)), True, 1),
             T(4, tuple(range(5, 69)), False, 1)]
    if P == 100:
        long_.append(T(0, tuple(range(1, 97)), True, 1))
    long_.append(T(10, tuple(range(11, 45)), True, (rem - len(long_)) % 8))
    un = (rem - len(gen)) % 8 or 8
    return br.make_tracks_window(P, gen + long_ + _chain(P), seed=200 + rem, C=8, unobserved=un)


WARP_FIXED = (6, 40)


def check_warps(pb, rt, rem):
    gen = {(rt.k[li], rt.K[li], bool(rt.self_[li])) for li in rt.gen}
    lng = {(rt.k[li], rt.K[li], bool(rt.self_[li])) for li in rt.long}
    assert {(9, 9, True), (8, 9, False), (16, 16, True), (16, 17, False), (32, 32, True), (31, 32, False),
            (0, 0, False)} <= gen, gen
    want = {(32, 33, False), (33, 33, True), (64, 64, True), (64, 65, False)} | ({(97, 97, True)} if rem == 0 else set())
    assert want <= lng, lng
    assert len(rt.gen) % 8 == rem and len(rt.long) % 8 == rem, "ngen, nlong mod 8 (8 warps per CTA)"
    by_anchor = {int(pb.e_anchor[pb.e_point == rt.order[li]][0]) for li in rt.long}
    assert WARP_FIXED[0] in by_anchor, "a long track anchored at the fixed pose"
    observed = {int(p) for li in rt.long for p in pb.e_pose[pb.e_point == rt.order[li]]
                if int(pb.e_anchor[pb.e_point == rt.order[li]][0]) != WARP_FIXED[1]}
    assert WARP_FIXED[1] in observed, "a long track observed by the fixed pose"


# (P, L, C, boundary): L + 6P one below / above a multiple of 256 ("rhs-" / "rhs+": k_grad_rhs, 256 threads per CTA),
# L < 256 or L = 256 m + 1 ("cam": k_grad_cam, one CTA of 256 threads); over the list C takes 0, 1, 255, 256 and 257
# (k_grad_constraints, 256 per CTA)
GRID = [(20, 135, 0, "rhs-"), (20, 137, 1, "rhs+"), (21, 257, 255, "cam"), (22, 379, 256, "rhs-"), (22, 381, 257, "rhs+"),
        (24, 513, 1, "cam")]


def grid_window(P, L, C):
    """Short tracks over P frames, three unobserved landmarks, L landmarks and C constraints, frames 0 and 1 fixed in
    the runs (constraints 0 and 1 join them both, 2 and 3 one of them)."""
    tracks = [T(a, (a + 1,) if a % 2 and a < P - 3 else (a + 1, a + 2), a % 3 != 0, 1) for a in range(P - 2)]
    chain = _chain(P, 1)
    n = L - 3 - len(tracks) - _total(chain)
    tracks = [T(t.anchor, t.observers, t.self_edge, 1 + n // len(tracks) + (1 if i < n % len(tracks) else 0))
              for i, t in enumerate(tracks)]
    return br.make_tracks_window(P, tracks + chain, seed=300 + L, C=C, unobserved=3)


def check_grid(pb, P, L, C, boundary):
    assert pb.P == P and pb.L == L and pb.C == C
    n = L + 6 * P
    if boundary == "cam":
        assert L % 256 == 1, "k_grad_cam: L one past a multiple of its CTA"
    else:
        assert n % 256 == (255 if boundary == "rhs-" else 1), "k_grad_rhs: L + 6P next to a multiple of 256"
    if C:
        assert {(int(pb.c_i[c]), int(pb.c_j[c])) for c in range(min(C, 4))} <= {(0, 1), (1, 0), (1, 2), (2, 1)}
