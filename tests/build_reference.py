"""Long-double reference of the Schur build (k_build_wave, k_build, k_build_long) and of one Levenberg step, a window
builder that emits exactly the tracks it is asked for, and a restatement of the rules that route a landmark to one of
the three build kernels.

Reduced system.  Per edge, Jpsi, Jp, Ja and the error come from oracle.edge_jacobians / oracle.edge_error (float64);
everything after that is accumulated in np.longdouble: Hll, b_l, the pose blocks and gradients of the direct J^T W J
terms, the Hpl block of every (landmark, pose) slot, (Hll + lambda I)^-1 by 3x3 cofactors, the Schur products and the
pose-pose constraint terms (oracle.posepose_*).  The Jacobians of fixed poses are zero and a fixed pose's diagonal gets
+1, as the oracle's sys_schur does.  A self edge (the anchor observing its own point) adds Jp^T W Jp + Ja^T W Ja +
Jp^T W Ja to the anchor's diagonal block, g2o's term B5 that the oracle's build_landmark reproduces; with skip_self
(SVS_BA_SKIP_SELF_ANCHOR_HESSIAN) its pose columns are summed into one, (Jp + Ja)^T W (Jp + Ja), which is what
ba_grad_reference.gauss_newton does.  Diagonal blocks are read from their upper triangle, as g2o reads them.

Every pose block of S and every 6-vector of bs has a magnitude companion M: the same sums with every term replaced by
its absolute value, |Hpp| + lambda + sum |Y_a| |B_b|^T.  A rounding error of the build is a small multiple of eps * M
in the block it lands in, so bars taken per block against M do not let a wrong small block hide behind a large one.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from scavislam_b200 import synth

LD = np.longdouble


# ------------------------------------------------------------------------------------------------ window builder

@dataclass(frozen=True)
class Track:
    """`count` landmarks anchored in frame `anchor`, observed by the frames `observers` (the anchor not among them)
    and, when `self_edge`, by the anchor itself."""
    anchor: int
    observers: tuple
    self_edge: bool
    count: int = 1


def make_tracks_window(P, tracks, seed=0, fixed=(), C=0, unobserved=0, obs_sigma=0.5, outlier_frac=0.05,
                       step=0.03, lam_scale=1.0):
    """A window of P keyframes on a camera that moves slowly forward (`step` metres per frame, a small yaw wobble), so
    that a point 6-12 m in front of its anchor stays in view with positive depth and disparity over 100 frames.
    Observations get Gaussian noise of `obs_sigma` pixels and `outlier_frac` of them an outlier of up to 15 px, so
    that Huber's kernel takes both branches.  `unobserved` landmarks without edges are interleaved with the others.
    C pose-pose constraints join frames 1-3 apart (both orders, repeated when C asks for more).  The edges of a
    landmark are listed by ascending frame."""
    rng = np.random.default_rng(seed)
    f, px, py, b = synth.CAM_F, synth.CAM_PX, synth.CAM_PY, synth.CAM_B
    cam = np.array([f, px, py, b])
    i = np.arange(P)
    yaw = 0.004 * np.sin(i / 5.0)
    R_wc = np.zeros((P, 3, 3))
    R_wc[:, 0, 0] = np.cos(yaw); R_wc[:, 0, 2] = np.sin(yaw); R_wc[:, 1, 1] = 1
    R_wc[:, 2, 0] = -np.sin(yaw); R_wc[:, 2, 2] = np.cos(yaw)
    pos = np.stack([0.02 * np.sin(i / 7.0), 0.01 * np.cos(i / 9.0), step * i], -1)
    R_cw = np.transpose(R_wc, (0, 2, 1))
    t_cw = -(R_cw @ pos[..., None])[..., 0]
    truth = synth._to_qt(R_cw, t_cw)

    psi_t, ep, eq, ea, eo = [], [], [], [], []
    for tr in tracks:
        obs_frames = sorted(set(int(o) for o in tr.observers))
        assert tr.anchor not in obs_frames and len(obs_frames) == len(tr.observers)
        frames = sorted(obs_frames + ([tr.anchor] if tr.self_edge else []))
        assert frames, "a track needs at least one edge"
        for _ in range(tr.count):
            u, v, z = px + rng.uniform(-80, 80), py + rng.uniform(-60, 60), rng.uniform(6.0, 12.0)
            xa = np.array([(u - px) / f * z, (v - py) / f * z, z])
            xw = R_wc[tr.anchor] @ xa + pos[tr.anchor]
            l = len(psi_t)
            psi_t.append([xa[0] / z, xa[1] / z, 1.0 / z])
            for j in frames:
                y = R_cw[j] @ xw + t_cw[j]
                uu, vv, ur = f * y[0] / y[2] + px, f * y[1] / y[2] + py, f * (y[0] - b) / y[2] + px
                if not (y[2] > 0.3 and 0 <= uu < synth.CAM_W and 0 <= vv < synth.CAM_H and uu - ur > 0):
                    raise ValueError(f"frame {j} does not see the point of anchor {tr.anchor}")
                ep.append(l); eq.append(j); ea.append(tr.anchor); eo.append([uu, vv, ur])
    L0, E = len(psi_t), len(ep)
    e_obs = np.asarray(eo, np.float64).reshape(E, 3) + rng.normal(0, obs_sigma, (E, 3))
    outl = rng.uniform(size=E) < outlier_frac
    e_obs[outl] += rng.uniform(-15, 15, (int(outl.sum()), 3))
    s = np.where(rng.uniform(size=E) < 0.25, 0.25, 1.0)
    e_info = np.stack([s, s, np.full(E, 0.333 ** 2)], -1)
    psi_t = np.asarray(psi_t, np.float64).reshape(L0, 3)
    psi0 = psi_t.copy()
    psi0[:, 2] *= 1 + rng.normal(0, 0.03, L0)

    # interleave the unobserved landmarks: they take evenly spaced labels
    L = L0 + unobserved
    lab_un = np.unique(np.linspace(0, L - 1, unobserved).round().astype(np.int64)) if unobserved else np.zeros(0, np.int64)
    assert len(lab_un) == unobserved
    lab_obs = np.setdiff1d(np.arange(L), lab_un)
    psi = np.zeros((L, 3)); psi_truth = np.zeros((L, 3))
    psi[lab_obs], psi_truth[lab_obs] = psi0, psi_t
    un = np.stack([rng.uniform(-.1, .1, unobserved), rng.uniform(-.1, .1, unobserved), rng.uniform(.08, .16, unobserved)], 1)
    psi[lab_un], psi_truth[lab_un] = un, un

    from oracle import pyoracle as po
    pose_qt = np.array([po.se3_mul(po.se3_exp(np.concatenate([rng.normal(0, 0.01, 3), rng.normal(0, 0.002, 3)])), truth[k])
                        for k in range(P)]).reshape(P, 7)
    ci, cj, cT, cL = [], [], [], []
    pairs = [(a, a + d) for d in (1, 2, 3) for a in range(P - d)]
    for c in range(C):
        a, bb = pairs[(c // 2) % len(pairs)]
        if c % 2:
            a, bb = bb, a
        T = po.se3_mul(po.se3_exp(rng.normal(0, 1e-3, 6)), po.se3_mul(truth[bb], po.se3_inv(truth[a])))
        ci.append(a); cj.append(bb); cT.append(T)
        cL.append((lam_scale * np.diag([4e4] * 3 + [1e5] * 3)).reshape(36))
    fx = np.zeros(P, np.uint8)
    fx[list(fixed)] = 1
    return synth.BAProblem(
        P=P, L=L, E=E, C=C, pose_qt=pose_qt, fixed=fx, psi=np.ascontiguousarray(psi),
        e_point=lab_obs[np.asarray(ep, np.int64)].astype(np.int32), e_pose=np.asarray(eq, np.int32),
        e_anchor=np.asarray(ea, np.int32), e_obs=np.ascontiguousarray(e_obs), e_info=np.ascontiguousarray(e_info),
        c_i=np.asarray(ci, np.int32), c_j=np.asarray(cj, np.int32), c_T=np.asarray(cT, np.float64).reshape(C, 7),
        c_Lambda=np.asarray(cL, np.float64).reshape(C, 36), cam=cam, truth_pose_qt=truth, truth_psi=psi_truth,
        name="tracks")


def tracks_of(pb):
    """The multiset of (anchor, observers, self edge) of a window's observed landmarks, and its unobserved count."""
    out = {}
    for l in range(pb.L):
        m = pb.e_point == l
        if not m.any():
            continue
        a = int(pb.e_anchor[m][0])
        assert (pb.e_anchor[m] == a).all()
        poses = sorted(int(p) for p in pb.e_pose[m])
        key = (a, tuple(p for p in poses if p != a), a in poses)
        out[key] = out.get(key, 0) + 1
    return out, pb.L - len(np.unique(pb.e_point))


# ------------------------------------------------------------------------------------------------ reduced system

def _huber_w(e2, robust, delta):
    if not robust:
        return np.ones_like(e2), e2.copy()
    big = e2 > delta * delta
    sq = np.sqrt(np.where(big, e2, 1.0))
    return np.where(big, delta / sq, 1.0), np.where(big, 2 * sq * delta - delta * delta, e2)


def _blocks(H, rows, cols, blk):
    """H[6 rows + r, 6 cols + c] += blk[..., r, c] (rows / cols broadcast against blk's leading axes)."""
    r = 6 * np.asarray(rows)[..., None, None] + np.arange(6)[:, None]
    c = 6 * np.asarray(cols)[..., None, None] + np.arange(6)[None, :]
    np.add.at(H, (r, c), blk)


def _inv3(A):
    """Batched 3x3 inverse by cofactors, in the dtype of A."""
    c00 = A[:, 1, 1] * A[:, 2, 2] - A[:, 1, 2] * A[:, 2, 1]
    c01 = A[:, 1, 2] * A[:, 2, 0] - A[:, 1, 0] * A[:, 2, 2]
    c02 = A[:, 1, 0] * A[:, 2, 1] - A[:, 1, 1] * A[:, 2, 0]
    det = A[:, 0, 0] * c00 + A[:, 0, 1] * c01 + A[:, 0, 2] * c02
    Ai = np.empty_like(A)
    Ai[:, 0, 0] = c00; Ai[:, 1, 0] = c01; Ai[:, 2, 0] = c02
    Ai[:, 0, 1] = A[:, 0, 2] * A[:, 2, 1] - A[:, 0, 1] * A[:, 2, 2]
    Ai[:, 1, 1] = A[:, 0, 0] * A[:, 2, 2] - A[:, 0, 2] * A[:, 2, 0]
    Ai[:, 2, 1] = A[:, 0, 1] * A[:, 2, 0] - A[:, 0, 0] * A[:, 2, 1]
    Ai[:, 0, 2] = A[:, 0, 1] * A[:, 1, 2] - A[:, 0, 2] * A[:, 1, 1]
    Ai[:, 1, 2] = A[:, 0, 2] * A[:, 1, 0] - A[:, 0, 0] * A[:, 1, 2]
    Ai[:, 2, 2] = A[:, 0, 0] * A[:, 1, 1] - A[:, 0, 1] * A[:, 1, 0]
    return Ai / det[:, None, None]


@dataclass
class Reduced:
    S: np.ndarray        # [6P, 6P] longdouble, diagonal blocks symmetric from their upper triangle
    M: np.ndarray        # magnitude companion of S
    bs: np.ndarray       # [6P] longdouble
    Mb: np.ndarray       # magnitude companion of bs
    chi2: LD
    Dinv: np.ndarray     # [L, 3, 3] (Hll + lambda I)^-1
    bl: np.ndarray       # [L, 3]
    W: np.ndarray        # [ns, 6, 3] Hpl block of every (landmark, pose) slot
    slot_l: np.ndarray
    slot_pose: np.ndarray
    has_edges: np.ndarray


def reduced_system(oracle, pb, robust=True, delta=1.0, lam=50.0, skip_self=False):
    P, L, E = pb.P, pb.L, pb.E
    cam = np.asarray(pb.cam, np.float64)
    ep, eq, ea = (np.asarray(x, np.int64) for x in (pb.e_point, pb.e_pose, pb.e_anchor))
    Jpsi, Jp, Ja, err = np.zeros((E, 3, 3)), np.zeros((E, 3, 6)), np.zeros((E, 3, 6)), np.zeros((E, 3))
    for e in range(E):
        Tp, Ta, psi = pb.pose_qt[eq[e]], pb.pose_qt[ea[e]], pb.psi[ep[e]]
        Jpsi[e], Jp[e], Ja[e] = oracle.edge_jacobians(cam, Tp, Ta, psi)
        err[e] = oracle.edge_error(cam, Tp, Ta, psi, pb.e_obs[e])
    fixed = np.asarray(pb.fixed, bool)
    Jp[fixed[eq]] = 0.0
    Ja[fixed[ea]] = 0.0
    om = np.asarray(pb.e_info, np.float64).astype(LD)
    err, Jpsi, Jp, Ja = err.astype(LD), Jpsi.astype(LD), Jp.astype(LD), Ja.astype(LD)
    e2 = np.sum(om * err * err, 1)
    r1, rho = _huber_w(e2, robust, LD(delta))
    w = r1[:, None] * om                       # rho' Omega
    we = -w * err                              # -rho' Omega e
    aw, awe = np.abs(w), np.abs(we)

    def AtWB(A, B, ww):
        return np.einsum("eki,ek,ekj->eij", A, ww, B)

    aJpsi, aJp, aJa = np.abs(Jpsi), np.abs(Jp), np.abs(Ja)
    Hll = np.zeros((L, 3, 3), LD); np.add.at(Hll, ep, AtWB(Jpsi, Jpsi, w))
    bl = np.zeros((L, 3), LD); np.add.at(bl, ep, np.einsum("eki,ek->ei", Jpsi, we))
    blm = np.zeros((L, 3), LD); np.add.at(blm, ep, np.einsum("eki,ek->ei", aJpsi, awe))
    n = 6 * P
    H, Hm = np.zeros((n, n), LD), np.zeros((n, n), LD)
    bp, bpm = np.zeros(n, LD), np.zeros(n, LD)
    six = np.arange(6)
    self_e = eq == ea
    o = ~self_e
    # observer edges
    _blocks(H, eq[o], eq[o], AtWB(Jp[o], Jp[o], w[o])); _blocks(Hm, eq[o], eq[o], AtWB(aJp[o], aJp[o], aw[o]))
    _blocks(H, ea[o], ea[o], AtWB(Ja[o], Ja[o], w[o])); _blocks(Hm, ea[o], ea[o], AtWB(aJa[o], aJa[o], aw[o]))
    X = AtWB(Ja[o], Jp[o], w[o]); Xm = AtWB(aJa[o], aJp[o], aw[o])
    _blocks(H, ea[o], eq[o], X); _blocks(H, eq[o], ea[o], np.swapaxes(X, 1, 2))
    _blocks(Hm, ea[o], eq[o], Xm); _blocks(Hm, eq[o], ea[o], np.swapaxes(Xm, 1, 2))
    for J, aJ, idx in ((Jp, aJp, eq), (Ja, aJa, ea)):
        np.add.at(bp, 6 * idx[o][:, None] + six, np.einsum("eki,ek->ei", J[o], we[o]))
        np.add.at(bpm, 6 * idx[o][:, None] + six, np.einsum("eki,ek->ei", aJ[o], awe[o]))
    # self edges: the pose columns coincide
    s = self_e
    Jc = Jp[s] + Ja[s]
    if skip_self:
        _blocks(H, ea[s], ea[s], AtWB(Jc, Jc, w[s]))
        _blocks(Hm, ea[s], ea[s], AtWB(np.abs(Jp[s]) + np.abs(Ja[s]), np.abs(Jp[s]) + np.abs(Ja[s]), aw[s]))
    else:
        _blocks(H, ea[s], ea[s], AtWB(Jp[s], Jp[s], w[s]) + AtWB(Ja[s], Ja[s], w[s]) + AtWB(Jp[s], Ja[s], w[s]))
        _blocks(Hm, ea[s], ea[s], AtWB(aJp[s], aJp[s], aw[s]) + AtWB(aJa[s], aJa[s], aw[s]) + AtWB(aJp[s], aJa[s], aw[s]))
    np.add.at(bp, 6 * ea[s][:, None] + six, np.einsum("eki,ek->ei", Jc, we[s]))
    np.add.at(bpm, 6 * ea[s][:, None] + six, np.einsum("eki,ek->ei", aJp[s] + aJa[s], awe[s]))

    # Hpl slots: one per (landmark, pose) pair
    keys = np.concatenate([ep * P + ea, ep * P + eq])
    uniq, inv = np.unique(keys, return_inverse=True)
    slot_l, slot_pose = uniq // P, uniq % P
    sa, sp = inv[:E], inv[E:]
    ns = len(uniq)
    W, Wm = np.zeros((ns, 6, 3), LD), np.zeros((ns, 6, 3), LD)
    np.add.at(W, sp[o], AtWB(Jp[o], Jpsi[o], w[o])); np.add.at(Wm, sp[o], AtWB(aJp[o], aJpsi[o], aw[o]))
    np.add.at(W, sa[o], AtWB(Ja[o], Jpsi[o], w[o])); np.add.at(Wm, sa[o], AtWB(aJa[o], aJpsi[o], aw[o]))
    np.add.at(W, sa[s], AtWB(Jc, Jpsi[s], w[s])); np.add.at(Wm, sa[s], AtWB(aJp[s] + aJa[s], aJpsi[s], aw[s]))

    # Schur complement, landmarks grouped by their slot count
    Dinv = _inv3(Hll + LD(lam) * np.eye(3, dtype=LD))
    Y = np.einsum("sij,sjk->sik", W, Dinv[slot_l])
    Ym = np.abs(Y)
    db = np.einsum("lij,lj->li", Dinv, bl)
    np.add.at(bp, 6 * slot_pose[:, None] + six, -np.einsum("sij,sj->si", W, db[slot_l]))
    np.add.at(bpm, 6 * slot_pose[:, None] + six, np.einsum("sij,sj->si", Ym, blm[slot_l]))
    cnt = np.bincount(slot_l, minlength=L)
    start = np.concatenate([[0], np.cumsum(cnt)])
    for K in np.unique(cnt[cnt > 0]):
        lms = np.nonzero(cnt == K)[0]
        per = max(1, 20000 // (K * K))
        for q in range(0, len(lms), per):
            idx = start[lms[q:q + per]][:, None] + np.arange(K)
            rows = slot_pose[idx]
            _blocks(H, rows[:, :, None], rows[:, None, :], -np.einsum("naij,nbkj->nabik", Y[idx], W[idx]))
            _blocks(Hm, rows[:, :, None], rows[:, None, :], np.einsum("naij,nbkj->nabik", Ym[idx], Wm[idx]))

    chi2 = np.sum(rho)
    for c in range(pb.C):
        i, j = int(pb.c_i[c]), int(pb.c_j[c])
        e6 = oracle.posepose_error(pb.c_T[c], pb.pose_qt[i], pb.pose_qt[j])
        Ji, Jj = oracle.posepose_jacobians(pb.c_T[c], e6)
        if fixed[i]:
            Ji = np.zeros((6, 6))
        if fixed[j]:
            Jj = np.zeros((6, 6))
        Lm = np.asarray(pb.c_Lambda[c], np.float64).reshape(6, 6).astype(LD)
        e6, Ji, Jj = e6.astype(LD), Ji.astype(LD), Jj.astype(LD)
        chi2 += e6 @ Lm @ e6
        Oe = -(Lm @ e6)
        for (qa, A), (qb, B) in (((i, Ji), (i, Ji)), ((j, Jj), (j, Jj)), ((i, Ji), (j, Jj)), ((j, Jj), (i, Ji))):
            H[6 * qa:6 * qa + 6, 6 * qb:6 * qb + 6] += A.T @ Lm @ B
            Hm[6 * qa:6 * qa + 6, 6 * qb:6 * qb + 6] += np.abs(A).T @ np.abs(Lm) @ np.abs(B)
        for q, A in ((i, Ji), (j, Jj)):
            bp[6 * q:6 * q + 6] += A.T @ Oe
            bpm[6 * q:6 * q + 6] += np.abs(A).T @ np.abs(Oe)
    for p in range(P):
        d = LD(lam) + (LD(1) if fixed[p] else LD(0))
        blk = H[6 * p:6 * p + 6, 6 * p:6 * p + 6]
        blk[:] = np.triu(blk) + np.triu(blk, 1).T
        blk[six, six] += d
        Hm[6 * p + six, 6 * p + six] += d
    return Reduced(H, Hm, bp, bpm, chi2, Dinv, bl, W, slot_l, slot_pose, cnt > 0)


def block_ratio(S, ref, P):
    """Worst over the 6x6 blocks of max|S - S_ref| / max M (a block with M = 0 must match exactly)."""
    d = np.abs(np.asarray(S, LD) - ref.S).reshape(P, 6, P, 6).max(axis=(1, 3))
    m = ref.M.reshape(P, 6, P, 6).max(axis=(1, 3))
    return _ratio(d, m)


def rhs_ratio(bs, ref, P):
    d = np.abs(np.asarray(bs, LD) - ref.bs).reshape(P, 6).max(1)
    return _ratio(d, ref.Mb.reshape(P, 6).max(1))


def _ratio(d, m):
    if np.any((m == 0) & (d != 0)):
        return float("inf")
    return float(np.max(np.where(m > 0, d / np.where(m > 0, m, 1), 0))) if d.size else 0.0


def back_substitute(ref, x):
    """dpsi = (Hll + lambda I)^-1 (b_l - sum_s B_s^T x_pose(s)) in long double for the pose step x [6P]."""
    x = np.asarray(x, LD).reshape(-1, 6)
    c = ref.bl.copy()
    np.add.at(c, ref.slot_l, -np.einsum("sij,si->sj", ref.W, x[ref.slot_pose]))
    dpsi = np.einsum("lij,lj->li", ref.Dinv, c)
    dpsi[~ref.has_edges] = 0
    return dpsi


def pose_step(ref):
    """x_p from S in float64 plus one refinement step with a long-double residual."""
    S64 = ref.S.astype(np.float64)
    x = np.linalg.solve(S64, ref.bs.astype(np.float64)).astype(LD)
    r = ref.bs - ref.S @ x
    return x + np.linalg.solve(S64, r.astype(np.float64)).astype(LD)


def apply_step(oracle, pb, x, dpsi):
    """The oracle's update: T <- exp(x_i) T for every free pose, psi <- psi + dpsi."""
    x = np.asarray(x, np.float64).reshape(-1, 6)
    poses = np.array([pb.pose_qt[i] if pb.fixed[i] else oracle.se3_mul(oracle.se3_exp(x[i]), pb.pose_qt[i])
                      for i in range(pb.P)]).reshape(pb.P, 7)
    return poses, pb.psi + np.asarray(dpsi, np.float64)


def one_step(oracle, pb, robust=True, delta=1.0, lam=50.0, skip_self=False):
    ref = reduced_system(oracle, pb, robust, delta, lam, skip_self)
    x = pose_step(ref)
    poses, psi = apply_step(oracle, pb, x, back_substitute(ref, x))
    return poses, psi, x, ref


def recovered_step(oracle, pose0, pose1, fixed):
    """x_i = log(T1 T0^-1): the pose step an update T1 = exp(x_i) T0 applied (0 for fixed poses)."""
    return np.concatenate([np.zeros(6) if fixed[i] else oracle.se3_log(oracle.se3_mul(pose1[i], oracle.se3_inv(pose0[i])))
                           for i in range(len(pose0))])


# ------------------------------------------------------------------------------------------------ route restatement

K_MAX_TRACK = 32      # slots k_build stages in shared memory; longer tracks go to k_build_long
WAVE_SLOTS = 40       # slots of one k_build_wave wave
WAVE_LMS = 8          # landmarks of one wave
MAX_WAVES = 64


def track_padding(m, lo, hi, anchor):
    if m < 2:
        return 0
    span = hi - lo + 1 - (1 if lo < anchor < hi else 0)
    np_ = span - m
    return np_ if (np_ > 0 and 1 + span <= 8 and np_ <= max(1, m // 2)) else 0


def locality_key(nself, K, first, last):
    return ((0 if nself else 1) << 61) | ((K & 0xfffff) << 40) | ((first & 0xfffff) << 20) | (last & 0xfffff)


def build_chunk(L, sms, env=None):
    chunk = min(32, max(4, L // (max(sms, 1) * 11)))
    if env is not None:
        chunk = max(1, int(env))
    return chunk


def nw_bounds(k, K):
    """(32 // k, 40 // K, 8): k_build_wave's landmarks per wave is their minimum."""
    return 32 // max(k, 1), WAVE_SLOTS // max(K, 1), WAVE_LMS


def nw_max(k, K):
    return min(nw_bounds(k, K))


def task_waves(k, K, cnt):
    nw = max(1, min(8, min(32 // max(k, 1), 40 // max(K, 1))))
    return min((cnt + nw - 1) // nw, MAX_WAVES)


@dataclass
class Route:
    order: list          # internal landmark order (user labels)
    k: list              # internal edges per internal landmark (with padding)
    K: list              # slots per internal landmark
    self_: list
    npad: list
    tasks: list          # (first internal landmark, count) in launch order
    gen: list            # internal landmarks of k_build
    long: list           # internal landmarks of k_build_long
    chunk: int

    def task_shape(self, t):
        li, cnt = self.tasks[t]
        return self.k[li], self.K[li], bool(self.self_[li]), cnt

    def launches_per_trial(self, C):
        return 2 + (1 if (self.tasks or C) else 0) + (1 if self.gen else 0) + (1 if self.long else 0)


def route(pb, sms, chunk_env=None, pad=True):
    """The host set-up's routing (set_problem_impl): per landmark its anchor, self flag, observers by pose and the
    padding of its track; the internal order (anchor bucket, then locality key, ties by label); runs of landmarks
    with identical slot lists capped at `chunk` for k_build_wave, more than 32 slots for k_build_long, the rest
    (9-32 slots, no edges) for k_build; wave tasks sorted by their cost in waves, longest first, stably."""
    P, L = pb.P, pb.L
    edges = [[] for _ in range(L)]
    for e in range(pb.E):
        edges[int(pb.e_point[e])].append(e)
    anchor, nself, K, npad, key, ipose = [-1] * L, [0] * L, [0] * L, [0] * L, [None] * L, [None] * L
    for l in range(L):
        es = edges[l]
        if not es:
            key[l] = (1 << 64) - 1
            ipose[l] = []
            continue
        a = int(pb.e_anchor[es[0]])
        obs = sorted(int(pb.e_pose[e]) for e in es if int(pb.e_pose[e]) != a)
        ns = len(es) - len(obs)
        Kl = 1 + len(obs)
        p = 0
        if pad and ns <= 1 and len(obs) >= 2:
            p = track_padding(len(obs), obs[0], obs[-1], a)
        anchor[l], nself[l], K[l], npad[l] = a, ns, Kl + p, p
        full = [q for q in range(obs[0], obs[-1] + 1) if q != a] if p else obs
        ipose[l] = ([a] if ns else []) + full
        first = obs[0] if obs else a
        last = obs[-1] if obs else a
        key[l] = locality_key(ns, K[l], first, last)
    order = sorted(range(L), key=lambda l: (P if anchor[l] < 0 else anchor[l], key[l], l))
    chunk = build_chunk(L, sms, chunk_env)
    ks = [len(ipose[l]) for l in order]
    Ks = [K[l] for l in order]
    tasks, gen, long_ = [], [], []
    for li, l in enumerate(order):
        kk, KK = ks[li], Ks[li]
        if kk > 0 and KK > K_MAX_TRACK:
            long_.append(li)
            continue
        if kk == 0 or KK > 8:
            gen.append(li)
            continue
        if tasks:
            t0, c0 = tasks[-1]
            lp = order[t0]
            if t0 + c0 == li and c0 < chunk and (anchor[lp], nself[lp], ipose[lp]) == (anchor[l], nself[l], ipose[l]):
                tasks[-1] = (t0, c0 + 1)
                continue
        tasks.append((li, 1))
    tasks.sort(key=lambda t: -task_waves(ks[t[0]], Ks[t[0]], t[1]))
    return Route(order, ks, Ks, [nself[l] for l in order], [npad[l] for l in order], tasks, gen, long_, chunk)


def persistent_threshold_tasks(sms, ctas_per_sm=2, warps=4):
    """k_build_wave runs a persistent grid when its task CTAs (4 tasks each) outnumber the resident CTAs: two per SM
    at 113 408 B of shared memory and 255 registers per thread."""
    return ctas_per_sm * sms * warps


def wave_smem_bytes():
    doubles = 2 * 32 * 19 + 32 * 9 + 32 * 3 + 2 * WAVE_SLOTS * 18 + WAVE_LMS * 56 + 32
    return 4 * (doubles * 8 + (8 + 40) * 4)
