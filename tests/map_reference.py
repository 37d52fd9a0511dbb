"""Maps at back-end scale, vectorised restatements of the window selection and assembly, the launch rules of the map and
constraint kernels, and a long-double reference of computeConstraint.  TEST INFRASTRUCTURE ONLY.

The device map (scavislam_b200/csrc/graph.cu) and svs_computeConstraint_batch (csrc/constraint.cu) change their
launch at fixed sizes: k_scan walks its input in chunks of 1024 on one CTA and carries a running total between them,
k_bfs pushes into a queue of nnzN + 1 entries, and k_compute_constraint keeps a pair's distances in shared memory while
the smaller of the two feature tables holds <= 2048 points and in a global scratch row of max_feat doubles otherwise.
The generator below builds maps that reach those sizes; the restatements give the bit-exact answer the device must
give (same IEEE operations where a value is computed), fast enough at 10^4..10^6 observations where the plain-Python
restatements of oracle/pyoracle.py would take minutes.

Map tables are those of scavislam_b200.synth_graph.make_map: poses [V][7] (T_me_from_world, q = x y z w, t),
point_anchor [Np], xyz_anchor [Np][3], vis_ptr [Np+1], vis_pose [nnz] (ascending per point), feat_center [nnz][3],
feat_level [nnz]."""
from __future__ import annotations

import hashlib

import numpy as np

CAM = (500.0, 320.0, 240.0, 0.1)   # f, px, py, baseline

# ------------------------------------------------------------------ launch rules (graph.cu, constraint.cu)
SCAN_CHUNK = 1024          # k_scan<<<1, 1024>>>: one chunk of 1024 elements per pass, a running total between passes
SMEM_DEPTHS = 2048         # k_compute_constraint: kSmemDepths
CONSTRAINT_THREADS = 128   # k_compute_constraint: kThreads, the stride of its feature walk and of its rank count


def scan_chunks(n):
    """Passes k_scan makes over n elements (the carry is used from the second pass on)."""
    return -(-int(n) // SCAN_CHUNK)


def bfs_queue_capacity(nnzN):
    """k_bfs's queue: the root plus one entry per directed neighbour entry."""
    return int(nnzN) + 1


def constraint_route(feat_ptr, v1, v2):
    """(in_smem[npairs], scratch_stride) of svs_computeConstraint_batch: a pair's distances stay in shared memory when
    min(|F1|, |F2|) <= 2048; scratch rows are max_feat doubles apart when any table exceeds 2048, else there are none."""
    fp = np.asarray(feat_ptr, np.int64)
    size = np.diff(fp)
    v1, v2 = np.asarray(v1, np.int64), np.asarray(v2, np.int64)
    in_smem = np.minimum(size[v1], size[v2]) <= SMEM_DEPTHS
    max_feat = int(size.max()) if len(size) else 0
    return in_smem, (max_feat if max_feat > SMEM_DEPTHS else 0)


# ------------------------------------------------------------------ generator
def _rot_y(theta):
    c, s = np.cos(theta), np.sin(theta)
    R = np.zeros((len(theta), 3, 3))
    R[:, 0, 0] = c; R[:, 0, 2] = s; R[:, 1, 1] = 1.0; R[:, 2, 0] = -s; R[:, 2, 2] = c
    return R


def _quat_y(theta):
    q = np.zeros((len(theta), 4))
    q[:, 1] = np.sin(theta / 2); q[:, 3] = np.cos(theta / 2)
    return q


def make_map(V, per_kf, track_len=(2, 8), long_tracks=0.0, unobserved=0.0, levels=(0, 3), seed=0, obs_sigma=0.5,
             pose_sigma=1e-3):
    """Keyframes along a trajectory (camera k at x = 0.05 k, turning about y by 1 mrad per keyframe); keyframe k starts
    `per_kf` points, each seen by a run of consecutive keyframes from k on and anchored there.  A track has
    track_len[0]..track_len[1] observers, a `long_tracks` share has 33..40; an `unobserved` share has none.  Pyramid
    levels are uniform in levels[0]..levels[1] (0..30).  Observations are stereo projections with `obs_sigma` px of
    noise; poses and anchored positions carry a small error, so an optimiser has something to do."""
    rng = np.random.default_rng(seed)
    th = 1e-3 * np.arange(V)
    Rcw = _rot_y(th)                                          # camera-to-world rotation of keyframe k
    c = np.stack([0.05 * np.arange(V), 0.01 * np.sin(0.1 * np.arange(V)), np.zeros(V)], 1)
    qwc = _quat_y(-th)                                        # T_me_from_world: R = Rcw^T, t = -Rcw^T c
    t_me = -np.einsum("kji,kj->ki", Rcw, c)
    Np = V * per_kf
    k0 = np.repeat(np.arange(V), per_kf)
    n_obs = rng.integers(track_len[0], track_len[1] + 1, Np)
    if long_tracks:
        lt = rng.random(Np) < long_tracks
        n_obs[lt] = rng.integers(33, 41, int(lt.sum()))
    if unobserved:
        n_obs[rng.random(Np) < unobserved] = 0
    n_obs = np.minimum(n_obs, V - k0)
    local = np.stack([rng.uniform(-2, 2, Np), rng.uniform(-1.5, 1.5, Np), rng.uniform(4, 12, Np)], 1)
    X = c[k0] + np.einsum("pij,pj->pi", Rcw[k0], local)        # world position
    vis_ptr = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int32)
    nnz = int(vis_ptr[-1])
    pt = np.repeat(np.arange(Np), n_obs)
    vis_pose = (k0[pt] + np.arange(nnz) - vis_ptr[pt]).astype(np.int32)
    xf = np.einsum("pji,pj->pi", Rcw[vis_pose], X[pt] - c[vis_pose])   # the point in the observer's frame
    f, px, py, b = CAM
    u = f * xf[:, 0] / xf[:, 2] + px
    center = np.stack([u, f * xf[:, 1] / xf[:, 2] + py, u - f * b / xf[:, 2]], 1) + rng.normal(0, obs_sigma, (nnz, 3))
    level = rng.integers(levels[0], levels[1] + 1, nnz).astype(np.int32)
    dq = rng.normal(0, pose_sigma, (V, 4)); dq[:, 3] = 0
    q = qwc + dq
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    poses = np.concatenate([q, t_me + rng.normal(0, 10 * pose_sigma, (V, 3))], 1)
    xyz = local * (1 + rng.normal(0, 1e-3, (Np, 1)))
    return dict(poses=poses, point_anchor=k0.astype(np.int32), xyz_anchor=xyz, vis_ptr=vis_ptr, vis_pose=vis_pose,
                feat_center=center, feat_level=level)


def map_digest(m):
    h = hashlib.sha256()
    for k in ("poses", "point_anchor", "xyz_anchor", "vis_ptr", "vis_pose", "feat_center", "feat_level"):
        h.update(np.ascontiguousarray(m[k]).tobytes())
    return h.hexdigest()


def _graph_from_lists(nbrs):
    ptr = np.concatenate([[0], np.cumsum([len(x) for x in nbrs])]).astype(np.int32)
    ids = np.concatenate([np.asarray(x, np.int64) for x in nbrs]).astype(np.int32) if len(nbrs) else np.zeros(0, np.int32)
    return ptr, ids


def _with_constraints(ptr, ids, rng):
    n = len(ids)
    q = rng.normal(0, 1, (n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    T = np.concatenate([q, rng.normal(0, 1, (n, 3))], 1)
    A = rng.normal(0, 1, (n, 6, 6))
    return ptr, ids, T, (A @ A.transpose(0, 2, 1) + 6 * np.eye(6)).reshape(n, 36)


def covisibility_graph(m, max_neighbours=6, hubs=(), hub_degree=300, seed=0, with_constraints=True):
    """The pose graph of synth_graph.make_pose_graph, vectorised for maps whose tracks are runs of consecutive
    keyframes: two frames are neighbours when they share points, one neighbour per strength value (the largest id of
    that strength), the `max_neighbours` strongest kept, lists strongest first (ties by id).  A hub vertex in `hubs`
    additionally lists about `hub_degree` vertices spread over the map (appended, weakest), and they list it.  Returns
    (nbr_ptr, nbr_id, nbr_T, nbr_Lambda); the last two are None without constraints."""
    V = len(m["poses"])
    vp = np.asarray(m["vis_ptr"], np.int64)
    n = np.diff(vp)
    obs = n > 0
    s = np.asarray(m["vis_pose"], np.int64)[vp[:-1][obs]]
    e = np.asarray(m["vis_pose"], np.int64)[vp[1:][obs] - 1]
    assert np.all(e - s == n[obs] - 1), "tracks must be runs of consecutive keyframes"
    dmax = int((e - s).max()) if len(s) else 0
    S = np.zeros((V, dmax + 1), np.int64)                     # S[a, d] = strength of (a, a + d)
    for d in range(1, dmax + 1):
        ok = e - d >= s
        diff = np.bincount(s[ok], minlength=V + 1) - np.bincount(e[ok] - d + 1, minlength=V + 1)
        S[:, d] = np.cumsum(diff)[:V]
    keep = set()
    for v in range(V):
        d = np.arange(1, dmax + 1)
        up, dn = v + d, v - d
        cb = np.concatenate([up[up < V], dn[dn >= 0]])
        cs = np.concatenate([S[v, d[up < V]], S[dn[dn >= 0], d[dn >= 0]]])
        cb, cs = cb[cs > 0], cs[cs > 0]
        by_strength = {}
        for b_, s_ in sorted(zip(cb.tolist(), cs.tolist())):
            by_strength[s_] = b_
        for s_ in sorted(by_strength, reverse=True)[:max_neighbours]:
            b_ = by_strength[s_]
            keep.add((min(v, b_), max(v, b_)))
    nb = [[] for _ in range(V)]
    for a, b_ in keep:
        st = S[a, b_ - a]
        nb[a].append((-st, b_)); nb[b_].append((-st, a))
    nbrs = [[b_ for _, b_ in sorted(x)] for x in nb]
    for h in hubs:                                            # spread over the ids: 0 and V - 1 first, then shuffled
        spread = np.linspace(0, V - 1, hub_degree + 2).round().astype(int)
        for b_ in [0, V - 1] + np.random.default_rng(h).permutation(spread[1:-1]).tolist():
            if b_ != h and b_ not in nbrs[h]:
                nbrs[h].append(b_); nbrs[b_].append(h)
    ptr, ids = _graph_from_lists(nbrs)
    if not with_constraints:
        return ptr, ids, None, None
    return _with_constraints(ptr, ids, np.random.default_rng(seed))


def complete_graph(V, seed=0, with_constraints=True):
    """Every vertex lists every other, nearest id first."""
    nbrs = [sorted((b for b in range(V) if b != v), key=lambda b: (abs(b - v), b)) for v in range(V)]
    ptr, ids = _graph_from_lists(nbrs)
    return _with_constraints(ptr, ids, np.random.default_rng(seed)) if with_constraints else (ptr, ids, None, None)


def chain_graph(V, seed=0, with_constraints=True):
    """v lists v - 1 and v + 1."""
    nbrs = [[b for b in (v - 1, v + 1) if 0 <= b < V] for v in range(V)]
    ptr, ids = _graph_from_lists(nbrs)
    return _with_constraints(ptr, ids, np.random.default_rng(seed)) if with_constraints else (ptr, ids, None, None)


def cut_graph(graph, piece):
    """The graph without the entries between the vertices of `piece` and the rest: a disconnected piece; a single
    vertex is an isolated root.  T and Lambda follow their entries."""
    ptr, ids, T, Lm = graph
    V = len(ptr) - 1
    inside = np.zeros(V, bool); inside[np.asarray(list(piece), np.int64)] = True
    src = np.repeat(np.arange(V), np.diff(ptr))
    keep = inside[src] == inside[ids]
    ptr2 = np.concatenate([[0], np.cumsum(np.bincount(src[keep], minlength=V))]).astype(np.int32)
    return ptr2, ids[keep], None if T is None else T[keep], None if Lm is None else Lm[keep]


# ------------------------------------------------------------------ restatements (vectorised)
def copy_data_to_g2o(m, window_vertex, active_point):
    """oracle.pyoracle.copy_data_to_g2o without the Python loop: the same edges in the same order (active points in the
    caller's order, observations in vis_set order), the same values bit for bit."""
    V = len(m["poses"])
    win = np.full(V, -1, np.int64)
    win[np.asarray(window_vertex, np.int64)] = np.arange(len(window_vertex))
    act = np.asarray(active_point, np.int64)
    vp = np.asarray(m["vis_ptr"], np.int64)
    n = vp[act + 1] - vp[act]
    l = np.repeat(np.arange(len(act)), n)
    i = vp[act][l] + np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    w = win[np.asarray(m["vis_pose"], np.int64)[i]]
    keep = w >= 0
    l, i, w = l[keep], i[keep], w[keep]
    x = np.asarray(m["xyz_anchor"], np.float64)[act].reshape(-1, 3)
    psi = np.stack([x[:, 0] / x[:, 2], x[:, 1] / x[:, 2], 1.0 / x[:, 2]], 1)
    f = 1.0 / np.left_shift(1, np.asarray(m["feat_level"], np.int64)[i]).astype(np.float64)
    s = f * f
    info = np.stack([s, s, np.full(len(s), 0.333 * 0.333)], 1)
    return dict(pose_qt=np.asarray(m["poses"], np.float64)[np.asarray(window_vertex, np.int64)].reshape(-1, 7),
                psi=psi.reshape(-1, 3), e_point=l.astype(np.int32), e_pose=w.astype(np.int32),
                e_anchor=win[np.asarray(m["point_anchor"], np.int64)[act]][l].astype(np.int32),
                e_obs=np.asarray(m["feat_center"], np.float64)[i].reshape(-1, 3), e_info=info.reshape(-1, 3))


def compute_double_window(nbr_ptr, nbr_id, root, inner_window_size, double_window_size):
    """computeInitialDoubleWin as k_bfs walks it (one queue, at most nnzN + 1 pushes).  Returns ({vertex: 1 | 2},
    number of queue entries pushed)."""
    ptr, ids = np.asarray(nbr_ptr).tolist(), np.asarray(nbr_id).tolist()
    cap = bfs_queue_capacity(len(ids))
    q = [int(root)]
    head, win = 0, {}
    while len(win) < double_window_size and head < len(q):
        v = q[head]; head += 1
        if v in win:
            continue
        win[v] = 1 if len(win) < inner_window_size else 2
        room = cap - len(q)
        q.extend(ids[ptr[v]:ptr[v + 1]][:max(room, 0)])
    return win, len(q)


def _window_types(V, win):
    t = np.zeros(V, np.int64)
    for v, k in win.items():
        t[v] = k
    return t


def compute_active_points(m, nbr_ptr, nbr_id, win):
    """computeActivePointsAndExtendOuterWindow over all observations at once: a point is active when an INNER frame
    sees it and its anchor is in the window, or that frame has an edge (either direction) to the anchor, which then
    joins the outer window.  Returns (sorted active ids, window dict with the extension, extended anchors {a: number of
    points that extend it})."""
    V = len(m["poses"])
    t = _window_types(V, win)
    ptr = np.asarray(nbr_ptr, np.int64)
    src = np.repeat(np.arange(V), np.diff(ptr))
    dst = np.asarray(nbr_id, np.int64)
    keys = np.unique(np.concatenate([src * V + dst, dst * V + src]))
    vp = np.asarray(m["vis_ptr"], np.int64)
    p = np.repeat(np.arange(len(vp) - 1), np.diff(vp))
    f = np.asarray(m["vis_pose"], np.int64)
    a = np.asarray(m["point_anchor"], np.int64)[p]
    inner = t[f] == 1
    k = f * V + a
    pos = np.minimum(np.searchsorted(keys, k), max(len(keys) - 1, 0))
    edge = (keys[pos] == k) if len(keys) else np.zeros(len(k), bool)
    inwin = t[a] != 0
    act_obs = inner & (inwin | edge)
    ext_obs = inner & ~inwin & edge
    active = np.unique(p[act_obs])
    ext_pts = np.unique(np.stack([p[ext_obs], a[ext_obs]], 1), axis=0) if ext_obs.any() else np.zeros((0, 2), np.int64)
    ea, ecount = np.unique(ext_pts[:, 1], return_counts=True)
    out = dict(win)
    out.update({int(x): 2 for x in ea})
    return active.astype(np.int32), out, dict(zip(ea.tolist(), ecount.tolist()))


def select_constraints(nbr_ptr, nbr_id, nbr_T, nbr_Lambda, win):
    """The pair loop of copyContraintsToG2o over the directed entries: (a, b) with b != a, both in the window, one of
    them OUTER, in ascending (a, b) order; identity T and zero Lambda when the graph carries none."""
    ptr = np.asarray(nbr_ptr, np.int64)
    V = len(ptr) - 1
    t = _window_types(V, win)
    src = np.repeat(np.arange(V), np.diff(ptr))
    dst = np.asarray(nbr_id, np.int64)
    sel = (dst != src) & (t[src] != 0) & (t[dst] != 0) & ((t[src] == 2) | (t[dst] == 2))
    e = np.nonzero(sel)[0]
    e = e[np.lexsort((e, dst[e], src[e]))]
    order = np.array(sorted(win), np.int64)
    pos = np.full(V, -1, np.int64); pos[order] = np.arange(len(order))
    if nbr_T is None:
        cT = np.tile(np.array([0, 0, 0, 1, 0, 0, 0.0]), (len(e), 1)); cL = np.zeros((len(e), 36))
    else:
        cT = np.asarray(nbr_T, np.float64)[e].reshape(-1, 7); cL = np.asarray(nbr_Lambda, np.float64)[e].reshape(-1, 36)
    return pos[src[e]].astype(np.int32), pos[dst[e]].astype(np.int32), cT, cL


def add_keyframe(m, oldkey, new_pose, new_anchor, new_xyz, new_anchor_center, new_anchor_level, new_center, new_level,
                 track_point, track_center, track_level):
    """oracle.pyoracle.add_keyframe's tables without the Python loop; the new vertex's pose `new_pose` is passed in
    (the caller composes it; the device does the same multiplication)."""
    V, Np = len(m["poses"]), len(m["point_anchor"])
    na = np.asarray(new_anchor, np.int64).reshape(-1)
    tp = np.asarray(track_point, np.int64).reshape(-1)
    nn = len(na)
    vp = np.asarray(m["vis_ptr"], np.int64)
    p_old = np.repeat(np.arange(Np), np.diff(vp))
    pt = np.concatenate([p_old, tp, Np + np.arange(nn), Np + np.arange(nn)])
    vs = np.concatenate([np.asarray(m["vis_pose"], np.int64), np.full(len(tp), V), na, np.full(nn, V)])
    cen = np.concatenate([np.asarray(m["feat_center"], np.float64).reshape(-1, 3), np.asarray(track_center, np.float64).reshape(-1, 3),
                          np.asarray(new_anchor_center, np.float64).reshape(-1, 3), np.asarray(new_center, np.float64).reshape(-1, 3)])
    lvl = np.concatenate([np.asarray(m["feat_level"], np.int64), np.asarray(track_level, np.int64).reshape(-1),
                          np.asarray(new_anchor_level, np.int64).reshape(-1), np.asarray(new_level, np.int64).reshape(-1)])
    o = np.lexsort((vs, pt))
    Np2 = Np + nn
    return dict(poses=np.vstack([m["poses"], np.asarray(new_pose, np.float64).reshape(1, 7)]),
                point_anchor=np.concatenate([m["point_anchor"], na]).astype(np.int32),
                xyz_anchor=np.vstack([m["xyz_anchor"], np.asarray(new_xyz, np.float64).reshape(-1, 3)]),
                vis_ptr=np.searchsorted(pt[o], np.arange(Np2 + 1)).astype(np.int32), vis_pose=vs[o].astype(np.int32),
                feat_center=cen[o], feat_level=lvl[o].astype(np.int32))


# ------------------------------------------------------------------ computeConstraint in long double
LD = np.longdouble


def _R(q):
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    return np.array([[1 - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
                     [ty * x + tz * w, 1 - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, 1 - (tx * x + ty * y)]], dtype=LD)


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], dtype=LD)


def _se3_mul(A, B):
    q = _qmul(A[:4], B[:4])
    q = q / np.sqrt(np.sum(q * q))
    return np.concatenate([q, A[4:] + _R(A[:4]) @ B[4:]])


def _se3_inv(A):
    q = np.array([-A[0], -A[1], -A[2], A[3]], dtype=LD)
    return np.concatenate([q, _R(q) @ (-A[4:])])


def compute_constraint(poses, feat_ptr, feat_point, point_anchor, xyz_anchor, v1, v2):
    """SlamGraph::computeConstraint (reference slam_graph.cpp:785-846) for one pair, in np.longdouble: T_1_from_2, the
    number n of points both frames see, and Lambda = n diag((350 |t12| / med)^2 I3, 100^2 I3) with med the exact
    multiset median of the shared points' distances in frame 1.  Also returns the magnitude companion of T (1 for the
    quaternion, |t1| + |t2| + |t12| for the translation) and of Lambda (n (350 (|t1| + |t2| + |t12|) / med)^2 for the
    translational block, the entry itself for the rotational one): the scale of the rounding a float64 evaluation of the
    same products may carry, so a pair of nearly equal poses (|t12| << |t1|) is judged on that scale."""
    P = np.asarray(poses, np.float64).astype(LD).reshape(-1, 7)
    T1, T2 = P[v1], P[v2]
    T12 = _se3_mul(T1, _se3_inv(T2))
    fp = np.asarray(feat_ptr, np.int64)
    f1 = np.asarray(feat_point, np.int64)[fp[v1]:fp[v1 + 1]]
    f2 = np.asarray(feat_point, np.int64)[fp[v2]:fp[v2 + 1]]
    shared = np.intersect1d(f1, f2)
    n = len(shared)
    xyz = np.asarray(xyz_anchor, np.float64).astype(LD).reshape(-1, 3)
    anc = np.asarray(point_anchor, np.int64)
    d = np.zeros(n, LD)
    for a in np.unique(anc[shared]):                           # v1.T_me_from_world * T_anchor_from_w.inverse() * xyz_anchor
        A = _se3_mul(T1, _se3_inv(P[a]))
        k = anc[shared] == a
        x = xyz[shared[k]] @ _R(A[:4]).T + A[4:]
        d[k] = np.sqrt(np.sum(x * x, 1))
    Lam = np.zeros((6, 6), LD)
    tn = lambda t: np.sqrt(np.sum(t * t))
    scale_t = tn(T1[4:]) + tn(T2[4:]) + tn(T12[4:])
    compT = np.array([1, 1, 1, 1, scale_t, scale_t, scale_t], LD)
    compL = np.zeros((6, 6), LD)
    if n:
        ds = np.sort(d)
        med = ds[n // 2] if n % 2 else (ds[n // 2 - 1] + ds[n // 2]) / 2
        a = 350 * tn(T12[4:]) / med
        for q in range(3):
            Lam[q, q] = n * a * a
            Lam[q + 3, q + 3] = n * LD(100) ** 2
            compL[q, q] = n * (350 * scale_t / med) ** 2
            compL[q + 3, q + 3] = Lam[q + 3, q + 3]
    return T12, Lam, n, compT, compL


def compute_constraints(poses, feat_ptr, feat_point, point_anchor, xyz_anchor, v1, v2):
    """compute_constraint over pairs: (T [n,7], Lambda [n,6,6], strength [n], compT [n,7], compL [n,6,6]), long double."""
    out = [compute_constraint(poses, feat_ptr, feat_point, point_anchor, xyz_anchor, int(a), int(b)) for a, b in zip(v1, v2)]
    return (np.array([o[0] for o in out], LD).reshape(-1, 7), np.array([o[1] for o in out], LD).reshape(-1, 6, 6),
            np.array([o[2] for o in out], np.int64), np.array([o[3] for o in out], LD).reshape(-1, 7),
            np.array([o[4] for o in out], LD).reshape(-1, 6, 6))


def constraint_ratio(got, ref, comp):
    """max |got - ref| / companion over entries whose companion is nonzero; entries with a zero companion must be exact
    (returns inf otherwise)."""
    got, ref, comp = np.asarray(got).astype(LD), np.asarray(ref, LD), np.asarray(comp, LD)
    err = np.abs(got - ref)
    z = comp == 0
    if np.any(err[z] != 0):
        return float("inf")
    return float(np.max(err[~z] / comp[~z])) if np.any(~z) else 0.0


def constraint_tables(P, tables, n_points, seed=0, poses=None, xyz=None, anchor=None):
    """Feature tables for svs_computeConstraint_batch: `tables[v]` is the set of point ids pose v sees (sorted here).
    Poses default to frames near the origin looking along z, points 3..12 m in front of their anchor (pose 0)."""
    rng = np.random.default_rng(seed)
    if poses is None:
        poses = np.zeros((P, 7)); poses[:, 3] = 1.0
        ang = rng.normal(0, 0.05, (P, 3))
        poses[:, :3] = np.sin(ang / 2); poses[:, 3] = np.sqrt(1 - np.sum(poses[:, :3] ** 2, 1))
        poses[:, 4:] = rng.normal(0, 0.5, (P, 3))
    if xyz is None:
        xyz = np.stack([rng.uniform(-2, 2, n_points), rng.uniform(-1.5, 1.5, n_points), rng.uniform(3, 12, n_points)], 1)
    if anchor is None:
        anchor = np.zeros(n_points, np.int32)
    feats = [np.unique(np.asarray(t, np.int64)) for t in tables]
    feat_ptr = np.concatenate([[0], np.cumsum([len(t) for t in feats])]).astype(np.int32)
    feat_point = np.concatenate(feats).astype(np.int32) if feats else np.zeros(0, np.int32)
    return dict(poses=poses, feat_ptr=feat_ptr, feat_point=feat_point, point_anchor=np.asarray(anchor, np.int32),
                xyz_anchor=np.asarray(xyz, np.float64))
