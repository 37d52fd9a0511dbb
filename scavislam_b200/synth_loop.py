"""Seeded synthetic revisit for loop verification (Backend::globalLoopClosure, reference backend.cpp:830-1001).

Keyframes rendered with synth_images.render_frame along a small closed path (a circle in the ground plane with a gentle
heading wobble) whose last keyframe comes back near the first.  The map is built like the back-end builds it: every
keyframe anchors points at its FAST corners that have a disparity (two pyramid levels), each seen by its anchor and by
the keyframes up to `reach` steps before or after it on the path where it projects into their frame.  The stored
poses of the second half of the path have drifted, so the loop keyframe's map pose is off by a few cm and about a
degree relative to the query, and the proposal T_query_from_loop is off by `prop_err` (metres, degrees) from the truth.  Input generation
only."""
from __future__ import annotations

import numpy as np

from . import frontend_inputs as fi
from .synth import CAM_B, CAM_F, CAM_H, CAM_PX, CAM_PY, CAM_W
from .synth_images import render_frame

NLV = 2


def _quat(R):
    w = np.sqrt(max(1e-12, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])


def _R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _roty(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _rotvec(v):
    th = np.linalg.norm(v)
    if th < 1e-15:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def pose(R, t):
    return np.concatenate([_quat(R), t])


def mul(A, B):
    return pose(_R(A[:4]) @ _R(B[:4]), _R(A[:4]) @ B[4:] + A[4:])


def inv(A):
    Rt = _R(A[:4]).T
    return pose(Rt, -Rt @ A[4:])


def act(A, X):
    return X @ _R(A[:4]).T + A[4:]


def perturb(T, dt, drot_deg, rng):
    """T with a translation of |dt| metres and a rotation of drot_deg degrees about random axes applied on the left."""
    a = rng.normal(size=3); a /= np.linalg.norm(a)
    b = rng.normal(size=3); b /= np.linalg.norm(b)
    return mul(pose(_rotvec(np.deg2rad(drot_deg) * b), dt * a), T)


def levels():
    cams = fi.level_cams(CAM_F, CAM_PX, CAM_PY, CAM_B, nlevels=NLV)
    return [(CAM_W >> l, CAM_H >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(NLV)]


def fast_features(oracle, pyr):
    """FAST corners per level as recomputeFastCorners gives them (x, y, content = index inside its cell)."""
    out = []
    for l in range(NLV):
        g = oracle.fast_grid(CAM_W >> l, CAM_H >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
        xy, off = oracle.fast_detect_adaptively(pyr[l], g, 5)
        content = np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(len(off) - 1)]).astype(np.int32)
        out.append((xy, content))
    return out


def make_scene(oracle, n_kf=8, radius=0.4, reach=2, per_level=(160, 60), drift=(0.03, 1.0), prop_err=(0.04, 1.5),
               revisit=(0.02, 0.5), seed=5):
    """Keyframes 0..n_kf on the path (n_kf = the query, back near keyframe 0 = the loop).  Returns a dict with the
    images, the map (svs_map_set's arrays), the true and stored poses and the proposal."""
    rng = np.random.default_rng(seed)
    cams = fi.level_cams(CAM_F, CAM_PX, CAM_PY, CAM_B, nlevels=NLV)
    lv = levels()
    true_T, frames = [], []
    for k in range(n_kf + 1):
        a = 2 * np.pi * k / n_kf
        c = np.array([radius * np.sin(a), 0.0, radius * (1 - np.cos(a))])
        yaw = np.deg2rad(3.0) * np.sin(a)
        if k == n_kf:                                   # the revisit: near, not on, keyframe 0
            c = c + np.array([revisit[0], 0.0, 0.5 * revisit[0]])
            yaw += np.deg2rad(revisit[1])
        img, disp = render_frame(c, yaw, seed=77)
        Rwc = _roty(yaw)
        true_T.append(pose(Rwc.T, -Rwc.T @ c))
        frames.append(dict(pyr=fi.uint8_pyramid(img, NLV), disp=disp))
    V = n_kf + 1
    # stored poses: the second half of the path has drifted rigidly (a world-frame offset of `drift`), so the loop
    # keyframe's map pose is off by that much relative to the query while the query's window stays consistent
    Dw = perturb(pose(np.eye(3), np.zeros(3)), drift[0], drift[1], rng)
    stored = [mul(true_T[k], Dw) if 2 * k >= n_kf else true_T[k] for k in range(V)]
    anchor, xyz, obs = [], [], []            # obs: per point a list of (vertex, centre[3], level)
    for k in range(V):
        pyr, disp = frames[k]["pyr"], frames[k]["disp"]
        for l in range(NLV):
            g = oracle.fast_grid(CAM_W >> l, CAM_H >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
            kxy, _ = oracle.fast_detect_adaptively(pyr[l], g, 5)
            d = disp[kxy[:, 1] << l, kxy[:, 0] << l] / (1 << l)
            kxy, d = kxy[d > 0.5], d[d > 0.5]
            if len(kxy) > per_level[l]:
                sel = np.sort(rng.choice(len(kxy), per_level[l], replace=False))
                kxy, d = kxy[sel], d[sel]
            f, px, py, _ = cams[l]
            z = CAM_F * CAM_B / (d * (1 << l))          # depth from the level-0 disparity
            X = np.stack([(kxy[:, 0] - px) / f * z, (kxy[:, 1] - py) / f * z, z], 1)
            s = float(1 << l)
            for i in range(len(kxy)):
                o = []
                Xw = act(inv(true_T[k]), X[i][None])[0]
                for j in range(max(0, k - reach), min(V, k + reach + 1)):
                    if j == k:
                        o.append((k, np.array([kxy[i, 0] * s, kxy[i, 1] * s, (kxy[i, 0] - d[i]) * s]), l))
                        continue
                    Xj = act(true_T[j], Xw[None])[0]
                    if Xj[2] < 0.5:
                        continue
                    u = CAM_F * Xj[0] / Xj[2] + CAM_PX
                    v = CAM_F * Xj[1] / Xj[2] + CAM_PY
                    if 0 <= u < CAM_W and 0 <= v < CAM_H:
                        o.append((j, np.array([u, v, CAM_F * (Xj[0] - CAM_B) / Xj[2] + CAM_PX]), l))
                anchor.append(k); xyz.append(X[i]); obs.append(o)
    vis_ptr = np.zeros(len(anchor) + 1, np.int32)
    vis_ptr[1:] = np.cumsum([len(o) for o in obs])
    m = dict(poses=np.array(stored), point_anchor=np.array(anchor, np.int32), xyz_anchor=np.array(xyz),
             vis_ptr=vis_ptr, vis_pose=np.array([v for o in obs for v, _, _ in o], np.int32),
             feat_center=np.array([c for o in obs for _, c, _ in o]).reshape(-1, 3),
             feat_level=np.array([l for o in obs for _, _, l in o], np.int32))
    query, loop = n_kf, 0
    T_true_ql = mul(true_T[query], inv(true_T[loop]))
    return dict(levels=lv, cam=(CAM_F, CAM_PX, CAM_PY, CAM_B), frames=frames, map=m, true_T=np.array(true_T),
                query=query, loop=loop, window=np.arange(max(0, n_kf - 2 * reach), n_kf + 1, dtype=np.int32),
                T_true_query_from_loop=T_true_ql, T_query_from_loop=perturb(T_true_ql, prop_err[0], prop_err[1], rng),
                loop_features=fast_features(oracle, frames[loop]["pyr"]))


def path_graph(m, V, reach):
    """The pose graph of the path: keyframes within `reach` steps are neighbours, with strength = the number of points
    both observe, listed strongest first (ties: the larger id first).  Returns svs_map_set_graph's (nbr_ptr, nbr_id)."""
    sees = [set() for _ in range(V)]
    for p in range(len(m["point_anchor"])):
        for v in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]]:
            sees[int(v)].add(p)
    ptr, ids = [0], []
    for v in range(V):
        nb = [(len(sees[v] & sees[j]), j) for j in range(max(0, v - reach), min(V, v + reach + 1)) if j != v]
        ids += [j for _, j in sorted(nb, reverse=True)]
        ptr.append(len(ids))
    return np.array(ptr, np.int32), np.array(ids, np.int32)


def make_register_scene(oracle, n_kf=8, reach=2, **kw):
    """A revisit inside the double window for Backend::localRegisterFrame: the path of make_scene with every keyframe
    0..n_kf in the window and the pose graph of path_graph.  Root is the last keyframe; its direct neighbours are the
    `reach` keyframes before it, and it sees the points of keyframes 0 and 1, which are in its window but not its
    neighbours.  Root's stored pose has drifted by make_scene's `drift`; every other stored pose is true, so the points
    the registration matches against all place root where it truly is."""
    sc = make_scene(oracle, n_kf=n_kf, reach=reach, **kw)
    T, st = sc["true_T"], sc["map"]["poses"]
    Dw = mul(inv(T[n_kf]), st[n_kf])
    poses = np.array([mul(T[k], Dw) if k == n_kf else T[k] for k in range(n_kf + 1)])
    m = dict(sc["map"], poses=poses)
    nbr_ptr, nbr_id = path_graph(m, n_kf + 1, reach)
    return dict(sc, map=m, root=n_kf, window=np.arange(n_kf + 1, dtype=np.int32), nbr_ptr=nbr_ptr, nbr_id=nbr_id,
                root_features=fast_features(oracle, sc["frames"][n_kf]["pyr"]))


def make_flat_register_scene(oracle, n, n_direct_anchored=0, seed=11):
    """A flat map for Backend::localRegisterFrame: vertices 0 (root), 1 (its only neighbour), 2 and 3 all at the
    identity and all seeing the same rendered image, with the pose graph 0-1-2-3.  n points at FAST corners (in the
    order `seed` shuffles them) are anchored in 2 and seen by 2 and 3 (3 observes them but anchors none); the next
    n_direct_anchored corners are anchored in the direct neighbour 1 and seen by 1 and 2.  Every candidate is predicted
    on the corner it was made from, so the number of tracks follows n."""
    from .synth_images import render_frame as _render
    img, disp = _render(np.zeros(3), 0.0, seed=77)
    pyr = fi.uint8_pyramid(img, NLV)
    xy = oracle.fast_detect_roi(img, 8, 632, 8, 472, 12)
    xy = xy[disp[xy[:, 1], xy[:, 0]] > 1]
    xy = xy[np.random.default_rng(seed).permutation(len(xy))]
    feats = []
    for l in range(NLV):
        k = oracle.fast_detect_roi(pyr[l], 0, CAM_W >> l, 0, CAM_H >> l, 12)
        feats.append((k, np.arange(len(k), dtype=np.int32)))
    N = n + n_direct_anchored
    assert N <= len(xy)
    u, v = xy[:N, 0].astype(np.float64), xy[:N, 1].astype(np.float64)
    d = disp[xy[:N, 1], xy[:N, 0]].astype(np.float64)
    z = CAM_F * CAM_B / d
    X = np.stack([(u - CAM_PX) / CAM_F * z, (v - CAM_PY) / CAM_F * z, z], 1)
    vp, vs, cen, anchor = [0], [], [], []
    for p in range(N):
        a, seen = (2, (2, 3)) if p < n else (1, (1, 2))
        anchor.append(a)
        for vert in seen:
            vs.append(vert); cen.append([u[p], v[p], u[p] - d[p]])
        vp.append(len(vs))
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    m = dict(poses=np.tile(I7, (4, 1)), point_anchor=np.array(anchor, np.int32), xyz_anchor=X.reshape(-1, 3),
             vis_ptr=np.array(vp, np.int32), vis_pose=np.array(vs, np.int32), feat_center=np.array(cen).reshape(-1, 3),
             feat_level=np.zeros(len(vs), np.int32))
    fr = dict(pyr=pyr, disp=disp)
    return dict(levels=levels(), cam=(CAM_F, CAM_PX, CAM_PY, CAM_B), frames=[fr] * 4, map=m, root=0,
                window=np.arange(4, dtype=np.int32), nbr_ptr=np.array([0, 1, 3, 5, 6], np.int32),
                nbr_id=np.array([1, 0, 2, 1, 3, 2], np.int32), root_features=feats)
