"""ctypes driver of the pose-graph growth oracle (oracle/graph_oracle.c, part of liboracle.so).

TEST INFRASTRUCTURE ONLY.  A map is a dict of svs_map_set's arrays (poses, point_anchor, xyz_anchor, vis_ptr, vis_pose,
feat_center, feat_level); a graph is a dict(nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        L = pyoracle.lib()
        L.ogr_compute_strength.argtypes = [C.c_int, c_ip, c_ip, C.c_int, c_ip, C.c_int, c_ip, c_dp, C.c_int, C.c_int, C.c_int,
                                           c_ip, c_ip]
        L.ogr_compute_strength.restype = None
        L.ogr_add_edges.argtypes = [C.c_int, C.c_int, c_ip, c_ip, c_ip, c_dp, c_dp, C.c_int, c_ip, c_ip, c_ip, c_dp, c_ip, c_ip,
                                    C.c_int, c_ip, c_dp, c_ip, c_ip, c_ip, c_dp, c_dp]
        L.ogr_add_edges.restype = None
        L.occ_compute_constraints.argtypes = [C.c_int, c_dp, c_ip, c_ip, C.c_int, c_ip, c_dp, C.c_int, c_ip, c_ip, c_dp, c_dp, c_ip]
        L.occ_compute_constraints.restype = None
        _LIB = L
    return _LIB


def _i(a):
    return np.ascontiguousarray(a, np.int32)


def _d(a):
    return np.ascontiguousarray(a, np.float64)


def _pi(a):
    return a.ctypes.data_as(c_ip)


def _pd(a):
    return a.ctypes.data_as(c_dp)


def compute_strength(m, new_anchor, track_point, track_center, covis_thr, width, height):
    """computeStrength's literal loops on the map before growth.  Returns (in_table [V] bool, strength [V])."""
    V = len(m["poses"])
    vp, vs = _i(m["vis_ptr"]), _i(np.concatenate([np.asarray(m["vis_pose"]), [0]]))
    na, tp = _i(np.concatenate([np.asarray(new_anchor, np.int64).reshape(-1), [0]])), _i(np.concatenate([np.asarray(track_point, np.int64).reshape(-1), [0]]))
    tc = _d(np.vstack([np.asarray(track_center, np.float64).reshape(-1, 3), np.zeros((1, 3))]))
    inn, st = np.zeros(V, np.int32), np.zeros(V, np.int32)
    lib().ogr_compute_strength(V, _pi(vp), _pi(vs), len(na) - 1, _pi(na), len(tp) - 1, _pi(tp), _pd(tc), int(covis_thr), int(width),
                               int(height), _pi(inn), _pi(st))
    return inn.astype(bool), st


def strength_table(m, oldkey, new_anchor, track_point, track_center, covis_thr, width, height):
    """The rows (vertex, strength) of addKeyframe's table after the oldkey bump, ascending vertex; None when oldkey is
    absent (the reference asserts)."""
    inn, st = compute_strength(m, new_anchor, track_point, track_center, covis_thr, width, height)
    if not inn[oldkey]:
        return None
    st = st.copy()
    st[oldkey] = max(st[oldkey], covis_thr)
    v = np.flatnonzero(inn)
    return np.stack([v, st[v]], 1).astype(np.int32)


def feature_tables(m):
    """Vertex::feature_table keys of every vertex, ascending point id: (feat_ptr [V+1], feat_point)."""
    V, Np = len(m["poses"]), len(m["point_anchor"])
    vp = np.asarray(m["vis_ptr"], np.int64)
    pt = np.repeat(np.arange(Np), np.diff(vp))
    vs = np.asarray(m["vis_pose"], np.int64)
    o = np.lexsort((pt, vs))
    return np.searchsorted(vs[o], np.arange(V + 1)).astype(np.int32), pt[o].astype(np.int32)


def constraints(poses, feat_ptr, feat_point, point_anchor, xyz_anchor, v1, v2):
    """computeConstraint(v1[k], v2[k]) by constraint_oracle.c: (T_1_from_2 [n,7], Lambda [n,36], strength [n])."""
    P, Np = len(poses), len(point_anchor)
    a, b = _i(np.concatenate([np.asarray(v1).reshape(-1), [0]])), _i(np.concatenate([np.asarray(v2).reshape(-1), [0]]))
    n = len(a) - 1
    pose = _d(np.asarray(poses).reshape(-1, 7))
    fp, ft = _i(feat_ptr), _i(np.concatenate([np.asarray(feat_point).reshape(-1), [0]]))
    anc, xyz = _i(np.concatenate([point_anchor, [0]])), _d(np.vstack([np.asarray(xyz_anchor).reshape(-1, 3), np.zeros((1, 3))]))
    T, L, s = np.zeros((n + 1, 7)), np.zeros((n + 1, 36)), np.zeros(n + 1, np.int32)
    lib().occ_compute_constraints(P, _pd(pose), _pi(fp), _pi(ft), Np, _pi(anc), _pd(xyz), n, _pi(a), _pi(b), _pd(T), _pd(L), _pi(s))
    return T[:n], L[:n], s[:n]


def add_edges(graph, m, v1, v2, strength, moved_vertex=-1, T_moved_from_w=None, feat=None):
    """The edges (v1[k], v2[k], strength[k]) inserted in order into `graph` (its lists may number fewer than the map's
    vertices: the rest start empty), each with computeConstraint(v1, v2) on the map, moved_vertex placed at
    T_moved_from_w.  feat: the map's feature_tables when the caller keeps them.  Returns the new graph."""
    V = len(m["poses"])
    gV = len(graph["nbr_ptr"]) - 1
    poses = _d(m["poses"]).copy()
    if moved_vertex >= 0:
        poses[moved_vertex] = np.asarray(T_moved_from_w, np.float64).reshape(7)
    fptr, fpt = feature_tables(m) if feat is None else feat
    fpt = _i(np.concatenate([fpt, [0]]))
    a, b, s = (_i(np.concatenate([np.asarray(x, np.int64).reshape(-1), [0]])) for x in (v1, v2, strength))
    n = len(a) - 1
    nn = len(graph["nbr_id"])
    pad = lambda x, w: np.vstack([np.asarray(x, np.float64).reshape(-1, w), np.zeros((1, w))])
    gp, gi, gs = _i(graph["nbr_ptr"]), _i(np.concatenate([graph["nbr_id"], [0]])), _i(np.concatenate([graph["nbr_strength"], [0]]))
    gT, gL = _d(pad(graph["nbr_T"], 7)), _d(pad(graph["nbr_Lambda"], 36))
    Np = len(m["point_anchor"])
    anc, xyz = _i(np.concatenate([m["point_anchor"], [0]])), _d(pad(m["xyz_anchor"], 3))
    op, oi, os_ = np.zeros(V + 1, np.int32), np.zeros(nn + 2 * n + 1, np.int32), np.zeros(nn + 2 * n + 1, np.int32)
    oT, oL = np.zeros((nn + 2 * n + 1, 7)), np.zeros((nn + 2 * n + 1, 36))
    lib().ogr_add_edges(gV, V, _pi(gp), _pi(gi), _pi(gs), _pd(gT), _pd(gL), n, _pi(a), _pi(b), _pi(s), _pd(poses), _pi(_i(fptr)),
                        _pi(fpt), Np, _pi(anc), _pd(xyz), _pi(op), _pi(oi), _pi(os_), _pd(oT), _pd(oL))
    k = nn + 2 * n
    return dict(nbr_ptr=op, nbr_id=oi[:k], nbr_strength=os_[:k], nbr_T=oT[:k], nbr_Lambda=oL[:k])


def local_edges(table, covis_thr, newkey):
    """addNewEdges(LOCAL)'s edges from the strength table, in ascending vertex order: (v1, v2, strength)."""
    t = np.asarray(table, np.int64).reshape(-1, 2)
    q = t[t[:, 1] >= covis_thr]
    return q[:, 0].astype(np.int32), np.full(len(q), newkey, np.int32), q[:, 1].astype(np.int32)
