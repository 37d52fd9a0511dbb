"""ctypes driver of the prepareForOptimization oracle (oracle/prepare_oracle.c, part of liboracle.so).

TEST INFRASTRUCTURE ONLY.  It takes and returns a device map's state: the graph as svs_map_get_graph lays it out
(dict(nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda)), the window state of svs_map_get_window_state and the map's
tables (svs_map_set's arrays with the current poses)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle
from oracle.graph_pyoracle import _d, _i, _pd, _pi, feature_tables

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
c_up = C.POINTER(C.c_ubyte)
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        L = pyoracle.lib()
        L.opr_prepare_for_optimization.argtypes = [C.c_int, c_ip, c_ip, c_dp, c_dp, c_up, c_ip, c_ip, C.c_int, C.c_int, c_dp, c_ip,
                                                   c_ip, C.c_int, c_ip, c_dp, c_dp, c_dp, c_up, c_up]
        L.opr_prepare_for_optimization.restype = None
        _LIB = L
    return _LIB


def _pu(a):
    return a.ctypes.data_as(c_up)


def prepare_for_optimization(graph, marginalized, old_type, m, root, loop, inner_window_size, double_window_size, feat=None):
    """SlamGraph::prepareForOptimization(root, loop) from a device map's state: `graph` as get_graph returns it,
    marginalized [nnzN] and old_type [V] as window_state returns them, `m` the map's tables with its current poses.
    The window is pyoracle's computeInitialDoubleWin + computeActivePointsAndExtendOuterWindow; the rest is
    opr_prepare_for_optimization.  Returns dict(poses, graph, marginalized, rewritten (bool per entry), window_type,
    window_vertex, inner, active_point, do_optimization)."""
    V = len(m["poses"])
    ptr, ids = _i(graph["nbr_ptr"]), _i(graph["nbr_id"])
    win = pyoracle.compute_double_window(ptr, ids, root, inner_window_size, double_window_size)
    active, win = pyoracle.compute_active_points(m, ptr, ids, win)
    new_t = np.zeros(V, np.int32)
    for v, t in win.items():
        new_t[v] = t
    nn = len(ids)
    pad = lambda x, w: _d(np.vstack([np.asarray(x, np.float64).reshape(-1, w), np.zeros((1, w))]))
    gi = _i(np.concatenate([ids, [0]]))
    gT, gL = pad(graph["nbr_T"], 7), pad(graph["nbr_Lambda"], 36)
    mg = np.ascontiguousarray(np.concatenate([np.asarray(marginalized, np.uint8), [0]]), np.uint8)
    old_t = _i(old_type)
    poses = _d(m["poses"]).copy()
    fptr, fpt = feature_tables(m) if feat is None else feat
    fpt = _i(np.concatenate([fpt, [0]]))
    Np = len(m["point_anchor"])
    anc, xyz = _i(np.concatenate([m["point_anchor"], [0]])), pad(m["xyz_anchor"], 3)
    oT, oL = np.zeros((nn + 1, 7)), np.zeros((nn + 1, 36))
    om, rw = np.zeros(nn + 1, np.uint8), np.zeros(nn + 1, np.uint8)
    lib().opr_prepare_for_optimization(V, _pi(ptr), _pi(gi), _pd(gT), _pd(gL), _pu(mg), _pi(old_t), _pi(new_t), int(root), int(loop),
                                       _pd(poses), _pi(_i(fptr)), _pi(fpt), Np, _pi(anc), _pd(xyz), _pd(oT), _pd(oL), _pu(om), _pu(rw))
    g = dict(graph)
    g["nbr_T"], g["nbr_Lambda"] = oT[:nn], oL[:nn]
    wv = np.array(sorted(win), np.int32)
    return dict(poses=poses, graph=g, marginalized=om[:nn], rewritten=rw[:nn].astype(bool), window_type=new_t.astype(np.uint8),
                window_vertex=wv, inner=(new_t[wv] == 1).astype(np.uint8), active_point=np.asarray(active, np.int32),
                do_optimization=len(wv) >= 2)
