"""ctypes driver of the local-registration oracle (oracle/register_oracle.c, part of liboracle.so).

TEST INFRASTRUCTURE ONLY, like loop_pyoracle.py (whose map structure and matcher bindings it shares)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import loop_pyoracle as lpo, pyoracle

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
_LIB = None

STATS_DTYPE = np.dtype([("vertex", np.int32), ("strength", np.int32), ("num_left", np.int32), ("num_right", np.int32),
                        ("num_upper", np.int32), ("num_lower", np.int32), ("qualified", np.int32)])
COUNTS = ("registered", "stage", "n_direct", "n_neighborhood", "n_candidates", "n_matched1", "n_matched2", "n_tracks",
          "n_stats", "n_neighbors", "n_committed")


class ORegResult(C.Structure):
    _fields_ = [(f, C.c_int) for f in COUNTS] + [
        ("T_align1", C.c_double * 7), ("T_newroot_from_oldroot", C.c_double * 7), ("T_newroot_from_w", C.c_double * 7),
        ("lm", pyoracle.OPOStats * 2), ("err", C.c_int), ("nnz2", C.c_int)]


def lib():
    global _LIB
    if _LIB is None:
        L = lpo.lib()
        L.oreg_local_register_frame.argtypes = [C.POINTER(lpo.OLoopMap), c_ip, c_ip, C.POINTER(pyoracle.OMatchFrame), C.c_void_p,
                                                C.c_int, c_dp, C.c_int, C.c_int, C.c_int, c_ip, c_ip, C.POINTER(ORegResult),
                                                c_ip, c_ip, c_ip, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, c_ip, c_dp,
                                                c_ip, c_ip, c_ip, c_ip, c_dp, c_ip]
        L.oreg_local_register_frame.restype = None
        _LIB = L
    return _LIB


def _d(a):
    return a.ctypes.data_as(c_dp)


def _i(a):
    return a.ctypes.data_as(c_ip)


def local_register_frame(m, nbr_ptr, nbr_id, levels, cur_pyr, disp, features, slot_pyrs, cam, covis_thr, root,
                         window_vertex, vertex_slot):
    """m: svs_map_set's arrays (dict poses, point_anchor, xyz_anchor, vis_ptr, vis_pose, feat_center, feat_level);
    nbr_ptr / nbr_id: the pose graph as svs_map_set_graph takes it; levels [(w, h, f, px, py)], cur_pyr / disp /
    features [(xy, content)] of the root keyframe, slot_pyrs[s] the pyramid in matcher slot s.  Returns (result dict,
    intermediates dict, grown map dict or None)."""
    keep = []
    arr = lambda a, t: keep.append(np.ascontiguousarray(a, t)) or keep[-1]
    poses, anchor, xyz = arr(m["poses"], np.float64), arr(m["point_anchor"], np.int32), arr(m["xyz_anchor"], np.float64)
    vptr, vpose = arr(m["vis_ptr"], np.int32), arr(m["vis_pose"], np.int32)
    cen, lvl = arr(m["feat_center"], np.float64), arr(m["feat_level"], np.int32)
    nptr, nid = arr(nbr_ptr, np.int32), arr(np.concatenate([np.asarray(nbr_id, np.int32), [0]]), np.int32)
    V, Np, nnz = len(poses), len(anchor), len(vpose)
    om = lpo.OLoopMap(V, Np, _d(poses), _i(anchor), _d(xyz), _i(vptr), _i(vpose), _d(cen), _i(lvl))
    fr = pyoracle.OMatchFrame()
    trees = [pyoracle.QuadTree(levels[l][0], levels[l][1], *features[l]) for l in range(len(levels))]
    for l, (w, h, f, px, py) in enumerate(levels):
        fr.levels[l] = pyoracle.OMatchLevel(int(w), int(h), float(f), float(px), float(py))
        im = arr(cur_pyr[l], np.uint8)
        fr.pyr[l] = im.ctypes.data_as(pyoracle.c_up); fr.pitch[l] = im.strides[0]
        fr.trees[l] = trees[l].ptr
    d = arr(disp, np.float32)
    fr.disp = d.ctypes.data_as(pyoracle.c_fp); fr.disp_pitch = d.shape[1]
    nkf = max(len(slot_pyrs), 1)
    kfs = (pyoracle.OMatchKeyframe * nkf)()
    for s, pyr in enumerate(slot_pyrs):
        for l in range(len(levels)):
            im = arr(pyr[l], np.uint8)
            kfs[s].pyr[l] = im.ctypes.data_as(pyoracle.c_up); kfs[s].pitch[l] = im.strides[0]
    win, slot = arr(window_vertex, np.int32), arr(vertex_slot, np.int32)
    camv = arr(cam, np.float64)
    cap = max(Np, 1)
    dr, nb = np.zeros(V, np.int32), np.zeros(V, np.int32)
    cp = np.zeros(cap, np.int32)
    cand = np.zeros(cap, pyoracle.MATCH_POINT_DTYPE)
    r1, r2 = np.zeros(cap, pyoracle.MATCH_RESULT_DTYPE), np.zeros(cap, pyoracle.MATCH_RESULT_DTYPE)
    st = np.zeros(V, STATS_DTYPE)
    tp, tu, tl, tc = np.zeros(cap, np.int32), np.zeros((cap, 3)), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    vp2, vs2, c2, l2 = np.zeros(Np + 1, np.int32), np.zeros(nnz + cap, np.int32), np.zeros((nnz + cap, 3)), np.zeros(nnz + cap, np.int32)
    r = ORegResult()
    lib().oreg_local_register_frame(C.byref(om), _i(nptr), _i(nid), C.byref(fr), kfs, nkf, _d(camv), int(covis_thr), int(root),
                                    len(win), _i(win), _i(slot), C.byref(r), _i(dr), _i(nb), _i(cp), cand.ctypes.data,
                                    r1.ctypes.data, r2.ctypes.data, st.ctypes.data, _i(tp), _d(tu), _i(tl), _i(tc), _i(vp2),
                                    _i(vs2), _d(c2), _i(l2))
    out = {f: getattr(r, f) for f in COUNTS + ("err",)}
    for f in ("T_align1", "T_newroot_from_oldroot", "T_newroot_from_w"):
        out[f] = np.array(getattr(r, f)[:])
    out["lm"] = [{f: getattr(r.lm[k], f) for f in ("initial_chi2", "chi2", "max_err", "num_obs", "iterations", "trials",
                                                   "nan_error")} for k in range(2)]
    nc = r.n_candidates
    gated = r.stage in (0, 4)
    nt, ns = (r.n_tracks, r.n_stats) if gated else (0, 0)
    inter = dict(direct=np.flatnonzero(dr), neighborhood=np.flatnonzero(nb), cand_point=cp[:nc].copy(), cand=cand[:nc].copy(),
                 res1=r1[:nc].copy(), res2=r2[:nc].copy(), stats=st[:ns].copy(),
                 tracks=dict(point=tp[:nt].copy(), uvu=tu[:nt].copy(), level=tl[:nt].copy(), committed=tc[:nt].copy()))
    grown = None
    if r.registered:
        n2 = r.nnz2
        grown = dict(m, vis_ptr=vp2, vis_pose=vs2[:n2].copy(), feat_center=c2[:n2].copy(), feat_level=l2[:n2].copy())
    return out, inter, grown
