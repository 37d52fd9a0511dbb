"""ctypes driver of the loop-verification oracle (oracle/loop_oracle.c, part of liboracle.so).

TEST INFRASTRUCTURE ONLY, like pyoracle.py (whose build of liboracle.so and matcher bindings it shares)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
_LIB = None


class OLoopMap(C.Structure):
    _fields_ = [("V", C.c_int), ("Np", C.c_int), ("pose", c_dp), ("anchor", c_ip), ("xyz", c_dp), ("vis_ptr", c_ip),
                ("vis_pose", c_ip), ("center", c_dp), ("level", c_ip)]


class OLoopResult(C.Structure):
    _fields_ = [("verified", C.c_int), ("stage", C.c_int), ("n_candidates", C.c_int), ("n_matched1", C.c_int),
                ("n_matched2", C.c_int), ("n_tracks", C.c_int), ("num_left", C.c_int), ("num_right", C.c_int),
                ("num_upper", C.c_int), ("num_lower", C.c_int), ("T_loop_from_w", C.c_double * 7),
                ("T_align1", C.c_double * 7), ("T_newloop_from_oldloop", C.c_double * 7),
                ("T_newloop_from_w", C.c_double * 7), ("lm", pyoracle.OPOStats * 2), ("err", C.c_int), ("nnz2", C.c_int)]


def lib():
    global _LIB
    if _LIB is None:
        L = pyoracle.lib()
        L.oloop_global_loop_closure.argtypes = [C.POINTER(OLoopMap), C.POINTER(pyoracle.OMatchFrame), C.c_void_p, C.c_int,
                                                c_dp, C.c_int, C.c_int, C.c_int, c_dp, C.c_int, c_ip, c_ip,
                                                C.POINTER(OLoopResult), c_ip, C.c_void_p, C.c_void_p, C.c_void_p, c_ip, c_dp,
                                                c_ip, c_ip, c_ip, c_dp, c_ip]
        L.oloop_global_loop_closure.restype = None
        L.oloop_map_uvu.argtypes = [c_dp] * 4
        L.oloop_map_uvu.restype = None
        for n, k in (("oloop_se3_mul", 3), ("oloop_se3_inv", 2), ("oloop_se3_act", 3)):
            getattr(L, n).argtypes = [c_dp] * k
            getattr(L, n).restype = None
        _LIB = L
    return _LIB


def _d(a):
    return a.ctypes.data_as(c_dp)


def _i(a):
    return a.ctypes.data_as(c_ip)


def se3(name, *args):
    args = [np.ascontiguousarray(a, np.float64) for a in args]
    out = np.zeros(7 if name != "oloop_se3_act" else 3)
    getattr(lib(), name)(*[_d(a) for a in args], _d(out))
    return out


def map_uvu(cam, T, xyz):
    out = np.zeros(3)
    lib().oloop_map_uvu(_d(np.ascontiguousarray(cam, np.float64)), _d(np.ascontiguousarray(T, np.float64)),
                        _d(np.ascontiguousarray(xyz, np.float64)), _d(out))
    return out


def global_loop_closure(m, levels, cur_pyr, disp, features, slot_pyrs, cam, covis_thr, query, loop, T_query_from_loop,
                        window_vertex, vertex_slot):
    """m: svs_map_set's arrays (dict poses, point_anchor, xyz_anchor, vis_ptr, vis_pose, feat_center, feat_level);
    levels [(w, h, f, px, py)], cur_pyr / disp / features [(xy, content)] of the loop keyframe, slot_pyrs[s] the pyramid
    in matcher slot s.  Returns (result dict, intermediates dict, grown map dict or None)."""
    keep = []
    arr = lambda a, t: keep.append(np.ascontiguousarray(a, t)) or keep[-1]
    poses, anchor, xyz = arr(m["poses"], np.float64), arr(m["point_anchor"], np.int32), arr(m["xyz_anchor"], np.float64)
    vptr, vpose = arr(m["vis_ptr"], np.int32), arr(m["vis_pose"], np.int32)
    cen, lvl = arr(m["feat_center"], np.float64), arr(m["feat_level"], np.int32)
    V, Np, nnz = len(poses), len(anchor), len(vpose)
    om = OLoopMap(V, Np, _d(poses), _i(anchor), _d(xyz), _i(vptr), _i(vpose), _d(cen), _i(lvl))
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
    Tq = arr(T_query_from_loop, np.float64)
    camv = arr(cam, np.float64)
    cap = max(Np, 1)
    cp = np.zeros(cap, np.int32)
    cand = np.zeros(cap, pyoracle.MATCH_POINT_DTYPE)
    r1, r2 = np.zeros(cap, pyoracle.MATCH_RESULT_DTYPE), np.zeros(cap, pyoracle.MATCH_RESULT_DTYPE)
    tp, tu, tl = np.zeros(cap, np.int32), np.zeros((cap, 3)), np.zeros(cap, np.int32)
    vp2, vs2, c2, l2 = np.zeros(Np + 1, np.int32), np.zeros(nnz + cap, np.int32), np.zeros((nnz + cap, 3)), np.zeros(nnz + cap, np.int32)
    r = OLoopResult()
    lib().oloop_global_loop_closure(C.byref(om), C.byref(fr), kfs, nkf, _d(camv), int(covis_thr), int(query), int(loop), _d(Tq),
                                    len(win), _i(win), _i(slot), C.byref(r), _i(cp), cand.ctypes.data, r1.ctypes.data,
                                    r2.ctypes.data, _i(tp), _d(tu), _i(tl), _i(vp2), _i(vs2), _d(c2), _i(l2))
    out = {f: getattr(r, f) for f in ("verified", "stage", "n_candidates", "n_matched1", "n_matched2", "n_tracks", "num_left",
                                      "num_right", "num_upper", "num_lower", "err")}
    for f in ("T_loop_from_w", "T_align1", "T_newloop_from_oldloop", "T_newloop_from_w"):
        out[f] = np.array(getattr(r, f)[:])
    out["lm"] = [{f: getattr(r.lm[k], f) for f in ("initial_chi2", "chi2", "max_err", "num_obs", "iterations", "trials",
                                                   "nan_error")} for k in range(2)]
    nc, nt = r.n_candidates, r.n_tracks if r.stage in (0, 3, 4) else 0
    inter = dict(cand_point=cp[:nc].copy(), cand=cand[:nc].copy(), res1=r1[:nc].copy() if r.stage >= 1 or r.stage == 0 else None,
                 res2=r2[:nc].copy(), tracks=dict(point=tp[:nt].copy(), uvu=tu[:nt].copy(), level=tl[:nt].copy()))
    grown = None
    if r.verified:
        n2 = r.nnz2
        grown = dict(m, vis_ptr=vp2, vis_pose=vs2[:n2].copy(), feat_center=c2[:n2].copy(), feat_level=l2[:n2].copy())
    return out, inter, grown
