"""The tracked frame's bookkeeping of StereoFrontend, twice: a ctypes driver of oracle/frontend_oracle.c (part of
liboracle.so), and an independent pure-Python restatement that builds the reference's adaptive quadtree literally
(quadtree.h: insert with splits, isWindowEmpty, an EquiIter walking it depth by depth with the seeded hash rules stated
in frontend_oracle.h).  The restatement pins the claim that the regular-tree formulation of the C oracle equals the
adaptive one.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from oracle import pyoracle

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
_LIB = None
M64 = (1 << 64) - 1

STATS_FIELDS = [("num_matched_points", C.c_int * 4), ("grid2x2", C.c_int * 4), ("grid3x3", C.c_int * 9),
                ("av_track_length", C.c_double), ("num_tracked", C.c_int), ("num_new", C.c_int)]
TRACKED_DTYPE = np.dtype([("index", "i4"), ("is_new", "i4"), ("anchor_level", "i4"), ("reserved", "i4"),
                          ("uvu", "f8", 3)])
NEW_POINT_DTYPE = np.dtype([("level", "i4"), ("reserved", "i4"), ("uv_pyr", "f8", 2), ("uvu_pyr", "f8", 3),
                            ("xyz", "f8", 3), ("normal", "f8", 3)])
MATCH_POINT_DTYPE = np.dtype([("keyframe", "i4"), ("anchor_level", "i4"), ("xyz_anchor", "f8", 3),
                              ("anchor_obs_pyr", "f8", 2)])
MATCH_RESULT_DTYPE = np.dtype([("predicted", "i4"), ("textured", "i4"), ("matched", "i4"), ("n_candidates", "i4"),
                               ("index", "i4"), ("min_dist", "i4"), ("uv_pyr", "i4", 2), ("obs", "f8", 3),
                               ("xyz_actkey", "f8", 3)])


class OFrontStats(C.Structure):
    _fields_ = STATS_FIELDS


def stats_dict(st):
    return dict(num_matched_points=list(st.num_matched_points), grid2x2=np.array(st.grid2x2[:]).reshape(2, 2),
                grid3x3=np.array(st.grid3x3[:]).reshape(3, 3), av_track_length=st.av_track_length,
                num_tracked=st.num_tracked, num_new=st.num_new)


def lib():
    global _LIB
    if _LIB is None:
        L = pyoracle.lib()
        vp = C.c_void_p
        L.ofront_budget.argtypes = [vp, C.c_int, c_ip, C.c_int, c_ip, c_ip]
        L.ofront_budget.restype = None
        L.ofront_process.argtypes = [vp, c_ip, C.c_int, C.c_int, c_dp, c_dp, C.c_int, C.c_int, C.c_float, C.c_int, vp,
                                     C.POINTER(OFrontStats), c_ip]
        L.ofront_drop.argtypes = [C.POINTER(OFrontStats), c_dp, C.c_int, C.c_float]
        L.ofront_seed.argtypes = [C.c_int, c_ip, c_ip, C.POINTER(c_ip), c_ip, C.POINTER(C.c_float), C.c_int, vp, C.c_int,
                                  c_ip, c_ip, C.c_int, C.c_int, C.c_ulonglong, c_dp, c_dp, C.c_int, vp, vp, c_ip]
        L.ofront_emission_order.argtypes = [C.c_int, C.c_int, C.c_int, c_ip, C.c_int, C.c_ulonglong, c_ip]
        L.ofront_hash5.argtypes = [C.c_ulonglong] * 5
        L.ofront_hash5.restype = C.c_ulonglong
        _LIB = L
    return _LIB


def _d(a):
    return a.ctypes.data_as(c_dp)


def _i(a):
    return a.ctypes.data_as(c_ip)


def c_budget(res, group_end, num_max_points):
    """res: MATCH_RESULT_DTYPE of all candidates; returns (res after the stop rule, num_new, num_obs)."""
    r = np.array(res, MATCH_RESULT_DTYPE)
    ge = np.ascontiguousarray(group_end, np.int32)
    a, b = C.c_int(), C.c_int()
    lib().ofront_budget(r.ctypes.data, len(ge), _i(ge), int(num_max_points), C.byref(a), C.byref(b))
    return r, a.value, b.value


def c_process(res, anchor_level, n_new, T, cam, w0, h0, max_err=2.0, min_num_points=25):
    r = np.ascontiguousarray(res, MATCH_RESULT_DTYPE)
    lv = np.ascontiguousarray(anchor_level, np.int32)
    out = np.zeros(len(r), TRACKED_DTYPE)
    st = OFrontStats()
    flags = np.zeros(9, np.int32)
    n = lib().ofront_process(r.ctypes.data, _i(lv), len(r), int(n_new), _d(np.ascontiguousarray(T, np.float64)),
                             _d(np.ascontiguousarray(cam, np.float64)), int(w0), int(h0), float(max_err),
                             int(min_num_points), out.ctypes.data, C.byref(st), _i(flags))
    return out[:n], st, flags


def c_drop(st, T, featureless_corners_thr=2, parallax_thr=0.75):
    return lib().ofront_drop(C.byref(st), _d(np.ascontiguousarray(T, np.float64)), featureless_corners_thr,
                             float(parallax_thr))


def c_seed(sizes, corners, disp, tree, num_in, flags, R, num_max_points, seed, T, cam, slot):
    """sizes: [(w, h)] per level; corners: [int array (n, 2)] per level; tree: TRACKED_DTYPE (gated points)."""
    L = len(sizes)
    w = np.array([s[0] for s in sizes], np.int32)
    h = np.array([s[1] for s in sizes], np.int32)
    xy = [np.ascontiguousarray(c, np.int32).reshape(-1, 2) for c in corners]
    xyp = (c_ip * L)(*[_i(a) for a in xy])
    nkp = np.array([len(a) for a in xy], np.int32)
    d = np.ascontiguousarray(disp, np.float32)
    tr = np.ascontiguousarray(tree, TRACKED_DTYPE)
    bound = sum((num_max_points >> l) + 1 for l in range(L))
    pts = np.zeros(bound, NEW_POINT_DTYPE)
    rows = np.zeros(bound, MATCH_POINT_DTYPE)
    counts = np.zeros(L, np.int32)
    n = lib().ofront_seed(L, _i(w), _i(h), xyp, _i(nkp), d.ctypes.data_as(C.POINTER(C.c_float)), d.shape[1],
                          tr.ctypes.data, len(tr), _i(np.ascontiguousarray(num_in, np.int32)),
                          _i(np.ascontiguousarray(flags, np.int32)), int(R), int(num_max_points), int(seed),
                          _d(np.ascontiguousarray(T, np.float64)), _d(np.ascontiguousarray(cam, np.float64)), int(slot),
                          pts.ctypes.data, rows.ctypes.data, _i(counts))
    return pts[:n], rows[:n], counts


def c_emission_order(w, h, level, xy, seed):
    xy = np.ascontiguousarray(xy, np.int32).reshape(-1, 2)
    out = np.zeros(max(len(xy), 1), np.int32)
    m = lib().ofront_emission_order(int(w), int(h), int(level), _i(xy), len(xy), int(seed), _i(out))
    return out[:m]


# ---------------------------------------------------------------------------------------------- pure Python
def sm64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    z = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def hash5(a, b, c, d, e):
    return sm64(sm64(sm64(sm64(sm64(a) ^ b) ^ c) ^ d) ^ e)


class Node:
    """QuadTreeNode (quadtree.h:60-150) with the reference's insert and isWindowEmpty; delta = 1."""

    def __init__(self, x, y, w, h, path, depth):
        self.bbox = (x, y, w, h)
        self.path, self.depth = path, depth
        self.children = None   # (xy, xY, Xy, XY)
        self.elem = None       # (pos, content)

    def _child_insert(self, e):
        x, y, w, h = self.bbox
        rel_x = 1 - (x + w - e[0][0]) / w
        rel_y = 1 - (y + h - e[0][1]) / h
        xy, xY, Xy, XY = self.children
        if rel_x < 0.5 and rel_y < 0.5:
            return xy.insert(e)
        if rel_x >= 0.5 and rel_y < 0.5:
            return Xy.insert(e)
        if rel_x < 0.5 and rel_y >= 0.5:
            return xY.insert(e)
        return XY.insert(e)

    def insert(self, e):
        if self.children is None:
            if self.elem is None:
                self.elem = e
                return True
            if math.hypot(self.elem[0][0] - e[0][0], self.elem[0][1] - e[0][1]) < 1:
                return False
            x, y, w, h = self.bbox
            x1, y1, hw, hh = x + w * 0.5, y + h * 0.5, w * 0.5, h * 0.5
            p, d = self.path << 2, self.depth + 1
            self.children = (Node(x, y, hw, hh, p | 0, d), Node(x, y1, hw, hh, p | 1, d),
                             Node(x1, y, hw, hh, p | 2, d), Node(x1, y1, hw, hh, p | 3, d))
            old, self.elem = self.elem, None
            self._child_insert(old)
            return self._child_insert(e)
        return self._child_insert(e)

    @staticmethod
    def _intersects(A, B):
        if A[1] + A[3] <= B[1] or A[1] >= B[1] + B[3] or A[0] + A[2] <= B[0] or A[0] >= B[0] + B[2]:
            return False
        return True

    def is_window_empty(self, win):
        if self.children is None:
            if self.elem is None:
                return True
            px, py = self.elem[0]
            return not (win[0] <= px < win[0] + win[2] and win[1] <= py < win[1] + win[3])
        for ch in self.children:
            if self._intersects(ch.bbox, win) and not ch.is_window_empty(win):
                return False
        return True

    def elements(self):
        if self.children is None:
            return [] if self.elem is None else [self.elem]
        return [e for ch in self.children for e in ch.elements()]


def equi_order(tree, level, seed):
    """EquiIter (quadtree.h:250-329) with the draws replaced: a node popped at depth d emits its subtree's not yet
    emitted element of smallest key H(seed, 0, level, u, v); the nodes of a depth pop in H(seed, 1, level, d, path)
    order, ties by path.  Returns the contents in emission order."""
    key = lambda e: (hash5(seed, 0, level, int(e[0][0]), int(e[0][1])), e[1])
    visited, out = set(), []
    queue = [tree]
    d = 0
    while queue:
        queue.sort(key=lambda nd: (hash5(seed, 1, level, d, nd.path), nd.path))
        nxt = []
        for nd in queue:
            if nd.children is None:
                if nd.elem is not None and nd.elem[1] not in visited:
                    visited.add(nd.elem[1])
                    out.append(nd.elem[1])
                continue
            nxt.extend(nd.children)
            cand = [e for e in nd.elements() if e[1] not in visited]
            if cand:
                e = min(cand, key=key)
                visited.add(e[1])
                out.append(e[1])
        queue, d = nxt, d + 1
    return out


def py_seed(sizes, corners, disp, tree, num_in, flags, R, num_max_points, seed, T, cam, slot, se3_act):
    """addMorePointsToOtherFrame (stereo_frontend.cpp:724-823) line by line.  se3_act(T, x) -> T * x."""
    w0, h0 = sizes[0]
    third = np.float32(1. / 3.)
    tw, th = int(np.float32(w0) * third), int(np.float32(h0) * third)
    ttw, tth = int(np.float32(w0 * 2) * third), int(np.float32(h0 * 2) * third)
    pts, counts = [], []
    f, px, py, b = cam
    for l, (wl, hl) in enumerate(sizes):
        ft = Node(0., 0., float(wl), float(hl), 0, 0)
        for i, (u, v) in enumerate(np.asarray(corners[l]).reshape(-1, 2).tolist()):
            ft.insert(((float(u), float(v)), i))
        pt = Node(0., 0., float(wl), float(hl), 0, 0)
        for k, t in enumerate(tree):
            if t["anchor_level"] == l:
                pt.insert(((t["uvu"][0] / (1 << l), t["uvu"][1] / (1 << l)), -1 - k))
        cap = num_max_points >> l
        num, kept = int(num_in[l]), 0
        xy = np.asarray(corners[l]).reshape(-1, 2)
        for c in equi_order(ft, l, seed):
            u, v = int(xy[c][0]), int(xy[c][1])
            uz, vz = u << l, v << l
            dsp = float(disp[vz, uz]) * (1. / (1 << l)) if uz < w0 and vz < h0 else 0.
            if not dsp > 0:
                continue
            if not (1 <= uz < w0 - 1 and 1 <= vz < h0 - 1):
                continue
            i = 0 if uz < tw else (1 if uz < ttw else 2)
            j = 0 if vz < th else (1 if vz < tth else 2)
            if flags[3 * i + j] == 0:
                continue
            if not pt.is_window_empty((u - R, v - R, 2 * R + 1, 2 * R + 1)):
                continue
            uvu = (float(u), float(v), u - dsp)
            s = float(1 << l)
            u0, v0, r0 = uvu[0] * s, uvu[1] * s, uvu[2] * s
            z = f / ((u0 - r0) / b)
            xc = np.array([(u0 - px) / f * z, (v0 - py) / f * z, z])
            pt.insert(((float(u), float(v)), c))
            dist = math.sqrt(xc[0] * xc[0] + xc[1] * xc[1] + xc[2] * xc[2])
            pts.append((l, (float(u), float(v)), uvu, se3_act(T, xc), -xc / dist))
            num += 1
            kept += 1
            if num > cap:
                break
        counts.append(kept)
    return pts, counts
