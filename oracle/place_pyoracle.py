"""ctypes binding of the place-recognition oracle (oracle/place_oracle.c, part of liboracle.so).

TEST INFRASTRUCTURE ONLY, like pyoracle.py (whose build of liboracle.so it shares)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

c_fp = C.POINTER(C.c_float)
c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)
_LIB = None


class OPlResult(C.Structure):
    _fields_ = [("best_keyframe_id", C.c_int), ("best_score", C.c_float), ("num_matches", C.c_int),
                ("num_inliers", C.c_int), ("loop_found", C.c_int), ("T_query_from_loop", C.c_double * 7),
                ("number_of_words", C.c_int), ("best_hypothesis", C.c_int), ("num_hypotheses", C.c_int)]


def lib():
    global _LIB
    if _LIB is None:
        L = pyoracle.lib()
        L.opl_create.argtypes = [C.c_int, c_fp, c_dp]
        L.opl_create.restype = C.c_void_p
        L.opl_destroy.argtypes = [C.c_void_p]
        L.opl_destroy.restype = None
        L.opl_num_places.argtypes = [C.c_void_p]
        L.opl_add_location.argtypes = [C.c_void_p, C.c_int, C.c_int, c_fp, c_dp, C.c_int, C.c_int, c_ip, C.c_int,
                                       C.c_double, C.c_ulonglong, C.POINTER(OPlResult), c_ip, c_ip, c_fp, c_ip, c_ip,
                                       c_fp, c_ip, c_ip, c_ip, c_ip]
        L.opl_sqdist.argtypes = [c_fp, c_fp]
        L.opl_sqdist.restype = C.c_float
        L.opl_nn.argtypes = [C.c_int, c_fp, C.c_int, c_fp, c_ip, c_fp]
        L.opl_nn.restype = None
        L.opl_kabsch.argtypes = [c_dp, c_dp, c_dp, c_dp]
        L.opl_kabsch.restype = None
        L.opl_splitmix_next.argtypes = [C.POINTER(C.c_ulonglong)]
        L.opl_splitmix_next.restype = C.c_ulonglong
        L.opl_draw_triple.argtypes = [C.c_ulonglong, C.c_int, C.c_int, c_ip, c_ip]
        _LIB = L
    return _LIB


def _f(a):
    return a.ctypes.data_as(c_fp)


def _d(a):
    return a.ctypes.data_as(c_dp)


def _i(a):
    return a.ctypes.data_as(c_ip)


def nn(query, train):
    q = np.ascontiguousarray(query, np.float32).reshape(-1, 64)
    t = np.ascontiguousarray(train, np.float32).reshape(-1, 64)
    idx, d = np.zeros(max(len(q), 1), np.int32), np.zeros(max(len(q), 1), np.float32)
    lib().opl_nn(len(q), _f(q), len(t), _f(t), _i(idx), _f(d))
    return idx[:len(q)], d[:len(q)]


def kabsch(p0, p1):
    p0 = np.ascontiguousarray(p0, np.float64).reshape(3, 3)
    p1 = np.ascontiguousarray(p1, np.float64).reshape(3, 3)
    R, t = np.zeros(9), np.zeros(3)
    lib().opl_kabsch(_d(p0), _d(p1), _d(R), _d(t))
    return R.reshape(3, 3), t


def splitmix(state, count):
    st = C.c_ulonglong(state)
    return [lib().opl_splitmix_next(C.byref(st)) for _ in range(count)]


def draw_triple(seed, h, train_idx):
    ti = np.ascontiguousarray(train_idx, np.int32)
    tri = np.zeros(3, np.int32)
    draws = lib().opl_draw_triple(int(seed) & (2 ** 64 - 1), h, len(ti), _i(ti), _i(tri))
    return draws, tri


class PlaceOracle:
    """The oracle's database; add_location returns the result and every intermediate."""

    def __init__(self, words, cam):
        self.words = np.ascontiguousarray(words, np.float32).reshape(-1, 64)
        cam = np.ascontiguousarray(cam, np.float64)
        self._db = lib().opl_create(len(self.words), _f(self.words), _d(cam))
        if not self._db:
            raise ValueError("opl_create refused its input")

    def close(self):
        if self._db:
            lib().opl_destroy(self._db)
            self._db = None

    def __del__(self):
        self.close()

    @property
    def num_places(self):
        return lib().opl_num_places(self._db)

    def add_location(self, keyframe_id, desc, uvu, do_loop_detection=True, exclude=(), num_ransac=100, pixel_thr=2.5,
                     seed=0):
        desc = np.ascontiguousarray(desc, np.float32).reshape(-1, 64)
        uvu = np.ascontiguousarray(uvu, np.float64).reshape(-1, 3)
        n, L, H = len(desc), self.num_places, max(int(num_ransac), 0)
        ex = np.ascontiguousarray(list(exclude), np.int32)
        n1 = max(n, 1)
        word, sid, sval, ns = np.zeros(n1, np.int32), np.zeros(L + 1, np.int32), np.zeros(L + 1, np.float32), C.c_int()
        tidx, dist = np.zeros(n1, np.int32), np.zeros(n1, np.float32)
        tri, hinl = np.zeros((max(H, 1), 3), np.int32), np.zeros(max(H, 1), np.int32)
        iq, it = np.zeros(n1, np.int32), np.zeros(n1, np.int32)
        r = OPlResult()
        rc = lib().opl_add_location(self._db, int(keyframe_id), n, _f(desc), _d(uvu), int(bool(do_loop_detection)),
                                    len(ex), _i(ex), int(num_ransac), float(pixel_thr), int(seed) & (2 ** 64 - 1),
                                    C.byref(r), _i(word), _i(sid), _f(sval), C.byref(ns), _i(tidx), _f(dist), _i(tri),
                                    _i(hinl), _i(iq), _i(it))
        if rc != 0:
            raise ValueError("opl_add_location refused its input")
        nm, ni, nh = r.num_matches, r.num_inliers, r.num_hypotheses
        return dict(best_keyframe_id=r.best_keyframe_id, best_score=r.best_score, num_matches=nm, num_inliers=ni,
                    loop_found=bool(r.loop_found), T_query_from_loop=np.array(r.T_query_from_loop[:]),
                    number_of_words=r.number_of_words, best_hypothesis=r.best_hypothesis,
                    words=word[:n].copy(), score_ids=sid[:ns.value].copy(), scores=sval[:ns.value].copy(),
                    train_idx=tidx[:nm].copy(), dist=dist[:nm].copy(), hyp_triple=tri[:nh].copy(),
                    hyp_inliers=hinl[:nh].copy(), inlier_query=iq[:ni].copy(), inlier_train=it[:ni].copy())
