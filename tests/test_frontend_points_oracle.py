"""CPU tests of oracle/frontend_oracle.c (the tracked frame's bookkeeping of StereoFrontend): its budget,
processMatchedPoints and seeding equal the pure-Python restatement of oracle/frontend_pyoracle.py exactly (ints, flags,
order, doubles).  The seeding is compared with the reference's adaptive quadtree built literally, which pins the claim
that the regular midpoint tree has the same emission order and window tests."""
import math

import numpy as np
import pytest

from oracle import frontend_pyoracle as fp
from oracle import loop_pyoracle as lo

# (level sizes, cam (f, px, py, b) of level 0)
SHAPES = {
    "640x480_2": ([(640, 480), (320, 240)], (500., 319.5, 239.5, 0.12)),
    "newcollege": ([(512, 384), (256, 192), (128, 96)], (389.956085, 254.903519, 201.899490, 0.110014)),
    "1241x376": ([(1241, 376), (620, 188)], (718.856, 607.1928, 185.2157, 0.537)),
}
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


def _corners(rng, w, h, n, dup=5):
    xy = np.stack([rng.integers(0, w, n), rng.integers(0, h, n)], 1).astype(np.int32)
    if dup and n > dup:
        xy[-dup:] = xy[:dup]          # corners at an earlier corner's position
    return xy


def _frame(rng, sizes, n0, disp_frac=0.8):
    w0, h0 = sizes[0]
    disp = rng.uniform(0.5, 40, (h0, w0)).astype(np.float32)
    disp[rng.random((h0, w0)) > disp_frac] = 0
    corners = [_corners(rng, w, h, max(n0 >> (2 * l), 8)) for l, (w, h) in enumerate(sizes)]
    return disp, corners


def _tree(rng, sizes, n):
    t = np.zeros(n, fp.TRACKED_DTYPE)
    for k in range(n):
        l = int(rng.integers(0, len(sizes)))
        w, h = sizes[l]
        t[k]["anchor_level"] = l
        t[k]["uvu"] = (int(rng.integers(0, w)) << l, int(rng.integers(0, h)) << l, 0.)
    return t


def _py_seed(sizes, corners, disp, tree, num_in, flags, R, nmax, seed, T, cam, slot=3):
    act = lambda T_, x: lo.se3("oloop_se3_act", T_, x)
    return fp.py_seed(sizes, corners, disp, tree, num_in, flags, R, nmax, seed, T, cam, slot, act)


def _assert_seed_equal(c, py):
    pts, rows, counts = c
    ppts, pcounts = py
    assert list(counts) == list(pcounts)
    assert len(pts) == len(ppts)
    for p, (l, uv, uvu, xyz, nrm) in zip(pts, ppts):
        assert p["level"] == l
        assert tuple(p["uv_pyr"]) == uv
        assert tuple(p["uvu_pyr"]) == uvu
        assert np.array_equal(p["xyz"], xyz)
        assert np.array_equal(p["normal"], nrm)
    assert np.array_equal(rows["xyz_anchor"], pts["xyz"]) and np.array_equal(rows["anchor_obs_pyr"], pts["uv_pyr"])
    assert np.array_equal(rows["anchor_level"], pts["level"])


@pytest.mark.parametrize("shape", list(SHAPES))
def test_emission_order_equals_adaptive_quadtree(shape):
    sizes, _ = SHAPES[shape]
    rng = np.random.default_rng(1)
    for l, (w, h) in enumerate(sizes):
        xy = _corners(rng, w, h, 600 >> l)
        tree = fp.Node(0., 0., float(w), float(h), 0, 0)
        for i, (u, v) in enumerate(xy.tolist()):
            tree.insert(((float(u), float(v)), i))
        for seed in (0, 7):
            assert fp.c_emission_order(w, h, l, xy, seed).tolist() == fp.equi_order(tree, l, seed)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("fresh", [1, 0])
def test_seed_equals_literal_restatement(shape, fresh):
    sizes, cam = SHAPES[shape]
    rng = np.random.default_rng(2 + fresh)
    disp, corners = _frame(rng, sizes, 1500)
    tree = _tree(rng, sizes, 0 if fresh else 120)
    num_in = [0] * len(sizes) if fresh else [int((tree["anchor_level"] == l).sum()) for l in range(len(sizes))]
    flags = np.ones(9, np.int32) if fresh else np.array([1, 0, 1, 1, 1, 0, 1, 1, 1], np.int32)
    T = np.array([0.01, -0.02, 0.005, 1, 0.1, -0.05, 0.2])
    T[:4] /= np.linalg.norm(T[:4])
    for nmax in (300, 40):
        c = fp.c_seed(sizes, corners, disp, tree, num_in, flags, 2, nmax, 5, T, cam, 3)
        _assert_seed_equal(c, _py_seed(sizes, corners, disp, tree, num_in, flags, 2, nmax, 5, T, cam))
        assert all(k <= (nmax >> l) + 1 for l, k in enumerate(c[2]))


def test_seed_cap_when_num_points_in_exceeds_it():
    sizes, cam = SHAPES["640x480_2"]
    rng = np.random.default_rng(4)
    disp, corners = _frame(rng, sizes, 800)
    flags = np.ones(9, np.int32)
    for num_in in ([500, 10], [301, 151], [300, 0], [0, 0]):
        c = fp.c_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), num_in, flags, 2, 300, 0, IDENT, cam, 0)
        _assert_seed_equal(c, _py_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), num_in, flags, 2, 300, 0,
                                       IDENT, cam))
        # min(taken, max(1, cap + 1 - num_in))
        free = fp.c_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), [0, 0], flags, 2, 10 ** 6, 0, IDENT, cam, 0)
        for l in range(2):
            assert c[2][l] == min(free[2][l], max(1, (300 >> l) + 1 - num_in[l]))


@pytest.mark.parametrize("R", [0, 1, 2, 3])
def test_window_edges(R):
    """A tree point at exactly x-R is inside the window, one at x+R+1 is not (cv::Rect_<double>::contains)."""
    sizes, cam = [(64, 48)], (50., 31.5, 23.5, 0.1)
    disp = np.full((48, 64), 5, np.float32)
    corners = [np.array([[30, 20]], np.int32)]
    flags = np.ones(9, np.int32)
    for dx, dy, inside in ((-R, 0, True), (R, R, True), (R + 1, 0, False), (0, -R - 1, False), (-R, -R, True)):
        t = np.zeros(1, fp.TRACKED_DTYPE)
        t[0]["uvu"] = (30 + dx, 20 + dy, 0)
        c = fp.c_seed(sizes, corners, disp, t, [1], flags, R, 300, 0, IDENT, cam, 0)
        py = _py_seed(sizes, corners, disp, t, [1], flags, R, 300, 0, IDENT, cam)
        _assert_seed_equal(c, py)
        assert c[2][0] == (0 if inside else 1)


def test_seed_all_flags_off_and_border_and_disparity():
    sizes, cam = SHAPES["640x480_2"]
    rng = np.random.default_rng(5)
    disp, corners = _frame(rng, sizes, 400)
    c = fp.c_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), [0, 0], np.zeros(9, np.int32), 2, 300, 0, IDENT,
                  cam, 0)
    assert len(c[0]) == 0
    # corners on the 1-px border and on disparity <= 0 are never seeded
    corners = [np.array([[0, 5], [639, 7], [5, 0], [9, 479], [100, 100], [200, 200]], np.int32), np.zeros((0, 2), np.int32)]
    disp = np.full((480, 640), 3, np.float32)
    disp[100, 100] = 0
    disp[200, 200] = -1
    c = fp.c_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), [0, 0], np.ones(9, np.int32), 2, 300, 0, IDENT,
                  cam, 0)
    assert len(c[0]) == 0


def _py_process(res, lvl, n_new, T, cam, w0, h0, max_err=np.float32(2), min_num=25):
    """stereo_frontend.cpp:856-969 line by line."""
    half_w, half_h = int(w0 * 0.5), int(h0 * 0.5)
    third = np.float32(1. / 3.)
    tw, th = int(np.float32(w0) * third), int(np.float32(h0) * third)
    ttw, tth = int(np.float32(w0 * 2) * third), int(np.float32(h0 * 2) * third)
    g2, g3, nm = np.zeros((2, 2), int), np.zeros((3, 3), int), [0] * 4
    out, s, cnt = [], 0., 0
    for i, r in enumerate(res):
        if not r["matched"]:
            continue
        pred = lo.map_uvu(cam, T, r["xyz_actkey"])
        d = r["obs"] - pred
        factor = 1 << int(lvl[i])
        thr = float(np.float32(max_err * np.float32(factor)))
        if not (abs(d[0]) < thr and abs(d[1]) < thr and abs(d[2]) < 3. * float(max_err)):
            continue
        uvu = r["obs"]
        g2[0 if uvu[0] < half_w else 1, 0 if uvu[1] < half_h else 1] += 1
        g3[0 if uvu[0] < tw else (1 if uvu[0] < ttw else 2), 0 if uvu[1] < th else (1 if uvu[1] < tth else 2)] += 1
        nm[int(lvl[i])] += 1
        X = r["xyz_actkey"]
        sc = float(factor)
        cu, cv = (cam[0] * (X[0] / X[2]) + cam[1]) / sc, (cam[0] * (X[1] / X[2]) + cam[2]) / sc
        du, dv = uvu[0] / sc - cu, uvu[1] / sc - cv
        s += math.sqrt(du * du + dv * dv)
        cnt += 1
        out.append((i, int(i < n_new), int(lvl[i]), tuple(uvu)))
    av = s / cnt if cnt else float("nan")
    return out, g2, g3, nm, av, (g3 <= min_num).astype(np.int32).reshape(-1)


def _results(rng, n, cam, w0, h0, noise=1.5):
    res = np.zeros(n, fp.MATCH_RESULT_DTYPE)
    lvl = rng.integers(0, 3, n).astype(np.int32)
    f, px, py, b = cam
    for i in range(n):
        X = np.array([rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(2, 12)])
        res[i]["xyz_actkey"] = X
        u, v = f * X[0] / X[2] + px, f * X[1] / X[2] + py
        s = 1 << int(lvl[i])
        uq, vq = float(int(max(0, min(w0 - 1, u + rng.normal(0, noise))) / s) * s), \
            float(int(max(0, min(h0 - 1, v + rng.normal(0, noise))) / s) * s)
        res[i]["obs"] = (uq, vq, uq - f * b / X[2] + rng.normal(0, noise))
        res[i]["matched"] = int(rng.random() < 0.8)
    return res, lvl


@pytest.mark.parametrize("shape", list(SHAPES))
def test_process_equals_transcription(shape):
    sizes, cam = SHAPES[shape]
    w0, h0 = sizes[0]
    rng = np.random.default_rng(6)
    res, lvl = _results(rng, 900, cam, w0, h0)
    T = np.array([0.002, -0.001, 0.0005, 1, 0.01, 0.0, -0.02])
    T[:4] /= np.linalg.norm(T[:4])
    for n_new in (0, 300, 900):
        out, st, flags = fp.c_process(res, lvl, n_new, T, cam, w0, h0)
        want, g2, g3, nm, av, wflags = _py_process(res, lvl, n_new, T, cam, w0, h0)
        assert [(int(o["index"]), int(o["is_new"]), int(o["anchor_level"]), tuple(o["uvu"])) for o in out] == want
        d = fp.stats_dict(st)
        assert np.array_equal(d["grid2x2"], g2) and np.array_equal(d["grid3x3"], g3)
        assert d["num_matched_points"][:3] == nm[:3]
        assert d["av_track_length"] == av
        assert d["num_new"] == sum(w[1] for w in want)
        assert np.array_equal(flags, wflags)
        # shallWeDropNewKeyframe
        featureless = int((g2 < 15).sum())
        assert fp.c_drop(st, T) == int(featureless > 2 or np.linalg.norm(T[4:]) > np.float32(0.75) or av > 75.)


def test_process_nothing_gated_gives_nan():
    sizes, cam = SHAPES["640x480_2"]
    rng = np.random.default_rng(7)
    res, lvl = _results(rng, 50, cam, 640, 480)
    res["matched"] = 0
    out, st, flags = fp.c_process(res, lvl, 10, IDENT, cam, 640, 480)
    assert len(out) == 0 and math.isnan(st.av_track_length)
    assert flags.tolist() == [1] * 9
    assert fp.c_drop(st, IDENT) == 1   # four featureless quadrants


def _py_budget(matched, ends, nmax):
    """stereo_frontend.cpp:989-1050: group 0, neighbours while 2 |obs| < nmax, then the neighbourhood's points."""
    m = np.array(matched)
    starts = [0] + list(ends[:-1])
    total = int(m[:ends[0]].sum())
    g = 1
    while g < len(ends) - 1 and 2 * total < nmax:
        total += int(m[starts[g]:ends[g]].sum())
        g += 1
    for k in range(g, len(ends) - 1):
        m[starts[k]:ends[k]] = 0
    num_new = total
    return m, num_new, total + int(m[starts[-1]:].sum())


@pytest.mark.parametrize("nmax", [0, 1, 40, 120, 10 ** 6])
def test_budget_equals_transcription(nmax):
    rng = np.random.default_rng(8)
    sizes = [30, 25, 0, 40, 35, 50]
    ends = np.cumsum(sizes).astype(np.int32)
    res = np.zeros(ends[-1], fp.MATCH_RESULT_DTYPE)
    res["matched"] = rng.random(ends[-1]) < 0.7
    r, a, b = fp.c_budget(res, ends, nmax)
    m, pa, pb = _py_budget(res["matched"], ends, nmax)
    assert np.array_equal(r["matched"], m) and (a, b) == (pa, pb)
