"""The pose-graph growth oracle (oracle/graph_oracle.c) against a literal Python transcription of SlamGraph's
computeStrength / addNewEdges / addLoopClosure (slam_graph.cpp:208-254, 424-552), and the closed form of quirk B15 the
device kernel computes against the literal loop.  CPU only."""
from __future__ import annotations

import numpy as np
import pytest

import map_reference as mr
from oracle import graph_pyoracle as gpo


# ------------------------------------------------------------------ literal transcriptions
def literal_strength(vis, new_anchor, track_point, track_center, covis_thr, width, height):
    """computeStrength as written: dicts for the IntTables, the zeroing loop inside the track loop."""
    table, top, bottom, left, right = {}, {}, {}, {}, {}
    half_width, half_height = int(width * 0.5), int(height * 0.5)
    add = lambda d, k: d.__setitem__(k, d.get(k, 0) + 1)
    for a in new_anchor:
        add(table, int(a))
    for t, p in enumerate(track_point):
        for f in vis[p]:
            add(table, f)
            u, v = track_center[t][0], track_center[t][1]
            add(left if u < half_width else right, f)
            add(top if v < half_height else bottom, f)
        for f in list(table):
            if (f in top and top[f] >= covis_thr // 2 and f in bottom and bottom[f] >= covis_thr // 2 and f in left
                    and left[f] >= covis_thr // 2 and f in right and right[f] >= covis_thr // 2):
                continue
            table[f] = 0
    return table


def closed_form_strength(vis, new_anchor, quads, covis_thr):
    """What k_str_closed computes: per vertex, its records in track order; t* = the first after which all four quadrant
    counts reach max(1, covis_thr // 2); strength = records from t* on (0 without t*), or the new-point count when
    there are no tracks.  quads[t] = (left, top) booleans of track t."""
    need = max(1, covis_thr // 2)
    rec = {}
    for t, fs in enumerate(vis):
        for f in fs:
            rec.setdefault(f, []).append(quads[t])
    out = {}
    for a in new_anchor:
        out[int(a)] = out.get(int(a), 0) + 1
    if not vis:
        return out
    for f in set(out) | set(rec):
        r = rec.get(f, [])
        c = [0, 0, 0, 0]
        s = 0
        for i, (l, tp) in enumerate(r):
            c[0 if l else 1] += 1
            c[2 if tp else 3] += 1
            if min(c) >= need:
                s = len(r) - i
                break
        out[f] = s
    return out


def plain_counts(vis, new_anchor):
    out = {}
    for a in new_anchor:
        out[int(a)] = out.get(int(a), 0) + 1
    for fs in vis:
        for f in fs:
            out[f] = out.get(f, 0) + 1
    return out


def literal_insert(lists, v, s, nbr, payload):
    """std::multimap<int, int>::insert (after the equal keys) on a list stored in rbegin order."""
    mm = lists[v][::-1]
    at = len(mm)
    while at > 0 and mm[at - 1][0] > s:
        at -= 1
    mm.insert(at, (s, nbr, payload))
    lists[v] = mm[::-1]


# ------------------------------------------------------------------ random cases
def _random_case(rng, V, n_track, n_new, width=640, height=480):
    vis = [sorted(rng.choice(V, size=int(rng.integers(1, min(V, 6) + 1)), replace=False).tolist()) for _ in range(n_track)]
    uv = np.stack([rng.uniform(0, width, n_track), rng.uniform(0, height, n_track), np.zeros(n_track)], 1)
    return vis, uv, rng.integers(0, V, n_new)


def _tables_equal(lit, inn, st):
    got = {int(f): int(st[f]) for f in np.flatnonzero(inn)}
    assert got == lit


@pytest.mark.parametrize("seed", range(40))
def test_oracle_strength_equals_literal(seed):
    rng = np.random.default_rng(seed)
    V = int(rng.integers(2, 12))
    n_track, n_new = int(rng.integers(0, 30)), int(rng.integers(0, 6))
    vis, uv, na = _random_case(rng, V, n_track, n_new)
    thr = int(rng.integers(1, 9))
    m = dict(poses=np.zeros((V, 7)), vis_ptr=np.concatenate([[0], np.cumsum([len(x) for x in vis])]).astype(np.int32),
             vis_pose=np.array([f for fs in vis for f in fs], np.int32))
    inn, st = gpo.compute_strength(m, na, np.arange(n_track), uv, thr, 640, 480)
    _tables_equal(literal_strength(vis, na, list(range(n_track)), uv, thr, 640, 480), inn, st)


def _closed_vs_literal(rng, cases, V_range=(1, 8), track_range=(0, 40), force=None):
    bad = 0
    for _ in range(cases):
        V = int(rng.integers(*V_range))
        n_track, n_new = int(rng.integers(*track_range)), int(rng.integers(0, 5))
        vis, uv, na = _random_case(rng, V, n_track, n_new)
        thr = int(rng.integers(1, 10)) if force is None else force
        lit = literal_strength(vis, na, list(range(n_track)), uv, thr, 640, 480)
        quads = [(u < 320, v < 240) for u, v, _ in uv]
        got = closed_form_strength(vis, na, quads, thr)
        bad += got != lit
    return bad


def test_b15_closed_form_equals_literal_loop():
    rng = np.random.default_rng(1)
    assert _closed_vs_literal(rng, 3000) == 0
    for thr in (1, 2, 3, 4, 7, 8):                     # covis_thr = 1 (need = 1) and odd / even thresholds
        assert _closed_vs_literal(rng, 300, force=thr) == 0
    assert _closed_vs_literal(rng, 300, track_range=(0, 1)) == 0   # n_track = 0: the new-point counts stay


def test_b15_edge_cases():
    # frames seen only through new points: their counts vanish with the first track
    vis, na = [[0]], [1, 1, 2]
    uv = np.array([[10., 10., 0.]])
    assert literal_strength(vis, na, [0], uv, 1, 640, 480) == {0: 0, 1: 0, 2: 0}
    assert closed_form_strength(vis, na, [(True, True)], 1) == {0: 0, 1: 0, 2: 0}
    # without tracks they stay
    assert literal_strength([], na, [], np.zeros((0, 3)), 4, 640, 480) == {1: 2, 2: 1}
    assert closed_form_strength([], na, [], 4) == {1: 2, 2: 1}
    # a frame that qualifies at the last track: strength 1
    vis = [[3], [3], [3], [3]]
    uv = np.array([[10., 10., 0.], [10., 10., 0.], [10., 10., 0.], [600., 400., 0.]])
    quads = [(u < 320, v < 240) for u, v, _ in uv]
    assert literal_strength(vis, [], list(range(4)), uv, 2, 640, 480) == {3: 1}
    assert closed_form_strength(vis, [], quads, 2) == {3: 1}
    # the centre line goes right / bottom: u = half_width is not left
    uv2 = np.array([[320., 240., 0.]] * 4)
    assert literal_strength(vis, [], list(range(4)), uv2, 1, 640, 480) == {3: 0}


def test_plain_counts_fail_the_literal_loop():
    """The closed form is needed: counting every observation does not reproduce the reference."""
    rng = np.random.default_rng(5)
    bad = 0
    for _ in range(300):
        vis, uv, na = _random_case(rng, 6, int(rng.integers(1, 30)), 2)
        bad += plain_counts(vis, na) != literal_strength(vis, na, list(range(len(vis))), uv, 4, 640, 480)
    assert bad > 250


def _random_graph(rng, V, density=0.4):
    lists = [[] for _ in range(V)]
    for a in range(V):
        for b in range(a + 1, V):
            if rng.random() < density:
                s = int(rng.integers(1, 6))
                literal_insert(lists, a, s, b, None)
                literal_insert(lists, b, s, a, None)
    return lists


def _graph_arrays(lists, rng):
    ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    ids = np.array([e[1] for x in lists for e in x], np.int32)
    st = np.array([e[0] for x in lists for e in x], np.int32)
    n = len(ids)
    return dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=st, nbr_T=rng.normal(size=(n, 7)), nbr_Lambda=rng.normal(size=(n, 36)))


def _small_map(rng, V, Np):
    poses = np.concatenate([np.tile([0, 0, 0, 1.0], (V, 1)), rng.normal(0, 0.3, (V, 3))], 1)
    vis = [sorted(rng.choice(V, size=int(rng.integers(1, V + 1)), replace=False).tolist()) for _ in range(Np)]
    return dict(poses=poses, point_anchor=np.array([v[0] for v in vis], np.int32),
                xyz_anchor=np.stack([rng.uniform(-1, 1, Np), rng.uniform(-1, 1, Np), rng.uniform(3, 8, Np)], 1),
                vis_ptr=np.concatenate([[0], np.cumsum([len(x) for x in vis])]).astype(np.int32),
                vis_pose=np.array([f for x in vis for f in x], np.int32))


@pytest.mark.parametrize("seed", range(20))
def test_oracle_insertion_equals_multimap(seed):
    """addNewEdges / addLoopClosure on random small graphs: list order (with equal strengths) and constraints."""
    rng = np.random.default_rng(100 + seed)
    V = int(rng.integers(3, 10))
    lists = _random_graph(rng, V)
    g = _graph_arrays(lists, rng)
    m = _small_map(rng, V, 40)
    # new edges between vertices that are not yet neighbours, some of equal strength
    free = [(a, b) for a in range(V) for b in range(a + 1, V) if all(e[1] != b for e in lists[a])]
    rng.shuffle(free)
    pairs = free[: int(rng.integers(0, len(free) + 1))]
    v1 = np.array([p[0] if rng.random() < 0.5 else p[1] for p in pairs], np.int32)
    v2 = np.array([p[1] if x == p[0] else p[0] for p, x in zip(pairs, v1)], np.int32)
    s = rng.integers(1, 4, len(pairs)).astype(np.int32)
    moved = int(rng.integers(-1, V))
    Tm = np.concatenate([[0, 0, 0, 1.0], rng.normal(0, 0.3, 3)])
    got = gpo.add_edges(g, m, v1, v2, s, moved, Tm)
    # literal: the lists with payload = (T, Lambda) per entry
    idx = 0
    lit = []
    for v in range(V):
        lit.append([(e[0], e[1], (g["nbr_T"][idx + i], g["nbr_Lambda"][idx + i])) for i, e in enumerate(lists[v])])
        idx += len(lists[v])
    poses = m["poses"].copy()
    if moved >= 0:
        poses[moved] = Tm
    fptr, fpt = gpo.feature_tables(m)
    for k in range(len(pairs)):
        T12, Lam, _, _, _ = mr.compute_constraint(poses, fptr, fpt, m["point_anchor"], m["xyz_anchor"], int(v1[k]), int(v2[k]))
        T12, Lam = np.asarray(T12, np.float64), np.asarray(Lam, np.float64).reshape(36)
        literal_insert(lit, v1[k], int(s[k]), int(v2[k]), (np.asarray(mr._se3_inv(T12), np.float64), Lam))
        literal_insert(lit, v2[k], int(s[k]), int(v1[k]), (T12, Lam))
    assert np.array_equal(got["nbr_ptr"], np.concatenate([[0], np.cumsum([len(x) for x in lit])]))
    assert np.array_equal(got["nbr_id"], [e[1] for x in lit for e in x])
    assert np.array_equal(got["nbr_strength"], [e[0] for x in lit for e in x])
    T = np.array([e[2][0] for x in lit for e in x]).reshape(-1, 7)
    L = np.array([e[2][1] for x in lit for e in x]).reshape(-1, 36)
    assert np.allclose(got["nbr_T"], T, rtol=1e-12, atol=1e-12)
    assert np.allclose(got["nbr_Lambda"], L, rtol=1e-10, atol=1e-9)


def test_local_edges_take_the_table_in_vertex_order():
    v1, v2, s = gpo.local_edges([[0, 3], [2, 9], [5, 4], [7, 1]], 4, 8)
    assert v1.tolist() == [2, 5] and v2.tolist() == [8, 8] and s.tolist() == [9, 4]
