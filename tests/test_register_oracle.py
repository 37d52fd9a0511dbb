"""CPU tests of oracle/register_oracle.c (Backend::localRegisterFrame): its neighbourhood, candidates and stats table
equal a literal Python transcription of backend.cpp:433-449, 472-546, 615-722 and slam_graph.cpp:105-140 on hand-made
maps and on the rendered revisit, and on the revisit the registration moves root towards its true pose relative to
keyframe 0."""
import collections
import functools

import numpy as np

from scavislam_b200 import synth_loop as sl

I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])


def _run_oracle(sc, covis_thr, slot=None):
    from oracle import register_pyoracle as ro
    V = len(sc["map"]["poses"])
    slot = np.arange(V, dtype=np.int32) if slot is None else slot
    rf = sc["frames"][sc["root"]]
    return ro.local_register_frame(sc["map"], sc["nbr_ptr"], sc["nbr_id"], sc["levels"], rf["pyr"], rf["disp"],
                                   sc["root_features"], [sc["frames"][v]["pyr"] for v in range(V)], sc["cam"], covis_thr,
                                   sc["root"], sc["window"], slot)


@functools.lru_cache(maxsize=1)
def _scene():
    from oracle import pyoracle
    sc = sl.make_register_scene(pyoracle)
    return sc, _run_oracle(sc, 20)


# ------------------------------------------------------------------ the transcription

def _direct_neighbors_of(nbr_ptr, nbr_id, root):                       # backend.cpp:433-449
    return {root} | {int(j) for j in nbr_id[nbr_ptr[root]:nbr_ptr[root + 1]]}


def _frames_in_neighborhood(nbr_ptr, nbr_id, root, size, window):      # slam_graph.cpp:105-140
    q, s = collections.deque([root]), set()
    while q and len(s) < size:
        v = q.popleft()
        if v in s:                                                     # Avoid cycles!
            continue
        if v not in window:
            continue
        s.add(v)
        for j in nbr_id[nbr_ptr[v]:nbr_ptr[v + 1]]:                    # rbegin .. rend: strongest first
            q.append(int(j))
    return s


def _observers(m, p):
    return [int(v) for v in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]]]


def _points_visible_in_root(m, larger, direct, window, root, levels, slot):   # backend.cpp:472-546, ascending points
    from oracle import loop_pyoracle as lo
    point_set = set()
    for k in larger:
        if k in direct:
            continue
        point_set |= {p for p in range(len(m["point_anchor"])) if k in _observers(m, p)}
    cand, vertex_table = [], {root}
    for p in sorted(point_set):
        a = int(m["point_anchor"][p])
        if a not in window:
            continue
        ia = m["vis_ptr"][p] + _observers(m, p).index(a)
        l = m["feat_level"][ia]
        w, h, f, px, py = levels[l]
        x = lo.se3("oloop_se3_act", lo.se3("oloop_se3_mul", m["poses"][root], lo.se3("oloop_se3_inv", m["poses"][a])),
                   m["xyz_anchor"][p])
        u, v = f * (x[0] / x[2]) + px, f * (x[1] / x[2]) + py
        if not (0 <= int(u) < w and 0 <= int(v) < h):                  # isInFrame(uv.cast<int>(), 0)
            continue
        cand.append((p, slot[a], l, m["feat_center"][ia][0] / (1 << l), m["feat_center"][ia][1] / (1 << l)))
        vertex_table.add(a)
    return cand, vertex_table


def _keyframes_to_register(m, direct, vertex_table, T, res2, cand, cand_point, cam, levels, covis_thr):   # :615-722
    from oracle import loop_pyoracle as lo
    W, H = levels[0][:2]
    table, tracks = {}, []
    for i in np.flatnonzero(res2["matched"]):
        uvu = res2["obs"][i]
        d = uvu - lo.map_uvu(cam, T, res2["xyz_actkey"][i])
        factor = 1 << cand["anchor_level"][i]
        if not (abs(d[0]) < 2.0 * factor and abs(d[1]) < 2.0 * factor and abs(d[2]) < 2.0 * 3):
            continue
        p = int(cand_point[i])
        tracks.append(p)
        for pose_id in vertex_table:
            if pose_id in direct or pose_id not in _observers(m, p):
                continue
            st = table.setdefault(pose_id, dict(points=[], num_left=0, num_right=0, num_upper=0, num_lower=0))
            st["points"].append(p)
            if uvu[0] > W * 0.5:
                st["num_left"] += 1
            else:
                st["num_right"] += 1
            if uvu[1] > H * 0.5:
                st["num_lower"] += 1
            else:
                st["num_upper"] += 1
    rows, committed = [], set()
    for v in sorted(table):
        st = table[v]
        q = (len(st["points"]) >= covis_thr and st["num_left"] >= covis_thr // 2 and st["num_right"] >= covis_thr // 2
             and st["num_upper"] >= covis_thr // 2 and st["num_lower"] >= covis_thr // 2)
        rows.append((v, len(st["points"]), st["num_left"], st["num_right"], st["num_upper"], st["num_lower"], int(q)))
        if q:
            committed |= set(st["points"])
    return rows, tracks, committed


def _assert_equals_transcription(sc, covis_thr, res, inter, slot=None):
    m = sc["map"]
    V = len(m["poses"])
    slot = np.arange(V, dtype=np.int32) if slot is None else slot
    window = set(np.asarray(sc["window"]).tolist())
    direct = _direct_neighbors_of(sc["nbr_ptr"], sc["nbr_id"], sc["root"])
    larger = _frames_in_neighborhood(sc["nbr_ptr"], sc["nbr_id"], sc["root"], len(direct) + 40, window)
    assert set(inter["direct"].tolist()) == direct and res["n_direct"] == len(direct)
    assert set(inter["neighborhood"].tolist()) == larger and res["n_neighborhood"] == len(larger)
    cand, vertex_table = _points_visible_in_root(m, larger, direct, window, sc["root"], sc["levels"], slot)
    c = inter["cand"]
    np.testing.assert_array_equal(inter["cand_point"], [w[0] for w in cand])
    np.testing.assert_array_equal(c["keyframe"], [w[1] for w in cand])
    np.testing.assert_array_equal(c["anchor_level"], [w[2] for w in cand])
    np.testing.assert_array_equal(c["anchor_obs_pyr"].reshape(-1, 2), np.array([[w[3], w[4]] for w in cand]).reshape(-1, 2))
    assert res["n_candidates"] == len(cand)
    if res["stage"] in (0, 4):
        rows, tracks, committed = _keyframes_to_register(m, direct, vertex_table, res["T_newroot_from_oldroot"], inter["res2"],
                                                         c, inter["cand_point"], sc["cam"], sc["levels"], covis_thr)
        assert [tuple(int(x) for x in r) for r in inter["stats"]] == rows
        np.testing.assert_array_equal(inter["tracks"]["point"], tracks)
        np.testing.assert_array_equal(inter["tracks"]["committed"], [int(p in committed) for p in tracks])
        assert res["n_neighbors"] == sum(r[-1] for r in rows) and res["n_committed"] == len(committed)
        assert res["stage"] == (0 if res["n_neighbors"] else 4)
    return direct, larger, cand


def test_scene_equals_the_transcription():
    sc, (res, inter, grown) = _scene()
    assert res["registered"] == 1 and res["stage"] == 0
    direct, larger, cand = _assert_equals_transcription(sc, 20, res, inter)
    assert direct == {6, 7, 8} and larger == set(range(9))
    anchors = {int(sc["map"]["point_anchor"][w[0]]) for w in cand}
    assert {0, 1} <= anchors                                  # root sees the points of keyframes 0 and 1
    assert {0, 1} <= {int(r["vertex"]) for r in inter["stats"] if r["qualified"]}


def test_registration_moves_root_towards_its_true_pose():
    sc, (res, _, grown) = _scene()
    T, P = sc["true_T"], sc["map"]["poses"]
    r = sc["root"]
    truth = sl.mul(T[r], sl.inv(T[0]))
    ang = lambda A: np.rad2deg(2 * np.arccos(min(1.0, abs(A[3]))))
    before = sl.mul(sl.mul(P[r], sl.inv(P[0])), sl.inv(truth))
    after = sl.mul(sl.mul(res["T_newroot_from_w"], sl.inv(P[0])), sl.inv(truth))
    assert np.linalg.norm(before[4:]) > 0.02 and ang(before) > 0.5
    assert np.linalg.norm(after[4:]) < 0.25 * np.linalg.norm(before[4:]) and ang(after) < 0.25 * ang(before)
    # the grown map: root observes each committed point once, its pose is the stored one
    assert grown is not None and len(grown["vis_pose"]) > len(sc["map"]["vis_pose"])
    np.testing.assert_array_equal(grown["poses"], P)


def _blank(levels):
    pyr = [np.zeros((l[1], l[0]), np.uint8) for l in levels]
    feats = [(np.zeros((0, 2), np.int32), np.zeros(0, np.int32)) for _ in levels]
    return dict(pyr=pyr, disp=np.zeros((levels[0][1], levels[0][0]), np.float32)), feats


def _hand_made(V, points, nbr, window, root=0):
    """Vertices at the identity; points = [(anchor, observers, (u, v))] at 5 m in front of the camera, level 0;
    nbr[v] = the neighbour list, strongest first."""
    levels = sl.levels()
    w, h, f, px, py = levels[0]
    z = 5.0
    anchor, xyz, vp, vs, cen = [], [], [0], [], []
    for a, obs, (u, v) in points:
        anchor.append(a); xyz.append([(u - px) / f * z, (v - py) / f * z, z])
        for o in sorted(set(obs) | {a}):
            vs.append(o); cen.append([u, v, u - 10])
        vp.append(len(vs))
    m = dict(poses=np.tile(I7, (V, 1)), point_anchor=np.array(anchor, np.int32), xyz_anchor=np.array(xyz).reshape(-1, 3),
             vis_ptr=np.array(vp, np.int32), vis_pose=np.array(vs, np.int32), feat_center=np.array(cen).reshape(-1, 3),
             feat_level=np.zeros(len(vs), np.int32))
    fr, feats = _blank(levels)
    ptr = np.cumsum([0] + [len(nbr.get(v, [])) for v in range(V)]).astype(np.int32)
    ids = np.array([j for v in range(V) for j in nbr.get(v, [])], np.int32)
    return dict(levels=levels, cam=(f, px, py, sl.CAM_B), frames=[fr] * V, map=m, root=root,
                window=np.array(sorted(window), np.int32), nbr_ptr=ptr, nbr_id=ids, root_features=feats)


def test_bfs_queue_with_duplicates_and_a_vertex_behind_the_window():
    """0-1, 0-2, 1-2 puts 2 in the queue twice; 5 is in the window but only reachable through 4, which is not."""
    nbr = {0: [1, 2], 1: [2, 0], 2: [1, 0, 3], 3: [2, 4], 4: [3, 5], 5: [4]}
    pts = [(v, [v], (100 + 40 * v, 200)) for v in range(6)] + [(1, [3], (500, 50)), (4, [3], (300, 300))]
    sc = _hand_made(6, pts, nbr, window={0, 1, 2, 3, 5})
    res, inter, _ = _run_oracle(sc, 10 ** 6)
    direct, larger, cand = _assert_equals_transcription(sc, 10 ** 6, res, inter)
    assert direct == {0, 1, 2} and larger == {0, 1, 2, 3} and res["stage"] == 1
    # frame 3 is the only one scanned: its own point, and the point it sees anchored in 1; not 4's (anchor outside)
    assert [w[0] for w in cand] == [3, 6]


def test_bfs_stops_at_direct_plus_forty():
    """A chain of 60 window vertices, each anchoring one in-frame point seen only by itself."""
    V = 60
    nbr = {v: [j for j in (v + 1, v - 1) if 0 <= j < V] for v in range(V)}
    pts = [(v, [v], (50 + 9 * v, 100 + 5 * v)) for v in range(V)]
    sc = _hand_made(V, pts, nbr, window=set(range(V)))
    res, inter, _ = _run_oracle(sc, 10 ** 6)
    direct, larger, cand = _assert_equals_transcription(sc, 10 ** 6, res, inter)
    assert len(direct) == 2 and len(larger) == 42 and larger == set(range(42))
    assert [w[0] for w in cand] == list(range(2, 42)) and res["stage"] == 1


def test_flat_map_stats_count_only_non_direct_anchors():
    """Vertex 3 observes every gated point but anchors none; the direct neighbour 1 anchors candidates and observes
    gated points: neither is counted.  Vertex 2's counts carry the reference's names (u > w/2 is num_left)."""
    from oracle import pyoracle
    sc = sl.make_flat_register_scene(pyoracle, 300, n_direct_anchored=60)
    res, inter, grown = _run_oracle(sc, 20)
    _assert_equals_transcription(sc, 20, res, inter)
    assert res["registered"] == 1 and inter["stats"]["vertex"].tolist() == [2]
    cand_anchor = sc["map"]["point_anchor"][inter["cand_point"]]
    assert (cand_anchor == 1).any()
    uvu = inter["tracks"]["uvu"]
    W, H = sc["levels"][0][:2]
    s = inter["stats"][0]
    assert s["strength"] == res["n_tracks"]                  # vertex 2 observes every point
    assert s["num_left"] == int((uvu[:, 0] > W * 0.5).sum()) and s["num_lower"] == int((uvu[:, 1] > H * 0.5).sum())
    assert s["num_left"] != s["num_right"]
