"""CPU tests of oracle/loop_oracle.c (Backend::globalLoopClosure): its candidate loop and gate equal a literal Python
transcription of backend.cpp:853-893 and :904-961, and on the rendered revisit it recovers the true loop pose from a
proposal that is off by several cm and degrees."""
import functools

import numpy as np

from scavislam_b200 import synth_loop as sl


@functools.lru_cache(maxsize=1)
def _run():
    from oracle import loop_pyoracle as lo, pyoracle
    sc = sl.make_scene(pyoracle)
    V = len(sc["map"]["poses"])
    slot = -np.ones(V, np.int32)
    verts = list(sc["window"]) + [sc["loop"]]
    for s, v in enumerate(verts):
        slot[v] = s
    lf = sc["frames"][sc["loop"]]
    out = lo.global_loop_closure(sc["map"], sc["levels"], lf["pyr"], lf["disp"], sc["loop_features"],
                                 [sc["frames"][v]["pyr"] for v in verts], sc["cam"], 20, sc["query"], sc["loop"],
                                 sc["T_query_from_loop"], sc["window"], slot)
    return sc, slot, out


def _transcribe(m, window, slot, Tql, query, levels):
    """backend.cpp:844-893 line by line, over the points in ascending index."""
    from oracle import loop_pyoracle as lo
    Tlw = lo.se3("oloop_se3_mul", lo.se3("oloop_se3_inv", Tql), m["poses"][query])
    win = set(np.asarray(window).tolist())
    want = []
    for p in range(len(m["point_anchor"])):
        a0, a1 = m["vis_ptr"][p], m["vis_ptr"][p + 1]
        if query not in m["vis_pose"][a0:a1]:
            continue
        a = m["point_anchor"][p]
        if a not in win:                                         # IS_IN_SET(p.anchorframe_id, double_window)
            continue
        ia = a0 + int(np.flatnonzero(m["vis_pose"][a0:a1] == a)[0])
        l = m["feat_level"][ia]
        w, h, f, px, py = levels[l]
        x = lo.se3("oloop_se3_act", lo.se3("oloop_se3_mul", Tlw, lo.se3("oloop_se3_inv", m["poses"][a])), m["xyz_anchor"][p])
        u, v = f * (x[0] / x[2]) + px, f * (x[1] / x[2]) + py
        if not (0 <= int(u) < w and 0 <= int(v) < h):            # isInFrame(uv.cast<int>(), 0): int() truncates toward 0
            continue
        want.append((p, slot[a], l, m["feat_center"][ia][0] / (1 << l), m["feat_center"][ia][1] / (1 << l)))
    return Tlw, want


def _assert_candidates(inter, want):
    c = inter["cand"]
    np.testing.assert_array_equal(inter["cand_point"], [w[0] for w in want])
    np.testing.assert_array_equal(c["keyframe"], [w[1] for w in want])
    np.testing.assert_array_equal(c["anchor_level"], [w[2] for w in want])
    np.testing.assert_array_equal(c["anchor_obs_pyr"].reshape(-1, 2), np.array([[w[3], w[4]] for w in want]).reshape(-1, 2))


def test_candidates_equal_the_transcription():
    sc, slot, (res, inter, _) = _run()
    Tlw, want = _transcribe(sc["map"], sc["window"], slot, sc["T_query_from_loop"], sc["query"], sc["levels"])
    np.testing.assert_array_equal(res["T_loop_from_w"], Tlw)
    assert len(want) == res["n_candidates"] > 100
    _assert_candidates(inter, want)


def test_hand_made_candidates_equal_the_transcription():
    """Points on both sides of the (int) frame edge (u in (-1, 0) truncates to 0 and is in; u just below w is in, at w
    out; likewise v), an anchor outside the window, and anchors equal to loop (its map pose projects them)."""
    from oracle import loop_pyoracle as lo
    levels = sl.levels()
    w, h, f, px, py = levels[0]
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    shift = np.array([0, 0, 0, 1, 0.05, 0, 0.0])              # loop's map pose: 5 cm to the side
    poses = np.stack([shift, I7, I7, I7])                     # 0 loop, 1 query, 2 anchor in the window, 3 anchor outside
    uv = [(-0.5, 100), (-1.5, 100), (w - 1e-7, 100), (w + 1e-7, 100), (50, -0.25), (50, -1.0), (50, h - 1e-7), (50, h),
          (320, 240), (321.5, 200.25)]
    z = 5.0
    anchor, xyz, vp, vs, cen, lvl = [], [], [0], [], [], []
    for a in (2, 3, 0):
        for (u, v) in uv:
            Tqa = lo.se3("oloop_se3_mul", I7, lo.se3("oloop_se3_inv", poses[a]))   # the query (= loop here) from the anchor
            Xq = np.array([(u - px) / f * z, (v - py) / f * z, z])
            X = lo.se3("oloop_se3_act", lo.se3("oloop_se3_inv", Tqa), Xq)
            anchor.append(a); xyz.append(X)
            for vert in sorted({a, 1}):
                vs.append(vert); cen.append([u, v, u - 10]); lvl.append(0)
            vp.append(len(vs))
    m = dict(poses=poses, point_anchor=np.array(anchor, np.int32), xyz_anchor=np.array(xyz), vis_ptr=np.array(vp, np.int32),
             vis_pose=np.array(vs, np.int32), feat_center=np.array(cen), feat_level=np.array(lvl, np.int32))
    window = np.array([0, 1, 2], np.int32)
    slot = np.array([1, -1, 0, -1], np.int32)
    pyr = [np.zeros((l[1], l[0]), np.uint8) for l in levels]
    feats = [(np.zeros((0, 2), np.int32), np.zeros(0, np.int32)) for _ in levels]
    res, inter, _ = lo.global_loop_closure(m, levels, pyr, np.zeros((h, w), np.float32), feats, [pyr, pyr],
                                           (f, px, py, sl.CAM_B), 5, 1, 0, I7, window, slot)
    _, want = _transcribe(m, window, slot, I7, 1, levels)
    _assert_candidates(inter, want)
    got = set(inter["cand_point"].tolist())
    n = len(uv)
    assert {0, 2, 4, 6, 8, 9} <= got and not ({1, 3, 5, 7} & got)          # the (int) edge cases of anchor 2
    assert not got & set(range(n, 2 * n))                                  # anchor 3 is outside the window
    assert got & set(range(2 * n, 3 * n))                                  # anchored in loop, projected from its map pose
    assert res["stage"] == 1 and res["n_candidates"] == len(want)


def test_gate_and_quadrants_equal_the_transcription():
    from oracle import loop_pyoracle as lo
    sc, slot, (res, inter, _) = _run()
    T, (W, H) = res["T_newloop_from_oldloop"], sc["levels"][0][:2]
    r2, cand = inter["res2"], inter["cand"]
    pts, lr, ud = [], [0, 0], [0, 0]
    for i in np.flatnonzero(r2["matched"]):
        d = r2["obs"][i] - lo.map_uvu(sc["cam"], T, r2["xyz_actkey"][i])
        factor = 1 << cand["anchor_level"][i]
        if abs(d[0]) < 2.0 * factor and abs(d[1]) < 2.0 * factor and abs(d[2]) < 2.0 * 3:
            pts.append(inter["cand_point"][i])
            lr[int(r2["obs"][i][0] > W * 0.5)] += 1
            ud[int(r2["obs"][i][1] > H * 0.5)] += 1
    np.testing.assert_array_equal(inter["tracks"]["point"], pts)
    assert (res["num_left"], res["num_right"], res["num_upper"], res["num_lower"]) == (lr[0], lr[1], ud[0], ud[1])
    half = 20 // 2
    assert res["verified"] == (len(pts) >= 20 and min(lr + ud) >= half)


def test_revisit_recovers_the_true_loop_pose():
    sc, _, (res, _, grown) = _run()
    assert res["verified"] == 1 and grown is not None
    Tq = sc["map"]["poses"][sc["query"]]
    D = sl.mul(sl.mul(res["T_newloop_from_w"], sl.inv(Tq)), sc["T_true_query_from_loop"])
    P0 = sl.mul(sl.inv(sc["T_query_from_loop"]), sc["T_true_query_from_loop"])
    ang = lambda T: np.rad2deg(2 * np.arccos(min(1.0, abs(T[3]))))
    assert np.linalg.norm(P0[4:]) > 0.03 and ang(P0) > 1.0          # the proposal is off by several cm and degrees
    assert np.linalg.norm(D[4:]) < 0.01 and ang(D) < 0.1
