"""GPU tests of svs_globalLoopClosure against oracle/loop_oracle.c on the rendered revisit (scavislam_b200/synth_loop.py).
Bar: counts, stages, quadrant counts, the track list and the committed map's observation lists bit-equal; the poses to
1e-9 (the LM sums in a different order than the oracle); a rejection or refusal leaves the map bit-identical."""
import functools

import numpy as np
import pytest

from scavislam_b200 import synth_loop as sl

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=1)
def _scene():
    from oracle import pyoracle
    return sl.make_scene(pyoracle)


def _slots(sc):
    V = len(sc["map"]["poses"])
    slot = -np.ones(V, np.int32)
    verts = list(sc["window"]) + [sc["loop"]]
    for s, v in enumerate(verts):
        slot[v] = s
    return slot, verts


def _setup(svs, sc, m=None):
    m = sc["map"] if m is None else m
    dm = svs.DeviceMap()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    slot, verts = _slots(sc)
    mt = svs.GuidedMatcher(sc["levels"], max_keyframes=len(verts), max_points=4096)
    for s, v in enumerate(verts):
        mt.set_keyframe(s, sc["map"]["poses"][v], sc["frames"][v]["pyr"])
    lf = sc["frames"][sc["loop"]]
    mt.set_current(lf["pyr"], lf["disp"])
    for l, (xy, content) in enumerate(sc["loop_features"]):
        mt.set_features(l, xy, content)
    po = svs.PoseOptimizer(max_obs=4096)
    return dm, mt, po, slot


def _oracle(sc, covis_thr, m=None, query=None, loop=None, Tql=None):
    from oracle import loop_pyoracle as lo
    m = sc["map"] if m is None else m
    slot, verts = _slots(sc)
    lf = sc["frames"][sc["loop"] if loop is None else loop]
    return lo.global_loop_closure(m, sc["levels"], lf["pyr"], lf["disp"], sc["loop_features"],
                                  [sc["frames"][v]["pyr"] for v in verts], sc["cam"], covis_thr,
                                  sc["query"] if query is None else query, sc["loop"] if loop is None else loop,
                                  sc["T_query_from_loop"] if Tql is None else Tql, sc["window"], slot)


def _observations(svs, dm, V, Np):
    """The device map's observation lists, read through an assembly of the whole map."""
    ba = svs.BundleAdjuster()
    E = dm.set_problem(ba, np.arange(V), np.arange(Np), (500.0, 320.0, 240.0, 0.1))
    ep, es, ea, obs, info = dm.last_edges(E)
    ba.close()
    return ep, es, obs, info


def _expected_observations(m):
    Np = len(m["point_anchor"])
    ep = np.repeat(np.arange(Np), np.diff(m["vis_ptr"])).astype(np.int32)
    s = (1.0 / (1 << m["feat_level"].astype(np.int64))) ** 2
    return ep, m["vis_pose"], m["feat_center"], np.stack([s, s, np.full_like(s, 0.333 * 0.333)], 1)


def _assert_same_map(got, want):
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)


def _call(dm, mt, po, sc, covis_thr, slot, **kw):
    a = dict(query=sc["query"], loop=sc["loop"], T_query_from_loop=sc["T_query_from_loop"], window_vertex=sc["window"],
             vertex_slot=slot)
    a.update(kw)
    return dm.global_loop_closure(mt, po, sc["cam"], covis_thr, a["query"], a["loop"], a["T_query_from_loop"],
                                  a["window_vertex"], a["vertex_slot"], cap=kw.get("cap"))


COUNTS = ("verified", "stage", "n_candidates", "n_matched1", "n_matched2", "n_tracks", "num_left", "num_right", "num_upper",
          "num_lower")


def _assert_result(res, tracks, ref, inter):
    for f in COUNTS:
        assert res[f] == ref[f], (f, res[f], ref[f])
    if res["stage"] == 0 or res["stage"] >= 2:
        np.testing.assert_allclose(res["T_align1"], ref["T_align1"], rtol=0, atol=1e-9)
        np.testing.assert_allclose(res["T_newloop_from_oldloop"], ref["T_newloop_from_oldloop"], rtol=0, atol=1e-9)
        for k in range(2):
            assert res["lm"][k]["num_obs"] == ref["lm"][k]["num_obs"]
    if res["stage"] == 0:
        np.testing.assert_allclose(res["T_newloop_from_w"], ref["T_newloop_from_w"], rtol=0, atol=1e-9)
    if res["stage"] in (0, 3, 4):
        np.testing.assert_array_equal(tracks["point"], inter["tracks"]["point"])
        np.testing.assert_array_equal(tracks["uvu"], inter["tracks"]["uvu"])
        np.testing.assert_array_equal(tracks["level"], inter["tracks"]["level"])


def test_verified_loop_equals_the_oracle_and_grows_the_map(svs):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    ref, inter, grown = _oracle(sc, 20)
    assert ref["verified"] == 1 and ref["n_tracks"] >= 20
    dm, mt, po, slot = _setup(svs, sc)
    res, tracks = _call(dm, mt, po, sc, 20, slot)
    _assert_result(res, tracks, ref, inter)
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown))
    Tm, xm = dm.get()
    np.testing.assert_array_equal(Tm, m["poses"])
    np.testing.assert_array_equal(xm, m["xyz_anchor"])
    # a second identical call on a fresh map gives the same bits
    dm2, mt2, po2, _ = _setup(svs, sc)
    res2, tracks2 = _call(dm2, mt2, po2, sc, 20, slot)
    for f in COUNTS:
        assert res2[f] == res[f]
    for f in ("T_align1", "T_newloop_from_oldloop", "T_newloop_from_w"):
        np.testing.assert_array_equal(res2[f], res[f])
    for f in ("point", "uvu", "level"):
        np.testing.assert_array_equal(tracks2[f], tracks[f])
    # calling again on the grown map: loop now observes every track's point, which keeps its observation
    ref3, inter3, grown3 = _oracle(sc, 20, m=grown)
    res3, tracks3 = _call(dm, mt, po, sc, 20, slot)
    _assert_result(res3, tracks3, ref3, inter3)
    assert ref3["verified"] == 1
    already = np.isin(tracks3["point"], tracks["point"])
    assert already.any()                                        # tracks of points loop observes since the first call
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown3))
    assert len(grown3["vis_pose"]) == len(grown["vis_pose"]) + int((~already).sum())
    for h in (dm, mt, po, dm2, mt2, po2):
        h.close()


def _stage_thresholds(ref):
    """covis_thr values that stop the reference at stages 1-4 on this scene (None where none exists)."""
    out = {1: ref["n_matched1"] + 1}
    out[2] = ref["n_matched2"] + 1 if ref["n_matched2"] + 1 <= ref["n_matched1"] else None
    out[3] = ref["n_tracks"] + 1 if ref["n_tracks"] + 1 <= ref["n_matched2"] else None
    q = min(ref["num_left"], ref["num_right"], ref["num_upper"], ref["num_lower"])
    out[4] = 2 * q + 2 if 2 * q + 2 <= ref["n_tracks"] else None
    return out


@pytest.mark.parametrize("stage", [1, 2, 3, 4])
def test_each_rejection_leaves_the_map_bit_identical(svs, stage):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    base, _, _ = _oracle(sc, 20)
    thr = _stage_thresholds(base)[stage]
    assert thr is not None, f"the scene has no threshold that stops at stage {stage}"
    ref, inter, _ = _oracle(sc, thr)
    assert ref["stage"] == stage and ref["verified"] == 0
    dm, mt, po, slot = _setup(svs, sc)
    before = _observations(svs, dm, V, Np)
    res, tracks = _call(dm, mt, po, sc, thr, slot)
    _assert_result(res, tracks, ref, inter)
    _assert_same_map(_observations(svs, dm, V, Np), before)
    for h in (dm, mt, po):
        h.close()


def test_refusals_leave_the_map_untouched(svs):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    dm, mt, po, slot = _setup(svs, sc)
    before = _observations(svs, dm, V, Np)
    bad = [dict(query=V), dict(loop=-1), dict(loop=sc["query"]), dict(vertex_slot=np.where(slot >= 0, 99, -1)),
           dict(window_vertex=np.array([sc["query"], sc["query"]], np.int32))]
    for kw in bad:
        with pytest.raises(svs.SvsError) as e:
            _call(dm, mt, po, sc, 20, slot, **kw)
        assert e.value.rc == -1, kw
    with pytest.raises(svs.SvsError) as e:
        _call(dm, mt, po, sc, 0, slot)                                          # covis_thr < 1
    assert e.value.rc == -1
    no_anchor_slot = slot.copy(); no_anchor_slot[sc["query"]] = -1
    with pytest.raises(svs.SvsError) as e:
        _call(dm, mt, po, sc, 20, no_anchor_slot)                               # a candidate's anchor without a slot
    assert e.value.rc == -1
    ref, inter, _ = _oracle(sc, 20)
    # the slots as a later svs_match sees them: points in loop's slot, whose refresh would move them
    probe = inter["cand"].copy()
    probe["keyframe"] = slot[sc["loop"]]
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    seen = mt.match(I7, m["poses"][sc["loop"]], probe, 10, 22, 10)
    with pytest.raises(svs.SvsError) as e:
        _call(dm, mt, po, sc, 20, slot, cap=ref["n_tracks"] - 1)                # cap < n_tracks, after the refresh
    assert e.value.rc == -1 and e.value.result["n_tracks"] == ref["n_tracks"]
    assert mt.match(I7, m["poses"][sc["loop"]], probe, 10, 22, 10).tobytes() == seen.tobytes()   # slots restored
    small = svs.GuidedMatcher(sc["levels"], max_keyframes=len(slot), max_points=8)
    with pytest.raises(svs.SvsError) as e:                                      # more candidates than max_points
        dm.global_loop_closure(small, po, sc["cam"], 20, sc["query"], sc["loop"], sc["T_query_from_loop"], sc["window"], slot)
    assert e.value.rc == -1 and e.value.result["n_candidates"] == ref["n_candidates"]
    po_small = svs.PoseOptimizer(max_obs=8)
    with pytest.raises(svs.SvsError) as e:                                      # more candidates than max_obs
        _call(dm, mt, po_small, sc, 20, slot)
    assert e.value.rc == -1
    po_small.close()
    # a candidate whose anchor has no observation of it, and one at a level the matcher lacks: other maps
    p0 = int(inter["cand_point"][0])
    a0, a1 = m["vis_ptr"][p0], m["vis_ptr"][p0 + 1]
    ia = a0 + int(np.flatnonzero(m["vis_pose"][a0:a1] == m["point_anchor"][p0])[0])
    keep = np.ones(len(m["vis_pose"]), bool); keep[ia] = False
    vp = m["vis_ptr"].copy(); vp[p0 + 1:] -= 1
    no_obs = dict(m, vis_ptr=vp, vis_pose=m["vis_pose"][keep], feat_center=m["feat_center"][keep], feat_level=m["feat_level"][keep])
    lvl = m["feat_level"].copy(); lvl[ia] = len(sc["levels"])
    for mm in (no_obs, dict(m, feat_level=lvl)):
        dmx = svs.DeviceMap()
        dmx.set(mm["poses"], mm["point_anchor"], mm["xyz_anchor"], mm["vis_ptr"], mm["vis_pose"], mm["feat_center"], mm["feat_level"])
        bx = _observations(svs, dmx, V, Np)
        with pytest.raises(svs.SvsError) as e:
            _call(dmx, mt, po, sc, 20, slot)
        assert e.value.rc == -1
        _assert_same_map(_observations(svs, dmx, V, Np), bx)
        dmx.close()
    assert mt.match(I7, m["poses"][sc["loop"]], probe, 10, 22, 10).tobytes() == seen.tobytes()
    _assert_same_map(_observations(svs, dm, V, Np), before)
    # after the refusals the same call still verifies exactly like the oracle
    ref, inter, grown = _oracle(sc, 20)
    res, tracks = _call(dm, mt, po, sc, 20, slot)
    _assert_result(res, tracks, ref, inter)
    for h in (dm, mt, po, small):
        h.close()


def test_candidate_anchored_in_loop(svs):
    """The loop vertex itself in the window: candidates anchored in it use its map pose for the projection and the
    predicted T_loop_from_world in its slot, as the reference's vertex_table does."""
    sc = _scene()
    win = np.unique(np.concatenate([sc["window"], [sc["loop"], 1]])).astype(np.int32)
    m = sc["map"]
    # the query observes some points anchored in the loop keyframe: add its observation of the first ones
    from oracle import loop_pyoracle as lo
    V, Np = len(m["poses"]), len(m["point_anchor"])
    pts = np.flatnonzero(m["point_anchor"] == sc["loop"])[:40]
    vp, vs, cen, lvl = [m["vis_ptr"][0]], [], [], []
    for p in range(Np):
        a, b = m["vis_ptr"][p], m["vis_ptr"][p + 1]
        vs += list(m["vis_pose"][a:b]); cen += list(m["feat_center"][a:b]); lvl += list(m["feat_level"][a:b])
        if p in pts:
            vs.append(sc["query"]); cen.append(m["feat_center"][a]); lvl.append(m["feat_level"][a])
        vp.append(len(vs))
    m2 = dict(m, vis_ptr=np.array(vp, np.int32), vis_pose=np.array(vs, np.int32), feat_center=np.array(cen),
              feat_level=np.array(lvl, np.int32))
    sc2 = dict(sc, window=win, map=m2)
    ref, inter, grown = _oracle(sc2, 20)
    assert np.isin(inter["cand_point"], pts).any()
    dm, mt, po, slot = _setup(svs, sc2, m2)
    res, tracks = _call(dm, mt, po, sc2, 20, slot)
    _assert_result(res, tracks, ref, inter)
    assert ref["verified"] == 1
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown))
    for h in (dm, mt, po):
        h.close()


# ------------------------------------------------------------------ launch boundaries on a flat map
# Vertices 0 (loop), 1 (query), 2 (anchor) at the identity, all seeing the same rendered image: every candidate is
# predicted on the FAST corner it was made from, so the number of candidates follows the query's observations and the
# number of tracks follows the candidates.  k_scan runs in chunks of 1024 (the query's observations are its n), the gate
# and k_count_matched in steps of kGate = 256.

KSCAN, KGATE = 1024, 256


@functools.lru_cache(maxsize=None)
def _flat_image(seed=11):
    from oracle import pyoracle
    from scavislam_b200 import frontend_inputs as fi, synth_images as si
    img, disp = si.render_frame(np.zeros(3), 0.0, seed=77)
    pyr = fi.uint8_pyramid(img, sl.NLV)
    xy = pyoracle.fast_detect_roi(img, 8, 632, 8, 472, 12)
    xy = xy[disp[xy[:, 1], xy[:, 0]] > 1]
    xy = xy[np.random.default_rng(seed).permutation(len(xy))]      # spread over the image, not in raster order
    feats = []
    for l in range(sl.NLV):
        k = pyoracle.fast_detect_roi(pyr[l], 0, 640 >> l, 0, 480 >> l, 12)
        feats.append((k, np.arange(len(k), dtype=np.int32)))
    return pyr, disp, xy, feats


def _flat_scene(nq, n_extra=300, seed=11):
    """nq points the query observes (the first nq corners in the order `seed` shuffles them), n_extra more seen by the
    anchor only."""
    pyr, disp, xy, feats = _flat_image(seed)
    f, px, py, b = sl.CAM_F, sl.CAM_PX, sl.CAM_PY, sl.CAM_B
    n = nq + n_extra
    assert n <= len(xy)
    u, v = xy[:n, 0].astype(np.float64), xy[:n, 1].astype(np.float64)
    d = disp[xy[:n, 1], xy[:n, 0]].astype(np.float64)
    z = f * b / d
    X = np.stack([(u - px) / f * z, (v - py) / f * z, z], 1)
    vp, vs, cen = [0], [], []
    for p in range(n):
        obs = [(1, [u[p], v[p], u[p] - d[p]])] if p < nq else []
        obs.append((2, [u[p], v[p], u[p] - d[p]]))
        for vert, c in obs:
            vs.append(vert); cen.append(c)
        vp.append(len(vs))
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    m = dict(poses=np.tile(I7, (3, 1)), point_anchor=np.full(n, 2, np.int32), xyz_anchor=X, vis_ptr=np.array(vp, np.int32),
             vis_pose=np.array(vs, np.int32), feat_center=np.array(cen).reshape(-1, 3), feat_level=np.zeros(len(vs), np.int32))
    fr = dict(pyr=pyr, disp=disp)
    return dict(levels=sl.levels(), cam=(f, px, py, b), frames={0: fr, 1: fr, 2: fr}, map=m, query=1, loop=0,
                window=np.array([1, 2], np.int32), T_query_from_loop=I7, loop_features=feats)


def _compare_on_gpu(svs, sc, covis_thr):
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    ref, inter, grown = _oracle(sc, covis_thr)
    dm, mt, po, slot = _setup(svs, sc)
    before = _observations(svs, dm, V, Np)
    res, tracks = _call(dm, mt, po, sc, covis_thr, slot)
    _assert_result(res, tracks, ref, inter)
    after = _observations(svs, dm, V, Np)
    _assert_same_map(after, _expected_observations(grown) if ref["verified"] else before)
    for h in (dm, mt, po):
        h.close()
    return ref


@pytest.mark.parametrize("nq", [0, 1, KSCAN - 1, KSCAN, KSCAN + 1, 2 * KSCAN + 52])
def test_candidate_scan_across_its_chunks(svs, nq):
    sc = _flat_scene(nq)
    m = sc["map"]
    observed = sum(1 in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]] for p in range(len(m["point_anchor"])))
    assert observed == nq                                       # the boundary this case is named for
    ref = _compare_on_gpu(svs, sc, 2 if nq <= 1 else 20)
    assert ref["n_candidates"] == nq
    if nq > 1:
        assert ref["verified"] == 1


def _flat_scene_with_tracks(nt):
    """A flat map whose query sees just enough points for exactly nt tracks.  The LM's pose, and with it the gate, moves
    a little with every added candidate, so not every count is reached by a prefix of one corner order: the prefix is
    searched over a few orders."""
    for seed in range(11, 31):
        lo, hi = nt, 3 * nt
        while lo < hi:
            mid = (lo + hi) // 2
            if _oracle(_flat_scene(mid, seed=seed), 20)[0]["n_tracks"] < nt:
                lo = mid + 1
            else:
                hi = mid
        sc = _flat_scene(lo, seed=seed)
        if _oracle(sc, 20)[0]["n_tracks"] == nt:
            return sc
    raise AssertionError(f"no corner order of the flat map gives {nt} tracks")


@pytest.mark.parametrize("nt", [KGATE - 1, KGATE, KGATE + 1, 2 * KGATE + 90])
def test_gate_across_its_cta_width(svs, nt):
    sc = _flat_scene_with_tracks(nt)
    ref, _, _ = _oracle(sc, 20)
    assert ref["n_tracks"] == nt                                 # the boundary this case is named for
    ref = _compare_on_gpu(svs, sc, 20)
    assert ref["verified"] == 1
