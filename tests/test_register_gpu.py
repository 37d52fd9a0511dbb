"""GPU tests of svs_localRegisterFrame against oracle/register_oracle.c on the rendered revisit inside the double window
(synth_loop.make_register_scene) and on flat maps.  Bar: counts, stages, the stats table, the track list and the
committed map's observation lists bit-equal; the poses to 1e-9 (the LM sums in a different order than the oracle); a
rejection or refusal leaves the map bit-identical."""
import functools

import numpy as np
import pytest

from scavislam_b200 import synth_loop as sl

pytestmark = pytest.mark.gpu

COUNTS = ("registered", "stage", "n_direct", "n_neighborhood", "n_candidates", "n_matched1", "n_matched2", "n_tracks",
          "n_stats", "n_neighbors", "n_committed")


@functools.lru_cache(maxsize=1)
def _scene():
    from oracle import pyoracle
    return sl.make_register_scene(pyoracle)


def _oracle(sc, covis_thr, m=None):
    from oracle import register_pyoracle as ro
    m = sc["map"] if m is None else m
    V = len(m["poses"])
    rf = sc["frames"][sc["root"]]
    return ro.local_register_frame(m, sc["nbr_ptr"], sc["nbr_id"], sc["levels"], rf["pyr"], rf["disp"], sc["root_features"],
                                   [sc["frames"][v]["pyr"] for v in range(V)], sc["cam"], covis_thr, sc["root"], sc["window"],
                                   np.arange(V, dtype=np.int32))


def _setup(svs, sc, m=None, graph=True, max_points=8192):
    m = sc["map"] if m is None else m
    V = len(m["poses"])
    dm = svs.DeviceMap()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    if graph:
        dm.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    mt = svs.GuidedMatcher(sc["levels"], max_keyframes=V, max_points=max_points)
    for v in range(V):
        mt.set_keyframe(v, m["poses"][v], sc["frames"][v]["pyr"])
    rf = sc["frames"][sc["root"]]
    mt.set_current(rf["pyr"], rf["disp"])
    for l, (xy, content) in enumerate(sc["root_features"]):
        mt.set_features(l, xy, content)
    po = svs.PoseOptimizer(max_obs=8192)
    return dm, mt, po, np.arange(V, dtype=np.int32)


def _call(dm, mt, po, sc, covis_thr, slot, **kw):
    return dm.local_register_frame(mt, po, sc["cam"], covis_thr, kw.get("root", sc["root"]), kw.get("window", sc["window"]),
                                   kw.get("vertex_slot", slot), cap_stats=kw.get("cap_stats"), cap_tracks=kw.get("cap_tracks"))


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


def _assert_result(res, stats, tracks, ref, inter):
    for f in COUNTS:
        assert res[f] == ref[f], (f, res[f], ref[f])
    if res["stage"] == 0 or res["stage"] >= 3:
        np.testing.assert_allclose(res["T_align1"], ref["T_align1"], rtol=0, atol=1e-9)
        np.testing.assert_allclose(res["T_newroot_from_oldroot"], ref["T_newroot_from_oldroot"], rtol=0, atol=1e-9)
    if res["stage"] == 0:
        np.testing.assert_allclose(res["T_newroot_from_w"], ref["T_newroot_from_w"], rtol=0, atol=1e-9)
    if res["stage"] in (0, 4):
        assert stats.tobytes() == inter["stats"].tobytes()
        for f in ("point", "uvu", "level", "committed"):
            np.testing.assert_array_equal(tracks[f], inter["tracks"][f])


def test_registered_root_equals_the_oracle_and_grows_the_map(svs):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    ref, inter, grown = _oracle(sc, 20)
    assert ref["registered"] == 1
    dm, mt, po, slot = _setup(svs, sc)
    res, stats, tracks = _call(dm, mt, po, sc, 20, slot)
    _assert_result(res, stats, tracks, ref, inter)
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown))
    Tm, xm = dm.get()
    np.testing.assert_array_equal(Tm, m["poses"])
    np.testing.assert_array_equal(xm, m["xyz_anchor"])
    dm2, mt2, po2, _ = _setup(svs, sc)                          # a second call on a fresh map gives the same bits
    res2, stats2, tracks2 = _call(dm2, mt2, po2, sc, 20, slot)
    for f in COUNTS:
        assert res2[f] == res[f]
    for f in ("T_align1", "T_newroot_from_oldroot", "T_newroot_from_w"):
        np.testing.assert_array_equal(res2[f], res[f])
    assert stats2.tobytes() == stats.tobytes()
    for f in ("point", "uvu", "level", "committed"):
        np.testing.assert_array_equal(tracks2[f], tracks[f])
    # again on the grown map, where root already observes the committed points
    ref3, inter3, grown3 = _oracle(sc, 20, m=grown)
    dm.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    res3, stats3, tracks3 = _call(dm, mt, po, sc, 20, slot)
    _assert_result(res3, stats3, tracks3, ref3, inter3)
    assert ref3["registered"] == 1
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown3))
    for h in (dm, mt, po, dm2, mt2, po2):
        h.close()


def _stage_thresholds(ref, inter):
    """covis_thr values that stop the reference at stages 1-4 on this scene (None where none exists)."""
    out = {1: ref["n_candidates"] + 1}
    out[2] = ref["n_matched1"] + 1 if ref["n_matched1"] + 1 <= ref["n_candidates"] else None
    out[3] = ref["n_matched2"] + 1 if ref["n_matched2"] + 1 <= ref["n_matched1"] else None
    s = int(inter["stats"]["strength"].max()) + 1
    out[4] = s if s <= ref["n_matched2"] else None
    return out


@pytest.mark.parametrize("stage", [1, 2, 3, 4])
def test_each_rejection_leaves_the_map_bit_identical(svs, stage):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    base, binter, _ = _oracle(sc, 20)
    thr = _stage_thresholds(base, binter)[stage]
    assert thr is not None, f"the scene has no threshold that stops at stage {stage}"
    ref, inter, _ = _oracle(sc, thr)
    assert ref["stage"] == stage and ref["registered"] == 0
    dm, mt, po, slot = _setup(svs, sc)
    before = _observations(svs, dm, V, Np)
    res, stats, tracks = _call(dm, mt, po, sc, thr, slot)
    _assert_result(res, stats, tracks, ref, inter)
    _assert_same_map(_observations(svs, dm, V, Np), before)
    np.testing.assert_array_equal(dm.get()[0], m["poses"])
    for h in (dm, mt, po):
        h.close()


def test_refusals_leave_the_map_and_the_slots_untouched(svs):
    sc = _scene()
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    dm, mt, po, slot = _setup(svs, sc, graph=False)
    before = _observations(svs, dm, V, Np)
    with pytest.raises(svs.SvsError) as e:                                      # no pose graph
        _call(dm, mt, po, sc, 20, slot)
    assert e.value.rc == -4
    dm.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    for kw in (dict(root=V), dict(root=-1), dict(vertex_slot=np.full(V, 99, np.int32)), dict(vertex_slot=np.zeros(V, np.int32)),
               dict(window=np.array([0, 0], np.int32))):
        with pytest.raises(svs.SvsError) as e:
            _call(dm, mt, po, sc, 20, slot, **kw)
        assert e.value.rc == -1, kw
    with pytest.raises(svs.SvsError) as e:
        _call(dm, mt, po, sc, 0, slot)                                          # covis_thr < 1
    assert e.value.rc == -1
    no_slot = slot.copy(); no_slot[0] = -1
    with pytest.raises(svs.SvsError) as e:                                      # a candidate's anchor without a slot
        _call(dm, mt, po, sc, 20, no_slot)
    assert e.value.rc == -1
    ref, inter, _ = _oracle(sc, 20)
    probe = inter["cand"].copy()
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    for v in range(V):                                                          # slots away from the map poses
        mt.set_keyframe(v, sl.mul(np.array([0, 0, 0, 1, 0.01, 0, 0.0]), m["poses"][v]), sc["frames"][v]["pyr"])
    seen = mt.match(I7, m["poses"][sc["root"]], probe, 10, 22, 10)
    for kw in (dict(cap_tracks=ref["n_tracks"] - 1), dict(cap_stats=ref["n_stats"] - 1)):   # after the refresh
        with pytest.raises(svs.SvsError) as e:
            _call(dm, mt, po, sc, 20, slot, **kw)
        assert e.value.rc == -1 and e.value.result["n_tracks"] == ref["n_tracks"] and e.value.result["n_stats"] == ref["n_stats"]
        assert mt.match(I7, m["poses"][sc["root"]], probe, 10, 22, 10).tobytes() == seen.tobytes()   # slots restored
    small = svs.GuidedMatcher(sc["levels"], max_keyframes=V, max_points=8)
    with pytest.raises(svs.SvsError) as e:                                      # more candidates than max_points
        _call(dm, small, po, sc, 20, slot)
    assert e.value.rc == -1 and e.value.result["n_candidates"] == ref["n_candidates"]
    _assert_same_map(_observations(svs, dm, V, Np), before)
    np.testing.assert_array_equal(dm.get()[0], m["poses"])
    for h in (dm, mt, po, small):
        h.close()


def test_bfs_stops_at_direct_plus_forty(svs):
    """60 window vertices on a chain, each anchoring one in-frame point seen only by itself; covis_thr above the count."""
    V = 60
    levels = sl.levels()
    w, h, f, px, py = levels[0]
    I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
    uv = [(50 + 9 * v, 100 + 5 * v) for v in range(V)]
    m = dict(poses=np.tile(I7, (V, 1)), point_anchor=np.arange(V, dtype=np.int32),
             xyz_anchor=np.array([[(u - px) / f * 5, (v - py) / f * 5, 5.0] for u, v in uv]), vis_ptr=np.arange(V + 1, dtype=np.int32),
             vis_pose=np.arange(V, dtype=np.int32), feat_center=np.array([[u, v, u - 10] for u, v in uv], np.float64),
             feat_level=np.zeros(V, np.int32))
    nbr = [[j for j in (v + 1, v - 1) if 0 <= j < V] for v in range(V)]
    fr = dict(pyr=[np.zeros((l[1], l[0]), np.uint8) for l in levels], disp=np.zeros((h, w), np.float32))
    sc = dict(levels=levels, cam=(f, px, py, sl.CAM_B), frames=[fr] * V, map=m, root=0, window=np.arange(V, dtype=np.int32),
              nbr_ptr=np.cumsum([0] + [len(n) for n in nbr]).astype(np.int32), nbr_id=np.array(sum(nbr, []), np.int32),
              root_features=[(np.zeros((0, 2), np.int32), np.zeros(0, np.int32)) for _ in levels])
    ref, inter, _ = _oracle(sc, 1000)
    assert ref["n_neighborhood"] == 42 and ref["n_candidates"] == 40 and ref["stage"] == 1
    dm, mt, po, slot = _setup(svs, sc)
    res, _, _ = _call(dm, mt, po, sc, 1000, slot)
    for f in COUNTS:
        assert res[f] == ref[f], f
    for hd in (dm, mt, po):
        hd.close()


# ------------------------------------------------------------------ launch boundaries on flat maps
# k_scan runs in chunks of 1024 over the flagged points (the candidate scan's n); the gate, the counting kernel and the
# commit kernels run one thread per match / track in CTAs of 256.

KSCAN, KCTA = 1024, 256


def _compare_on_gpu(svs, sc, covis_thr):
    m = sc["map"]
    V, Np = len(m["poses"]), len(m["point_anchor"])
    ref, inter, grown = _oracle(sc, covis_thr)
    dm, mt, po, slot = _setup(svs, sc)
    before = _observations(svs, dm, V, Np)
    res, stats, tracks = _call(dm, mt, po, sc, covis_thr, slot)
    _assert_result(res, stats, tracks, ref, inter)
    _assert_same_map(_observations(svs, dm, V, Np), _expected_observations(grown) if ref["registered"] else before)
    for h in (dm, mt, po):
        h.close()
    return ref


@pytest.mark.parametrize("nq", [KSCAN - 1, KSCAN, KSCAN + 1])
def test_candidate_scan_across_its_chunks(svs, nq):
    from oracle import pyoracle
    sc = sl.make_flat_register_scene(pyoracle, nq)
    assert len(sc["map"]["point_anchor"]) == nq                 # every point is seen by frame 2 or 3: the scan's n
    ref = _compare_on_gpu(svs, sc, 20)
    assert ref["n_candidates"] == nq and ref["registered"] == 1


def _flat_with_tracks(nt):
    from oracle import pyoracle
    for seed in range(11, 31):
        lo, hi = nt, 3 * nt
        while lo < hi:
            mid = (lo + hi) // 2
            if _oracle(sl.make_flat_register_scene(pyoracle, mid, seed=seed), 20)[0]["n_tracks"] < nt:
                lo = mid + 1
            else:
                hi = mid
        sc = sl.make_flat_register_scene(pyoracle, lo, seed=seed)
        if _oracle(sc, 20)[0]["n_tracks"] == nt:
            return sc
    raise AssertionError(f"no corner order of the flat map gives {nt} tracks")


@pytest.mark.parametrize("nt", [KCTA - 1, KCTA, KCTA + 1])
def test_counting_and_commit_across_a_cta(svs, nt):
    sc = _flat_with_tracks(nt)
    ref = _compare_on_gpu(svs, sc, 20)
    assert ref["n_tracks"] == nt and ref["n_committed"] == nt and ref["registered"] == 1


def test_backend_tick_after_registration(svs):
    """select_window -> set_problem_from_map -> optimize(2) -> absorb on the grown map; its edge count equals the same
    assembly of the oracle's grown map."""
    sc = _scene()
    ref, _, grown = _oracle(sc, 20)
    dm, mt, po, slot = _setup(svs, sc)
    res, _, _ = _call(dm, mt, po, sc, 20, slot)
    assert res["registered"] == 1
    dm.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    want = svs.DeviceMap()
    want.set(grown["poses"], grown["point_anchor"], grown["xyz_anchor"], grown["vis_ptr"], grown["vis_pose"], grown["feat_center"],
             grown["feat_level"])
    want.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    E = []
    for d in (dm, want):
        w = d.select_window(sc["root"], 3, 9)
        ba = svs.BundleAdjuster()
        fixed = np.zeros(len(w["window_vertex"]), np.uint8); fixed[0] = 1
        E.append(d.set_problem(ba, w["window_vertex"], w["active_point"], sc["cam"], fixed=fixed))
        if d is dm:
            it, _ = ba.optimize(2)
            assert it >= 1
            d.absorb(ba)
        ba.close()
    assert E[0] == E[1] > 0
    for h in (dm, mt, po, want):
        h.close()
