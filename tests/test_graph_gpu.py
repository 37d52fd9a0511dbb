"""The pose graph grown on the device (csrc/graph.cu): svs_map_add_keyframe_graph (SlamGraph::addKeyframe with
computeStrength's quirk B15, the growth and addNewEdges(LOCAL)) and svs_map_add_edges (registerKeyframes' and
addLoopClosure's edges) against the C oracle (oracle/graph_oracle.c) on a host mirror of the map.

Every step is checked from the device's graph before it: nbr_ptr, nbr_id, nbr_strength and the strength table bit for
bit, the copied entries' T / Lambda bit for bit, the new entries' within 1e-12 of the long-double computeConstraint's
magnitude companion (tests/map_reference.py), and svs_map_select_window on the grown graph equal to the window of the
oracle's graph uploaded with svs_map_set_pose_graph."""
import numpy as np
import pytest

import functools

import map_reference as mr
from oracle import graph_pyoracle as gpo
from scavislam_b200 import capi, synth_loop as sl

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
W, H = 640, 480
BAR = 1e-12


def _load(dm, m):
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])


def _set_graph(dm, g):
    dm.set_pose_graph(g["nbr_ptr"], g["nbr_id"], g["nbr_strength"], g["nbr_T"], g["nbr_Lambda"])


def _empty_graph(V):
    return dict(nbr_ptr=np.zeros(V + 1, np.int32), nbr_id=np.zeros(0, np.int32), nbr_strength=np.zeros(0, np.int32),
                nbr_T=np.zeros((0, 7)), nbr_Lambda=np.zeros((0, 36)))


def _check_graph(got, ref, m, v1, v2, moved=-1, T_moved=None):
    for k in ("nbr_ptr", "nbr_id", "nbr_strength"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    poses = np.asarray(m["poses"], np.float64).copy()
    if moved >= 0:
        poses[moved] = T_moved
    fptr, fpt = gpo.feature_tables(m)
    new = np.zeros(len(ref["nbr_id"]), bool)
    ptr = ref["nbr_ptr"]
    worst = 0.0
    for k, (a, b) in enumerate(zip(v1, v2)):
        T12, L, _, cT, cL = mr.compute_constraint(poses, fptr, fpt, m["point_anchor"], m["xyz_anchor"], int(a), int(b))
        for me, nb in ((a, b), (b, a)):
            row = ptr[me] + int(np.flatnonzero(ref["nbr_id"][ptr[me]:ptr[me + 1]] == nb)[0])
            new[row] = True
            worst = max(worst, mr.constraint_ratio(got["nbr_T"][row], ref["nbr_T"][row], cT),
                        mr.constraint_ratio(got["nbr_Lambda"][row], ref["nbr_Lambda"][row], np.asarray(cL).reshape(36)))
    assert worst <= BAR, worst
    np.testing.assert_array_equal(got["nbr_T"][~new], ref["nbr_T"][~new])
    np.testing.assert_array_equal(got["nbr_Lambda"][~new], ref["nbr_Lambda"][~new])
    return worst


def _check_window(dm, m, ref, root):
    twin = capi.DeviceMap(device=0)
    _load(twin, m)
    _set_graph(twin, ref)
    V = len(m["poses"])
    a = dm.select_window(root, min(3, V - 1) if V > 1 else 0, min(8, V) if V > 1 else 1)
    b = twin.select_window(root, min(3, V - 1) if V > 1 else 0, min(8, V) if V > 1 else 1)
    for k in ("window_vertex", "inner", "active_point", "c_i", "c_j"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    np.testing.assert_allclose(a["c_T"], b["c_T"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(a["c_Lambda"], b["c_Lambda"], rtol=1e-9, atol=1e-6)
    twin.close()


def _keyframe_step(dm, m, oldkey, kf, covis_thr, check_window=True):
    """Grow the device map by one keyframe and check graph, table and window against the oracle."""
    g0 = dm.get_graph()
    V = len(m["poses"])
    table_ref = gpo.strength_table(m, oldkey, kf["new_anchor"], kf["track_point"], kf["track_center"], covis_thr, W, H)
    assert table_ref is not None
    v, q, table, ne = dm.add_keyframe_graph(oldkey, kf["T"], covis_thr, W, H, **{k: kf[k] for k in KF_ARGS})
    assert (v, q) == (V, len(m["point_anchor"]))
    np.testing.assert_array_equal(table, table_ref)
    poses, _ = dm.get()
    np.testing.assert_allclose(poses[V], np.asarray(mr._se3_mul(np.asarray(kf["T"], np.longdouble), m["poses"][oldkey].astype(np.longdouble)), np.float64), atol=1e-12)
    m2 = mr.add_keyframe(m, oldkey, poses[V], kf["new_anchor"], kf["new_xyz"], kf["new_anchor_center"], kf["new_anchor_level"],
                         kf["new_center"], kf["new_level"], kf["track_point"], kf["track_center"], kf["track_level"])
    v1, v2, s = gpo.local_edges(table_ref, covis_thr, V)
    assert ne == len(v1)
    ref = gpo.add_edges(g0, m2, v1, v2, s)
    got = dm.get_graph()
    _check_graph(got, ref, m2, v1, v2)
    if check_window:
        _check_window(dm, m2, ref, V)
    return m2, table_ref, ne


KF_ARGS = ("new_anchor", "new_xyz", "new_anchor_center", "new_anchor_level", "new_center", "new_level", "track_point",
           "track_center", "track_level")


def _uv(rng, n, mode):
    """Track centres: 'all' over the image, 'left' / 'top' in one half (a frame seen only so never qualifies), 'late'
    in the top-left quadrant but for the last few (frames qualify late)."""
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    if mode == "left":
        u = rng.uniform(0, W / 2 - 1, n)
    elif mode == "top":
        v = rng.uniform(0, H / 2 - 1, n)
    elif mode == "late":
        k = max(n - 4, 0)
        u[:k], v[:k] = rng.uniform(0, W / 2 - 1, k), rng.uniform(0, H / 2 - 1, k)
    return np.stack([u, v, u - 20.0], 1)


def make_keyframe(rng, m, oldkey, n_new=(4, 20), n_track=(10, 60), recent=4, mode=None, anchor_old=True):
    """One keyframe in the style of map_reference.make_map: new points anchored in the last `recent` frames (one at
    least in oldkey when anchor_old), tracks of points some recent frame observes, distinct, in random order."""
    V, Np = len(m["poses"]), len(m["point_anchor"])
    nn = int(rng.integers(*n_new))
    na = rng.integers(max(0, V - recent), V, nn).astype(np.int32)
    if anchor_old and nn:
        na[0] = oldkey
    vp, vs = np.asarray(m["vis_ptr"]), np.asarray(m["vis_pose"])
    seen = np.zeros(Np, bool)
    if Np:
        pt = np.repeat(np.arange(Np), np.diff(vp))
        seen[pt[vs >= V - recent]] = True
    cand = np.flatnonzero(seen)
    nt = min(len(cand), int(rng.integers(*n_track)))
    tp = rng.permutation(cand)[:nt].astype(np.int32)
    mode = mode or rng.choice(["all", "all", "left", "top", "late"])
    T = np.concatenate([[0, 0, 0, 1.0], [-0.05, 0.001 * rng.normal(), 0.0]])
    return dict(T=T, new_anchor=na, new_xyz=np.stack([rng.uniform(-2, 2, nn), rng.uniform(-1.5, 1.5, nn), rng.uniform(3, 10, nn)], 1),
                new_anchor_center=_uv(rng, nn, "all"), new_anchor_level=rng.integers(0, 4, nn).astype(np.int32),
                new_center=_uv(rng, nn, "all"), new_level=rng.integers(0, 4, nn).astype(np.int32), track_point=tp,
                track_center=_uv(rng, nt, mode), track_level=rng.integers(0, 4, nt).astype(np.int32))


def _first_map(rng, n=30):
    m = dict(poses=np.array([[0, 0, 0, 1.0, 0, 0, 0]]), point_anchor=np.zeros(n, np.int32),
             xyz_anchor=np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 10, n)], 1),
             vis_ptr=np.arange(n + 1, dtype=np.int32), vis_pose=np.zeros(n, np.int32), feat_center=_uv(rng, n, "all"),
             feat_level=np.zeros(n, np.int32))
    return m


@pytest.mark.parametrize("covis_thr", [4, 1, 7])
def test_sequence_of_keyframes(covis_thr):
    rng = np.random.default_rng(covis_thr)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    never = 0
    for k in range(60):
        kf = make_keyframe(rng, m, len(m["poses"]) - 1)
        m, table, ne = _keyframe_step(dm, m, len(m["poses"]) - 1, kf, covis_thr, check_window=k % 5 == 4)
        never += np.any(table[:, 1] == 0)
    assert len(m["poses"]) == 61
    assert never > 0            # some frames never qualify
    g = dm.get_graph()
    assert len(g["nbr_id"]) > 60
    dm.close()


def test_add_edges_with_a_moved_vertex():
    """svs_map_add_edges on a grown map with chosen vertices and strengths: three edges into one vertex that is moved
    while their constraints are computed, then one edge between an old and the newest vertex with the old one moved,
    then two more keyframes.  (The edges of a verified registration and loop: the two tests below.)"""
    rng = np.random.default_rng(21)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    for _ in range(24):
        m, _, _ = _keyframe_step(dm, m, len(m["poses"]) - 1, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"), 4,
                                 check_window=False)
    V = len(m["poses"])
    g = dm.get_graph()
    has = lambda a, b: b in g["nbr_id"][g["nbr_ptr"][a]:g["nbr_ptr"][a + 1]]
    root = V - 1
    reg = [v for v in range(V - 12, V - 4) if not has(v, root)][:3]
    assert reg
    T_root = m["poses"][root].copy(); T_root[4:] += [0.01, -0.02, 0.005]
    strength = rng.integers(4, 30, len(reg)).astype(np.int32)
    dm.add_edges(reg, [root] * len(reg), strength, root, T_root)
    ref = gpo.add_edges(g, m, reg, [root] * len(reg), strength, root, T_root)
    _check_graph(dm.get_graph(), ref, m, reg, [root] * len(reg), root, T_root)
    _check_window(dm, m, ref, root)
    poses, _ = dm.get()
    np.testing.assert_array_equal(poses, m["poses"])          # the moved vertex's map pose is not changed
    # loop: loop = an old vertex, query = the newest
    g = dm.get_graph()
    loop, query = 2, V - 1
    assert not has(loop, query)
    T_loop = m["poses"][loop].copy(); T_loop[4:] += [0.03, 0.0, -0.01]
    dm.add_edges([loop], [query], [17], loop, T_loop)
    ref = gpo.add_edges(g, m, [loop], [query], [17], loop, T_loop)
    _check_graph(dm.get_graph(), ref, m, [loop], [query], loop, T_loop)
    _check_window(dm, m, ref, query)
    for _ in range(2):
        m, _, _ = _keyframe_step(dm, m, len(m["poses"]) - 1, make_keyframe(rng, m, len(m["poses"]) - 1), 4)
    dm.close()


# ------------------------------------------------------------------ a verified registration and a verified loop
def _path_pose_graph(m, V, reach):
    """synth_loop.path_graph's lists with their strengths (the points both frames observe) and constraints."""
    ptr, ids = sl.path_graph(m, V, reach)
    sees = [set() for _ in range(V)]
    for p in range(len(m["point_anchor"])):
        for v in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]]:
            sees[int(v)].add(p)
    st = np.array([len(sees[v] & sees[int(j)]) for v in range(V) for j in ids[ptr[v]:ptr[v + 1]]], np.int32)
    fptr, fpt = gpo.feature_tables(m)
    src = np.repeat(np.arange(V), np.diff(ptr))
    T, L, _ = gpo.constraints(m["poses"], fptr, fpt, m["point_anchor"], m["xyz_anchor"], ids, src)   # T_nbr_from_me
    return dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=st, nbr_T=T, nbr_Lambda=L)


@functools.lru_cache(maxsize=1)
def _register_scene():
    from oracle import pyoracle
    return sl.make_register_scene(pyoracle)


@functools.lru_cache(maxsize=1)
def _loop_scene():
    from oracle import pyoracle
    return sl.make_scene(pyoracle)


def _grow_two_more(dm, m, seed):
    rng = np.random.default_rng(seed)
    for _ in range(2):
        m, _, _ = _keyframe_step(dm, m, len(m["poses"]) - 1, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"), 20)
    return m


def test_verified_registration_commits_its_edges():
    """Backend::localRegisterFrame then registerKeyframes' addNewEdges(METRIC): svs_localRegisterFrame on
    synth_loop.make_register_scene with the pose graph set by svs_map_set_pose_graph, its commit (which reallocates the
    map) keeps the graph, and svs_map_add_edges(v1 = each qualified stats vertex, v2 = root, strength, moved = root at
    T_newroot_from_w) on the grown map equals the oracle; then two more keyframes."""
    from oracle import register_pyoracle as ro
    sc = _register_scene()
    m = sc["map"]
    V, root, thr = len(m["poses"]), sc["root"], 20
    g = _path_pose_graph(m, V, 2)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, g)
    mt = capi.GuidedMatcher(sc["levels"], max_keyframes=V, max_points=8192)
    for v in range(V):
        mt.set_keyframe(v, m["poses"][v], sc["frames"][v]["pyr"])
    rf = sc["frames"][root]
    mt.set_current(rf["pyr"], rf["disp"])
    for l, (xy, content) in enumerate(sc["root_features"]):
        mt.set_features(l, xy, content)
    po = capi.PoseOptimizer(max_obs=8192)
    slot = np.arange(V, dtype=np.int32)
    res, stats, _ = dm.local_register_frame(mt, po, sc["cam"], thr, root, sc["window"], slot)
    ref, inter, grown = ro.local_register_frame(m, g["nbr_ptr"], g["nbr_id"], sc["levels"], rf["pyr"], rf["disp"],
                                                sc["root_features"], [sc["frames"][v]["pyr"] for v in range(V)], sc["cam"],
                                                thr, root, sc["window"], slot)
    assert res["registered"] == 1 and ref["registered"] == 1 and res["n_committed"] == ref["n_committed"] > 0
    assert stats.tobytes() == inter["stats"].tobytes()
    g0 = dm.get_graph()
    for k in g:                                                     # the commit kept the pose graph
        np.testing.assert_array_equal(g0[k], g[k], err_msg=k)
    q = stats[stats["qualified"] == 1]
    assert len(q) >= 1
    v1, v2, s = q["vertex"].astype(np.int32), np.full(len(q), root, np.int32), q["strength"].astype(np.int32)
    T_root = res["T_newroot_from_w"]
    dm.add_edges(v1, v2, s, root, T_root)
    ref_g = gpo.add_edges(g0, grown, v1, v2, s, root, T_root)
    _check_graph(dm.get_graph(), ref_g, grown, v1, v2, root, T_root)
    _check_window(dm, grown, ref_g, root)
    poses, _ = dm.get()
    np.testing.assert_array_equal(poses, m["poses"])                # root's map pose is not changed
    # the constraints see root's committed observations: without them root and the new neighbours share fewer points
    fptr, fpt = gpo.feature_tables(grown)
    fptr0, fpt0 = gpo.feature_tables(m)
    shared = lambda fp, pt, a, b: len(np.intersect1d(pt[fp[a]:fp[a + 1]], pt[fp[b]:fp[b + 1]]))
    assert any(shared(fptr, fpt, a, root) > shared(fptr0, fpt0, a, root) for a in v1)
    with pytest.raises(capi.SvsError) as e:                         # committing twice is a duplicate edge
        dm.add_edges(v1, v2, s, root, T_root)
    assert e.value.rc == ERR_INVALID
    _grow_two_more(dm, grown, 5)
    for h in (dm, mt, po):
        h.close()


def test_verified_loop_commits_its_edge():
    """Backend::globalLoopClosure then addLoopClosure's edge: svs_globalLoopClosure on synth_loop.make_scene with the
    pose graph set by svs_map_set_pose_graph, its commit keeps the graph, and svs_map_add_edges(v1 = loop, v2 = query,
    strength = n_tracks, moved = loop at T_newloop_from_w) on the grown map equals the oracle; then two more keyframes."""
    from oracle import loop_pyoracle as lo
    sc = _loop_scene()
    m = sc["map"]
    V, thr, query, loop = len(m["poses"]), 20, sc["query"], sc["loop"]
    g = _path_pose_graph(m, V, 2)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, g)
    slot = -np.ones(V, np.int32)
    verts = list(sc["window"]) + [loop]
    for k, v in enumerate(verts):
        slot[v] = k
    mt = capi.GuidedMatcher(sc["levels"], max_keyframes=len(verts), max_points=4096)
    for k, v in enumerate(verts):
        mt.set_keyframe(k, m["poses"][v], sc["frames"][v]["pyr"])
    lf = sc["frames"][loop]
    mt.set_current(lf["pyr"], lf["disp"])
    for l, (xy, content) in enumerate(sc["loop_features"]):
        mt.set_features(l, xy, content)
    po = capi.PoseOptimizer(max_obs=4096)
    res, tracks = dm.global_loop_closure(mt, po, sc["cam"], thr, query, loop, sc["T_query_from_loop"], sc["window"], slot)
    ref, inter, grown = lo.global_loop_closure(m, sc["levels"], lf["pyr"], lf["disp"], sc["loop_features"],
                                               [sc["frames"][v]["pyr"] for v in verts], sc["cam"], thr, query, loop,
                                               sc["T_query_from_loop"], sc["window"], slot)
    assert res["verified"] == 1 and ref["verified"] == 1 and res["n_tracks"] == ref["n_tracks"]
    g0 = dm.get_graph()
    for k in g:
        np.testing.assert_array_equal(g0[k], g[k], err_msg=k)
    T_loop = res["T_newloop_from_w"]
    v1, v2, s = np.array([loop], np.int32), np.array([query], np.int32), np.array([res["n_tracks"]], np.int32)
    dm.add_edges(v1, v2, s, loop, T_loop)
    ref_g = gpo.add_edges(g0, grown, v1, v2, s, loop, T_loop)
    _check_graph(dm.get_graph(), ref_g, grown, v1, v2, loop, T_loop)
    _check_window(dm, grown, ref_g, query)
    fptr, fpt = gpo.feature_tables(grown)
    fptr0, fpt0 = gpo.feature_tables(m)
    shared = lambda fp, pt, a, b: len(np.intersect1d(pt[fp[a]:fp[a + 1]], pt[fp[b]:fp[b + 1]]))
    assert shared(fptr, fpt, loop, query) > shared(fptr0, fpt0, loop, query)   # the tracks the commit added
    _grow_two_more(dm, grown, 6)
    for h in (dm, mt, po):
        h.close()


def _flat_map(Np, V, observers):
    """Np points anchored in vertex 0, point p seen by observers(p) (ascending)."""
    vis = [observers(p) for p in range(Np)]
    rng = np.random.default_rng(Np)
    return dict(poses=np.concatenate([np.tile([0, 0, 0, 1.0], (V, 1)), np.stack([-0.05 * np.arange(V), np.zeros(V), np.zeros(V)], 1)], 1),
                point_anchor=np.array([v[0] for v in vis], np.int32),
                xyz_anchor=np.stack([rng.uniform(-2, 2, Np), rng.uniform(-1.5, 1.5, Np), rng.uniform(3, 10, Np)], 1),
                vis_ptr=np.concatenate([[0], np.cumsum([len(v) for v in vis])]).astype(np.int32),
                vis_pose=np.array([f for v in vis for f in v], np.int32), feat_center=_uv(rng, sum(len(v) for v in vis), "all"),
                feat_level=np.zeros(sum(len(v) for v in vis), np.int32))


@pytest.mark.parametrize("pairs", [1023, 1024, 1025, 2049])
@pytest.mark.parametrize("spread", [1, 3])
def test_record_counts_at_scan_chunks(pairs, spread):
    """(track, observer) pair counts at k_scan's chunk of 1024; spread = 1 puts every record in one vertex's segment
    (k_str_closed's warp walks it in chunks of 32), spread = 3 splits them over three vertices."""
    V = 4
    m = _flat_map(pairs, V, lambda p: [p % spread])
    rng = np.random.default_rng(pairs + spread)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(V))
    tp = rng.permutation(pairs).astype(np.int32)
    kf = dict(T=np.array([0, 0, 0, 1.0, -0.05, 0, 0]), new_anchor=np.zeros(0, np.int32), new_xyz=np.zeros((0, 3)),
              new_anchor_center=np.zeros((0, 3)), new_anchor_level=np.zeros(0, np.int32), new_center=np.zeros((0, 3)),
              new_level=np.zeros(0, np.int32), track_point=tp, track_center=_uv(rng, pairs, "late"),
              track_level=np.zeros(pairs, np.int32))
    _, table, ne = _keyframe_step(dm, m, 0, kf, 2)
    assert len(table) == spread
    dm.close()


def test_list_grows_past_32_and_256():
    """A hub vertex whose list grows to 40 and then 300 entries, with equal strengths among old and new entries."""
    V = 302
    m = _flat_map(900, V, lambda p: sorted({0, 1 + p % (V - 1), 1 + (p * 7) % (V - 1)}))
    rng = np.random.default_rng(3)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    g = _empty_graph(V)
    _set_graph(dm, g)
    for lo, hi in ((1, 41), (41, 301)):
        nb = np.arange(lo, hi, dtype=np.int32)
        s = rng.integers(1, 6, len(nb)).astype(np.int32)
        g0 = dm.get_graph()
        dm.add_edges(np.zeros(len(nb), np.int32), nb, s)
        ref = gpo.add_edges(g0, m, np.zeros(len(nb), np.int32), nb, s)
        _check_graph(dm.get_graph(), ref, m, np.zeros(len(nb), np.int32), nb)
    assert np.diff(dm.get_graph()["nbr_ptr"])[0] == 300
    dm.close()


@pytest.mark.parametrize("per_kf", [1, 100])
def test_map_scale(per_kf):
    """Maps of V = 1 000 vertices and 1 000 / 100 000 points."""
    m = mr.make_map(1000, per_kf, seed=per_kf)
    rng = np.random.default_rng(per_kf)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1000))
    for _ in range(2):
        kf = make_keyframe(rng, m, len(m["poses"]) - 1, n_track=(200, 400), recent=8, mode="all")
        m, _, _ = _keyframe_step(dm, m, len(m["poses"]) - 1, kf, 4, check_window=False)
    dm.close()


def _snapshot(dm):
    poses, xyz = dm.get()
    return poses, xyz, dm.get_graph()


def _same(a, b):
    np.testing.assert_array_equal(a[0], b[0]); np.testing.assert_array_equal(a[1], b[1])
    for k in a[2]:
        np.testing.assert_array_equal(a[2][k], b[2][k], err_msg=k)


def test_refusals_leave_map_and_graph():
    rng = np.random.default_rng(9)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    for _ in range(6):
        m, _, _ = _keyframe_step(dm, m, len(m["poses"]) - 1, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"), 4,
                                 check_window=False)
    V = len(m["poses"])
    before = _snapshot(dm)
    # oldkey absent from the strength table: no new point anchored there and no track it observes
    kf = make_keyframe(rng, m, V - 1, anchor_old=False)
    kf["new_anchor"][:] = V - 1
    kf["track_point"] = kf["track_point"][:0]; kf["track_center"] = kf["track_center"][:0]; kf["track_level"] = kf["track_level"][:0]
    with pytest.raises(capi.SvsError) as e:
        dm.add_keyframe_graph(0, kf["T"], 4, W, H, **{k: kf[k] for k in KF_ARGS})
    assert e.value.rc == ERR_INVALID
    dm.V, dm.Np = V, len(m["point_anchor"])
    _same(before, _snapshot(dm))
    g = before[2]
    a = 0
    b = int(g["nbr_id"][g["nbr_ptr"][a]])
    for v1, v2 in (([a], [b]), ([b], [a]), ([1], [1]), ([1, 3], [3, 1]), ([0], [V])):
        with pytest.raises(capi.SvsError) as e:
            dm.add_edges(v1, v2, [5] * len(v1))
        assert e.value.rc == ERR_INVALID, (v1, v2)
        _same(before, _snapshot(dm))
    # a graph without strengths
    dm.set_graph(g["nbr_ptr"], g["nbr_id"], g["nbr_T"], g["nbr_Lambda"])
    before = _snapshot(dm)
    with pytest.raises(capi.SvsError) as e:
        dm.add_edges([0], [V - 1], [5])
    assert e.value.rc == ERR_STATE
    kf = make_keyframe(rng, m, V - 1)
    with pytest.raises(capi.SvsError) as e:
        dm.add_keyframe_graph(V - 1, kf["T"], 4, W, H, **{k: kf[k] for k in KF_ARGS})
    assert e.value.rc == ERR_STATE
    dm.V, dm.Np = V, len(m["point_anchor"])
    _same(before, _snapshot(dm))
    # an unordered list is refused by svs_map_set_pose_graph
    bad = dict(g)
    bad["nbr_strength"] = g["nbr_strength"].copy()
    i = int(np.flatnonzero(np.diff(g["nbr_ptr"]) >= 2)[0])
    lo = g["nbr_ptr"][i]
    bad["nbr_strength"][lo], bad["nbr_strength"][lo + 1] = 1, 1000
    with pytest.raises(capi.SvsError) as e:
        _set_graph(dm, bad)
    assert e.value.rc == ERR_INVALID
    dm.close()
