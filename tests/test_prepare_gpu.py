"""SlamGraph::prepareForOptimization on the device map (svs_map_prepare_for_optimization, csrc/graph.cu) against the
C oracle (oracle/prepare_oracle.c: opr_prepare_for_optimization) run from the device's own state before each call
(get_graph, window_state, get), and against the long-double transcription of tests/prepare_reference.py.

Exact: the window, the inner flags, the active points, c_i / c_j, the window state, the marginalisation flags and every
graph entry the call does not re-marginalise (bit for bit).  Within BAR of the long-double computeConstraint's magnitude
companion (map_reference.constraint_ratio): the re-marginalised constraints, and c_T / c_Lambda, which must be those
entries.  Reinitialised poses: within POSE_TOL of the long-double restatement of the re-posing chain."""
import ctypes as C
import functools

import numpy as np
import pytest

import map_reference as mr
import prepare_reference as pr
from oracle import graph_pyoracle as gpo
from oracle import prepare_pyoracle as ppo
from scavislam_b200 import capi, synth_loop as sl
from test_graph_gpu import KF_ARGS, W, H, _empty_graph, _first_map, _flat_map, _load, _path_pose_graph, _set_graph, make_keyframe

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
BAR = 1e-12
POSE_TOL = 1e-11   # float64 SE3 products along a chain from the root, against the same chain in long double


def _grow(dm, m, kf, covis_thr=4):
    V = len(m["poses"])
    dm.add_keyframe_graph(V - 1, kf["T"], covis_thr, W, H, **{k: kf[k] for k in KF_ARGS})
    poses, _ = dm.get()
    return mr.add_keyframe(dict(m, poses=poses[:V]), V - 1, poses[V], kf["new_anchor"], kf["new_xyz"], kf["new_anchor_center"],
                           kf["new_anchor_level"], kf["new_center"], kf["new_level"], kf["track_point"], kf["track_center"],
                           kf["track_level"])


def _ld_rows(m_after, g, rewritten):
    """The long-double constraint of every re-marginalised entry: computeConstraint(max, min) at the poses after the
    call, stored as T_1_from_2 on min's entry and its inverse on max's.  {entry: (T, Lambda, cT, cL)}"""
    fptr, fpt = gpo.feature_tables(m_after)
    ptr, ids = g["nbr_ptr"], g["nbr_id"]
    src = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    rows, cache = {}, {}
    for i in np.flatnonzero(rewritten):
        a, b = int(src[i]), int(ids[i])
        v1, v2 = max(a, b), min(a, b)
        if (v1, v2) not in cache:
            T, L, _, cT, cL = mr.compute_constraint(m_after["poses"], fptr, fpt, m_after["point_anchor"], m_after["xyz_anchor"], v1, v2)
            cache[(v1, v2)] = (T, L.reshape(36), cT, np.asarray(cL).reshape(36))
        T, L, cT, cL = cache[(v1, v2)]
        rows[i] = (T if a == v2 else mr._se3_inv(T), L, cT, cL)
    return rows


def _prepare_step(dm, m, root, loop, inner, dbl, ld=True):
    """One prepare checked from the device state before it.  Returns (map mirror with the new poses, result, oracle)."""
    g = dm.get_graph()
    wt, mg = dm.window_state()
    poses, _ = dm.get()
    m = dict(m, poses=poses)
    ref = ppo.prepare_for_optimization(g, mg, wt.astype(np.int32), m, root, loop, inner, dbl)
    out = dm.prepare_for_optimization(root, loop, inner, dbl)
    for k in ("window_vertex", "inner", "active_point"):
        np.testing.assert_array_equal(out[k], ref[k], err_msg=k)
    assert out["do_optimization"] == ref["do_optimization"]
    wt2, mg2 = dm.window_state()
    np.testing.assert_array_equal(wt2, ref["window_type"])
    np.testing.assert_array_equal(mg2, ref["marginalized"])
    g2 = dm.get_graph()
    for k in ("nbr_ptr", "nbr_id", "nbr_strength"):
        np.testing.assert_array_equal(g2[k], g[k], err_msg=k)
    rew = ref["rewritten"]
    np.testing.assert_array_equal(g2["nbr_T"][~rew], g["nbr_T"][~rew])
    np.testing.assert_array_equal(g2["nbr_Lambda"][~rew], g["nbr_Lambda"][~rew])
    poses2, _ = dm.get()
    if ld:
        pl, _, moved = pr.prepare(g, mg, wt, ref["window_type"], m, root, loop)
        assert np.abs(poses2 - np.asarray(pl, np.float64)).max() <= POSE_TOL
        still = np.setdiff1d(np.arange(len(poses)), list(moved))
        np.testing.assert_array_equal(poses2[still], poses[still])
    else:
        assert np.abs(poses2 - ref["poses"]).max() <= POSE_TOL
    m2 = dict(m, poses=poses2)
    worst = 0.0
    for i, (T, L, cT, cL) in _ld_rows(m2, g, rew).items():
        worst = max(worst, mr.constraint_ratio(g2["nbr_T"][i], T, cT), mr.constraint_ratio(g2["nbr_Lambda"][i], L, cL))
    assert worst <= BAR, worst
    # the pairs of copyContraintsToG2o, read after the marginalisation
    win = {int(v): 1 if f else 2 for v, f in zip(out["window_vertex"], out["inner"])}
    ci, cj, cT, cL = mr.select_constraints(g2["nbr_ptr"], g2["nbr_id"], g2["nbr_T"], g2["nbr_Lambda"], win)
    for a, b in ((out["c_i"], ci), (out["c_j"], cj), (out["c_T"], cT), (out["c_Lambda"], cL)):
        np.testing.assert_array_equal(a, b)
    return m2, out, ref


@pytest.mark.parametrize("inner,dbl", [(3, 8), (7, 100), (15, 100)])
def test_sequence_with_a_prepare_at_every_keyframe(inner, dbl):
    """60 keyframes grown with add_keyframe_graph, a prepare at each (root = the newest).  (7, 100) and (15, 100) are the
    window sizes of the reference's rgbd_example.cfg and rgbd_live.cfg."""
    rng = np.random.default_rng(inner)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    n_rew = 0
    for _ in range(60):
        m = _grow(dm, m, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"))
        m, out, ref = _prepare_step(dm, m, len(m["poses"]) - 1, -1, inner, dbl)
        n_rew += ref["rewritten"].sum()
    assert n_rew > 0
    dm.close()


@functools.lru_cache(maxsize=1)
def _loop_scene():
    from oracle import pyoracle
    return sl.make_scene(pyoracle)


@functools.lru_cache(maxsize=1)
def _register_scene():
    from oracle import pyoracle
    return sl.make_register_scene(pyoracle)


def test_verified_loop_then_prepare_reposes_the_loop_side():
    sc = _loop_scene()
    m = sc["map"]
    V, thr, query, loop = len(m["poses"]), 20, sc["query"], sc["loop"]
    g = _path_pose_graph(m, V, 2)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, g)
    m, _, _ = _prepare_step(dm, m, query, -1, 3, 8)
    slot = -np.ones(V, np.int32)
    verts = list(sc["window"]) + [loop]
    for k, v in enumerate(verts):
        slot[v] = k
    mt = capi.GuidedMatcher(sc["levels"], max_keyframes=len(verts), max_points=4096)
    for k, v in enumerate(verts):
        mt.set_keyframe(k, sc["map"]["poses"][v], sc["frames"][v]["pyr"])
    lf = sc["frames"][loop]
    mt.set_current(lf["pyr"], lf["disp"])
    for l, (xy, content) in enumerate(sc["loop_features"]):
        mt.set_features(l, xy, content)
    po = capi.PoseOptimizer(max_obs=4096)
    res, _ = dm.global_loop_closure(mt, po, sc["cam"], thr, query, loop, sc["T_query_from_loop"], sc["window"], slot)
    from oracle import loop_pyoracle as lo
    _, _, grown = lo.global_loop_closure(sc["map"], sc["levels"], lf["pyr"], lf["disp"], sc["loop_features"],
                                         [sc["frames"][v]["pyr"] for v in verts], sc["cam"], thr, query, loop,
                                         sc["T_query_from_loop"], sc["window"], slot)
    assert res["verified"] == 1
    dm.add_edges([loop], [query], [res["n_tracks"]], loop, res["T_newloop_from_w"])
    poses0, _ = dm.get()
    m, out, ref = _prepare_step(dm, dict(grown, poses=poses0), query, loop, 3, 8)
    assert loop in out["window_vertex"]
    assert not np.array_equal(m["poses"][loop], poses0[loop])      # the loop side moved
    for h in (dm, mt, po):
        h.close()


def test_verified_registration_then_prepare():
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
    _, _, grown = ro.local_register_frame(m, g["nbr_ptr"], g["nbr_id"], sc["levels"], rf["pyr"], rf["disp"], sc["root_features"],
                                          [sc["frames"][v]["pyr"] for v in range(V)], sc["cam"], thr, root, sc["window"], slot)
    assert res["registered"] == 1
    q = stats[stats["qualified"] == 1]
    dm.add_edges(q["vertex"].astype(np.int32), np.full(len(q), root, np.int32), q["strength"].astype(np.int32), root,
                 res["T_newroot_from_w"])
    _prepare_step(dm, grown, root, -1, 3, 8)
    _prepare_step(dm, grown, root, -1, 3, 8)
    for h in (dm, mt, po):
        h.close()


# ------------------------------------------------------------------ edge cases
def _snapshot(dm):
    poses, xyz = dm.get()
    return poses, xyz, dm.get_graph(), dm.window_state()


def _same(a, b):
    np.testing.assert_array_equal(a[0], b[0]); np.testing.assert_array_equal(a[1], b[1])
    for k in a[2]:
        np.testing.assert_array_equal(a[2][k], b[2][k], err_msg=k)
    np.testing.assert_array_equal(a[3][0], b[3][0]); np.testing.assert_array_equal(a[3][1], b[3][1])


def _grown_map(seed, n=12):
    rng = np.random.default_rng(seed)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    for _ in range(n):
        m = _grow(dm, m, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"))
    return dm, m


def test_refusals_leave_the_map_bit_identical():
    dm, m = _grown_map(9)
    V = len(m["poses"])
    m, _, _ = _prepare_step(dm, m, V - 1, -1, 3, 8)
    m, _, _ = _prepare_step(dm, m, V - 3, -1, 3, 8)
    before = _snapshot(dm)
    for root, loop, inner, dbl in ((-1, -1, 3, 8), (V, -1, 3, 8), (2, -2, 3, 8), (2, V, 3, 8), (2, -1, 8, 8), (2, -1, 9, 8)):
        with pytest.raises(capi.SvsError) as e:
            dm.prepare_for_optimization(root, loop, inner, dbl)
        assert e.value.rc == ERR_INVALID, (root, loop, inner, dbl)
        _same(before, _snapshot(dm))
    # a capacity too small: the sizes needed come back, nothing changes
    P, L, Cn, do = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    win, inner, act = np.zeros(V, np.int32), np.zeros(V, np.uint8), np.zeros(max(dm.Np, 1), np.int32)
    nn = len(before[2]["nbr_id"])
    ci, cj, cT, cL = np.zeros(nn, np.int32), np.zeros(nn, np.int32), np.zeros((nn, 7)), np.zeros((nn, 36))
    up = lambda a: a.ctypes.data_as(C.POINTER(C.c_ubyte))
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    for capP, capL, capC in ((1, len(act), nn), (V, 0, nn), (V, len(act), 0)):
        rc = capi.lib().svs_map_prepare_for_optimization(dm._h, 2, -1, 3, 8, C.byref(do), capP, C.byref(P), ip(win), up(inner), capL,
                                                         C.byref(L), ip(act), capC, C.byref(Cn), ip(ci), ip(cj), dp(cT), dp(cL))
        assert rc == ERR_INVALID
        _same(before, _snapshot(dm))
    need = (P.value, L.value, Cn.value)
    got = dm.prepare_for_optimization(2, -1, 3, 8)
    assert need == (len(got["window_vertex"]), len(got["active_point"]), len(got["c_i"])) and need[2] > 0
    dm.close()


def test_graph_without_strengths_is_refused():
    dm, m = _grown_map(4, 6)
    g = dm.get_graph()
    dm.set_graph(g["nbr_ptr"], g["nbr_id"], g["nbr_T"], g["nbr_Lambda"])
    before = _snapshot(dm)
    with pytest.raises(capi.SvsError) as e:
        dm.prepare_for_optimization(len(m["poses"]) - 1, -1, 3, 8)
    assert e.value.rc == ERR_STATE
    _same(before, _snapshot(dm))
    dm.close()


def test_graph_upload_resets_the_state_and_select_window_reads_only():
    dm, m = _grown_map(5)
    V = len(m["poses"])
    m, _, _ = _prepare_step(dm, m, V - 1, -1, 3, 8)
    m, _, _ = _prepare_step(dm, m, V - 4, -1, 3, 8)
    wt, mg = dm.window_state()
    assert wt.any() and not mg.all()
    before = _snapshot(dm)
    dm.select_window(V - 2, 3, 8)                                  # between two prepares: changes nothing
    _same(before, _snapshot(dm))
    m, _, _ = _prepare_step(dm, m, V - 2, -1, 3, 8)
    _set_graph(dm, dm.get_graph())                                 # an upload: every entry marginalised, no window
    wt, mg = dm.window_state()
    assert not wt.any() and mg.all()
    m, _, _ = _prepare_step(dm, m, V - 1, -1, 3, 8)
    m = _grow(dm, m, make_keyframe(np.random.default_rng(1), m, V - 1, mode="all"))
    wt, mg = dm.window_state()                                     # the new vertex is outside; its entries are marginalised
    assert wt[V] == 0
    g = dm.get_graph()
    assert mg[g["nbr_ptr"][V]:g["nbr_ptr"][V + 1]].all()
    m, _, _ = _prepare_step(dm, m, V, -1, 3, 8)
    dm.close()


def test_absorb_is_refused_after_a_prepare():
    dm, m = _grown_map(6)
    V = len(m["poses"])
    out = dm.prepare_for_optimization(V - 1, -1, 3, 8)
    ba = capi.BundleAdjuster(device=0)
    dm.set_problem(ba, out["window_vertex"], out["active_point"], mr.CAM, fixed=1 - out["inner"], c_i=out["c_i"], c_j=out["c_j"],
                   c_T=out["c_T"], c_Lambda=out["c_Lambda"])
    dm.prepare_for_optimization(V - 1, -1, 3, 8)
    before = _snapshot(dm)
    with pytest.raises(capi.SvsError) as e:
        dm.absorb(ba)
    assert e.value.rc == ERR_STATE
    _same(before, _snapshot(dm))
    ba.close(); dm.close()


# ------------------------------------------------------------------ launch shapes
def _hub_map(k, shared=2, big=0):
    """Hub 0 with k leaves 1..k (each sharing `shared` points anchored in 0; leaf 1 shares `big` more), and a separate
    pair B = k + 1, C = k + 2 that share points with each other only."""
    V = k + 3
    obs = [[0, 1 + p % k] for p in range(shared * k)] + [[0, 1]] * big + [[k + 1, k + 2]] * 4
    m = _flat_map(len(obs), V, lambda p: obs[p])
    m["point_anchor"] = np.array([o[0] for o in obs], np.int32)
    nbrs = [list(range(1, k + 1))] + [[0] for _ in range(k)] + [[k + 2], [k + 1]]
    ptr, ids = mr._graph_from_lists(nbrs)
    fptr, fpt = gpo.feature_tables(m)
    src = np.repeat(np.arange(V), np.diff(ptr))
    T, L, st = gpo.constraints(m["poses"], fptr, fpt, m["point_anchor"], m["xyz_anchor"], ids, src)
    return m, dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=np.maximum(st, 1), nbr_T=T, nbr_Lambda=L)


@pytest.mark.parametrize("n", [1023, 1024, 1025, 2049])
@pytest.mark.parametrize("what", ["pairs", "vertices"])
def test_marginalised_pairs_and_vertices_at_scan_chunks(n, what):
    """All k hub edges leave the inner window at once: k marginalised pairs (what = pairs: k = n) on V = k + 3 vertices
    (what = vertices: V = n), k_scan's chunks of 1024 over both."""
    k = n if what == "pairs" else n - 3
    m, g = _hub_map(k)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, g)
    m, out, _ = _prepare_step(dm, m, 0, -1, k + 1, k + 2, ld=False)
    assert out["inner"].sum() == k + 1
    m, out, ref = _prepare_step(dm, m, k + 1, -1, 1, 2, ld=False)
    assert ref["rewritten"].sum() == 2 * k
    dm.close()


def test_marginalised_pair_on_the_scratch_route():
    """A re-marginalised pair whose feature tables exceed k_compute_constraint's 2048 shared-memory depths."""
    m, g = _hub_map(4, big=2100)
    fptr, _ = gpo.feature_tables(m)
    assert mr.constraint_route(fptr, [1], [0])[1] > mr.SMEM_DEPTHS
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, g)
    m, _, _ = _prepare_step(dm, m, 0, -1, 5, 6)
    m, _, ref = _prepare_step(dm, m, 5, -1, 1, 2)
    assert ref["rewritten"].sum() == 8
    dm.close()


# ------------------------------------------------------------------ one back end
def test_back_end_loop_on_the_device():
    """20 keyframes of add_keyframe_graph -> prepare_for_optimization -> set_problem_from_map -> optimize(2) -> absorb,
    with no host edit of the map: at each step the assembled problem equals the oracle's prepare and copy_data_to_g2o
    from the device state before the step."""
    rng = np.random.default_rng(12)
    m = _first_map(rng)
    dm = capi.DeviceMap(device=0)
    _load(dm, m)
    _set_graph(dm, _empty_graph(1))
    ba = capi.BundleAdjuster(device=0)
    for _ in range(20):
        m = _grow(dm, m, make_keyframe(rng, m, len(m["poses"]) - 1, mode="all"))
        xyz = dm.get()[1]
        m = dict(m, xyz_anchor=xyz)
        m, out, ref = _prepare_step(dm, m, len(m["poses"]) - 1, -1, 3, 8)
        if not out["do_optimization"]:
            continue
        E = dm.set_problem(ba, out["window_vertex"], out["active_point"], mr.CAM, fixed=1 - out["inner"], c_i=out["c_i"],
                           c_j=out["c_j"], c_T=out["c_T"], c_Lambda=out["c_Lambda"])
        exp = mr.copy_data_to_g2o(dict(m, poses=ref["poses"]), ref["window_vertex"], ref["active_point"])
        ep, es, ea, obs, info = dm.last_edges(E)
        for a, b in ((ep, exp["e_point"]), (es, exp["e_pose"]), (ea, exp["e_anchor"]), (obs, exp["e_obs"]), (info, exp["e_info"])):
            np.testing.assert_array_equal(a, b)
        ba.optimize(2)
        dm.absorb(ba)
    ba.close(); dm.close()
