"""The device map (csrc/graph.cu) and svs_computeConstraint_batch (csrc/constraint.cu) at map scale and at the sizes where
their kernels change: k_scan past its first, second and third chunk of 1024, k_bfs with a full queue, k_active's
outer-window extension, k_pair_emit on hub vertices and without T / Lambda, growth across chunk boundaries, and
k_compute_constraint at shared counts 0..129, at the shared-memory / scratch boundary of 2048, with mixed batches, median
ties and more than 65 535 pairs.  Every case first asserts, from the launch-rule restatement of tests/map_reference.py,
the boundary it is named for; window, flags, active points, constraints and edge lists must then equal the vectorised
restatement bit for bit, and T / Lambda the long-double computeConstraint within 1e-12 of its magnitude companion.

The last group checks that svs_map_absorb refuses, and leaves the map as it was, when the BA handle no longer holds the
window the map assembled last: after svs_map_set reloads a map of the same size, after a refused assembly, and after
the handle was loaded with another problem of the same P and L."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import map_reference as mr
from scavislam_b200 import synth

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4


def _load(dm, m):
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])


def _problem(g, fixed=None):
    P, L, E = len(g["pose_qt"]), len(g["psi"]), len(g["e_point"])
    fx = np.zeros(P, np.uint8) if fixed is None else np.asarray(fixed, np.uint8)
    return synth.BAProblem(P=P, L=L, E=E, C=0, pose_qt=g["pose_qt"], fixed=fx, psi=g["psi"], e_point=g["e_point"],
                           e_pose=g["e_pose"], e_anchor=g["e_anchor"], e_obs=g["e_obs"], e_info=g["e_info"],
                           c_i=np.zeros(0, np.int32), c_j=np.zeros(0, np.int32), c_T=np.zeros((0, 7)),
                           c_Lambda=np.zeros((0, 36)), cam=np.array(mr.CAM))


def _assert_edges(dm, E, g):
    assert E == len(g["e_point"])
    ep, es, ea, obs, info = dm.last_edges(E)
    np.testing.assert_array_equal(ep, g["e_point"]); np.testing.assert_array_equal(es, g["e_pose"])
    np.testing.assert_array_equal(ea, g["e_anchor"])
    np.testing.assert_array_equal(obs, g["e_obs"]); np.testing.assert_array_equal(info, g["e_info"])


# ------------------------------------------------------------------ window assembly (svs_ba_set_problem_from_map)
_ASM = {}


def _assembly_map():
    """400 keyframes, 240 points each (tracks of 2..8, 5 % of 33..40, 3 % unobserved, levels 0..30); the window is
    keyframes 100..399 without those = 3 mod 7, in a shuffled order."""
    if not _ASM:
        m = mr.make_map(400, 240, track_len=(2, 8), long_tracks=0.05, unobserved=0.03, levels=(0, 30), seed=11)
        rng = np.random.default_rng(0)
        v = np.arange(100, 400)
        win = rng.permutation(v[v % 7 != 3]).astype(np.int32)
        inwin = np.zeros(400, bool); inwin[win] = True
        cand = rng.permutation(np.nonzero(inwin[m["point_anchor"]])[0]).astype(np.int32)
        _ASM.update(m=m, win=win, cand=cand)
    return _ASM["m"], _ASM["win"], _ASM["cand"]


def _assembly_case(L):
    m, win, cand = _assembly_map()
    act = cand[:L] if L else cand
    assert mr.scan_chunks(len(act)) == {1: 1, 1023: 1, 1024: 1, 1025: 2, 2049: 3}.get(L, mr.scan_chunks(len(act)))
    g = mr.copy_data_to_g2o(m, win, act)
    n = np.diff(m["vis_ptr"])[act]
    seen = np.zeros(len(act), bool); seen[g["e_point"]] = True
    return m, win, act, g, n, seen


@pytest.mark.parametrize("L", [1, 1023, 1024, 1025, 2049])
def test_assembly_edges_across_scan_chunks(svs, L):
    m, win, act, g, n, seen = _assembly_case(L)
    if L >= 1023:
        assert not np.all(np.diff(act) > 0)                       # the caller's order, not sorted
        assert n.max() > 32 and (~seen).any()                     # long tracks; points without an edge in the window
    dm, ba = svs.DeviceMap(), svs.BundleAdjuster()
    _load(dm, m)
    E = dm.set_problem(ba, win, act, mr.CAM)
    _assert_edges(dm, E, g)
    np.testing.assert_array_equal(ba.poses(), g["pose_qt"]); np.testing.assert_array_equal(ba.points(), g["psi"])
    dm.close(); ba.close()


def test_assembly_at_sixty_thousand_points_optimises_like_set_problem(svs):
    m, win, act, g, n, seen = _assembly_case(0)
    L = len(act)
    assert 55000 <= L <= 65000 and mr.scan_chunks(L) >= 54
    lv = np.unique(np.round(-np.log2(g["e_info"][:, 0]) / 2).astype(int))
    assert lv[0] == 0 and lv[-1] == 30
    assert n.max() > 32 and (~seen).any()
    dm, ba, ba2 = svs.DeviceMap(), svs.BundleAdjuster(), svs.BundleAdjuster()
    _load(dm, m)
    fixed = np.zeros(len(win), np.uint8); fixed[:2] = 1
    E = dm.set_problem(ba, win, act, mr.CAM, fixed=fixed)
    _assert_edges(dm, E, g)
    it, st = ba.optimize(2)
    ba2.set_problem(_problem(g, fixed))
    it2, st2 = ba2.optimize(2)
    assert it == it2 == 2
    np.testing.assert_allclose(st["chi2_iter"], st2["chi2_iter"], rtol=1e-12)
    np.testing.assert_allclose(ba.poses(), ba2.poses(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(ba.points(), ba2.points(), rtol=1e-10, atol=1e-12)
    for h in (dm, ba, ba2):
        h.close()


# ------------------------------------------------------------------ window selection (svs_map_select_window)
def _restated_selection(m, graph, root, inner, dbl):
    ptr, ids, T, Lm = graph
    w, pushes = mr.compute_double_window(ptr, ids, root, inner, dbl)
    act, x, ext = mr.compute_active_points(m, ptr, ids, w)
    return w, pushes, act, x, ext, mr.select_constraints(ptr, ids, T, Lm, x)


def _check_selection(got, act, x, cons):
    wv = np.array(sorted(x), np.int32)
    np.testing.assert_array_equal(got["window_vertex"], wv)
    np.testing.assert_array_equal(got["inner"], [x[v] == 1 for v in wv])
    np.testing.assert_array_equal(got["active_point"], act)
    for k, r in zip(("c_i", "c_j", "c_T", "c_Lambda"), cons):
        np.testing.assert_array_equal(got[k], r, err_msg=k)


def _later_observer_extensions(m, graph, w):
    """Points whose anchor joins the outer window only through an inner observer after the first one."""
    ptr, ids = graph[0], graph[1]
    nb = [set(ids[ptr[v]:ptr[v + 1]].tolist()) for v in range(len(ptr) - 1)]
    n = 0
    for p in range(len(m["point_anchor"])):
        a = int(m["point_anchor"][p])
        if a in w:
            continue
        inner = [int(f) for f in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]] if w.get(int(f)) == 1]
        ok = [a in nb[f] or f in nb[a] for f in inner]
        n += bool(ok) and not ok[0] and any(ok)
    return n


_SEL = {}


def _selection_case(V):
    """V keyframes, 4 points each; the co-visibility graph with a hub of 300 spread neighbours in the middle; the root is
    the hub, 24 INNER of 200: the window spreads over the whole id range and leaves most of the hub's list out."""
    if V not in _SEL:
        m = mr.make_map(V, 4, track_len=(2, 9), long_tracks=0.02, unobserved=0.02, levels=(0, 30), seed=V)
        hub = V // 2
        graph = mr.covisibility_graph(m, max_neighbours=5, hubs=(hub,), hub_degree=300, seed=V)
        _SEL[V] = (m, graph, hub) + _restated_selection(m, graph, hub, 24, 200)
    return _SEL[V]


@pytest.mark.parametrize("V", [1023, 1024, 1025, 2049, 3000])
def test_selection_across_scan_chunks_with_a_hub(svs, V):
    m, graph, hub, w, pushes, act, x, ext, cons = _selection_case(V)
    ptr, ids, T, Lm = graph
    Np = len(m["point_anchor"])
    wv = np.array(sorted(x))
    assert np.diff(ptr)[hub] >= 300 and len(w) == 200
    assert len(set(ids[ptr[hub]:ptr[hub + 1]].tolist()) - set(x)) > 50     # many of the hub's neighbours stay out
    assert mr.scan_chunks(V) == (V + 1023) // 1024 and mr.scan_chunks(Np) >= 4
    for b in range(1024, V, 1024):                                         # the window on both sides of each boundary
        assert wv.min() < b <= wv.max()
    assert act.min() < 1024 and act.max() >= 1024 * (mr.scan_chunks(Np) - 1)   # active points in the first and last chunk
    assert len(ext) > 0 and max(ext.values()) > 1                          # extended anchors, one by several points
    assert len(cons[0]) > 0
    dm = svs.DeviceMap()
    _load(dm, m)
    dm.set_graph(ptr, ids, T, Lm)
    got = dm.select_window(hub, 24, 200)
    _check_selection(got, act, x, cons)
    dm.set_graph(ptr, ids)                                                 # without T / Lambda: identity and zero
    got = dm.select_window(hub, 24, 200)
    _check_selection(got, act, x, mr.select_constraints(ptr, ids, None, None, x))
    dm.close()


def _small_selection_map():
    return mr.make_map(300, 6, track_len=(2, 7), long_tracks=0.02, unobserved=0.02, levels=(0, 3), seed=5)


@pytest.mark.parametrize("inner", [0, 150, 299])
def test_selection_complete_graph_fills_the_bfs_queue(svs, inner):
    m = _small_selection_map()
    V = len(m["poses"])
    graph = mr.complete_graph(V, seed=1)
    dbl = V if inner < V - 1 else inner + 1
    w, pushes, act, x, ext, cons = _restated_selection(m, graph, 7, inner, dbl)
    assert len(w) == V and pushes == mr.bfs_queue_capacity(len(graph[1]))
    assert sum(t == 1 for t in w.values()) == inner
    dm = svs.DeviceMap()
    _load(dm, m)
    dm.set_graph(*graph)
    _check_selection(dm.select_window(7, inner, dbl), act, x, cons)
    dm.close()


@pytest.mark.parametrize("shape", ["isolated root", "isolated root, inner 1", "piece smaller than the window",
                                   "chain, inner 0", "chain, inner double-1"])
def test_selection_graph_shapes(svs, shape):
    m = _small_selection_map()
    V = len(m["poses"])
    cov = mr.covisibility_graph(m, max_neighbours=5, seed=2)
    root = 120
    graph, inner, dbl = {
        "isolated root": (mr.cut_graph(cov, [root]), 0, 10),
        "isolated root, inner 1": (mr.cut_graph(cov, [root]), 1, 10),
        "piece smaller than the window": (mr.cut_graph(cov, range(100, 140)), 5, 100),
        "chain, inner 0": (mr.chain_graph(V, seed=3), 0, 30),
        "chain, inner double-1": (mr.chain_graph(V, seed=3), 29, 30),
    }[shape]
    w, pushes, act, x, ext, cons = _restated_selection(m, graph, root, inner, dbl)
    if shape.startswith("isolated"):
        assert np.diff(graph[0])[root] == 0 and list(w) == [root] and pushes == 1
    if shape.startswith("piece"):
        assert sorted(w) == list(range(100, 140)) and len(w) < dbl
    if "inner 0" in shape:
        assert all(t == 2 for t in w.values()) and len(act) == 0
    if "double-1" in shape:
        assert sum(t == 2 for t in w.values()) == 1 and len(act) > 0
    dm = svs.DeviceMap()
    _load(dm, m)
    dm.set_graph(*graph)
    _check_selection(dm.select_window(root, inner, dbl), act, x, cons)
    dm.close()


def test_selection_extension_through_a_later_inner_observer(svs):
    """k_active walks a point's observers until one is INNER and either sees the anchor in the window or has an edge to
    it: here the first inner observer of each chosen point has no edge to the anchor and a later one has, and one
    anchor is extended by several points."""
    m = _small_selection_map()
    V = len(m["poses"])
    root, inner, dbl = 120, 11, 31
    ptr, ids, T, Lm = mr.chain_graph(V, seed=4)
    w, _ = mr.compute_double_window(ptr, ids, root, inner, dbl)
    inner_set = sorted(v for v, t in w.items() if t == 1)
    # anchors outside the window whose points reach at least two inner frames
    vp, vs = m["vis_ptr"], m["vis_pose"]
    extra = {}
    for p in range(len(m["point_anchor"])):
        a = int(m["point_anchor"][p])
        obs = [int(f) for f in vs[vp[p]:vp[p + 1]] if w.get(int(f)) == 1]
        if a not in w and len(obs) >= 2 and abs(obs[0] - a) > 1:
            extra.setdefault(a, set()).add(obs[1])
    assert extra, "the map has no track from outside the window into two inner frames"
    a0 = max(extra, key=lambda a: sum(int(m["point_anchor"][p]) == a for p in range(len(m["point_anchor"]))))
    nbrs = [list(ids[ptr[v]:ptr[v + 1]]) for v in range(V)]
    for f in sorted(extra[a0]):
        nbrs[a0].append(f)                                     # a directed entry anchor -> later inner observer only
    graph = mr._with_constraints(*mr._graph_from_lists(nbrs), np.random.default_rng(5))
    w2, pushes, act, x, ext, cons = _restated_selection(m, graph, root, inner, dbl)
    assert w2 == w and a0 in ext and ext[a0] >= 1
    assert _later_observer_extensions(m, graph, w) > 0
    dm = svs.DeviceMap()
    _load(dm, m)
    dm.set_graph(*graph)
    _check_selection(dm.select_window(root, inner, dbl), act, x, cons)
    dm.close()


def _raw_select(svs, dm, root, inner, dbl, capP, capL, capC):
    win, inn, act = np.zeros(max(capP, 1), np.int32), np.zeros(max(capP, 1), np.uint8), np.zeros(max(capL, 1), np.int32)
    ci, cj, cT, cL = (np.zeros(max(capC, 1), np.int32), np.zeros(max(capC, 1), np.int32), np.zeros((max(capC, 1), 7)),
                      np.zeros((max(capC, 1), 36)))
    P, L, Cn = C.c_int(-1), C.c_int(-1), C.c_int(-1)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    rc = svs.lib().svs_map_select_window(dm._h, root, inner, dbl, capP, C.byref(P), ip(win), inn.ctypes.data_as(C.POINTER(C.c_ubyte)),
                                         capL, C.byref(L), ip(act), capC, C.byref(Cn), ip(ci), ip(cj), dp(cT), dp(cL))
    return rc, (P.value, L.value, Cn.value), dict(window_vertex=win[:max(P.value, 0)], inner=inn[:max(P.value, 0)],
                                                  active_point=act[:max(L.value, 0)], c_i=ci[:max(Cn.value, 0)],
                                                  c_j=cj[:max(Cn.value, 0)], c_T=cT[:max(Cn.value, 0)], c_Lambda=cL[:max(Cn.value, 0)])


def test_selection_capacity_error_reports_the_sizes(svs):
    m, graph, hub, w, pushes, act, x, ext, cons = _selection_case(1025)
    need = (len(x), len(act), len(cons[0]))
    dm = svs.DeviceMap()
    _load(dm, m)
    dm.set_graph(*graph)
    for short in range(3):
        caps = [need[0], need[1], need[2]]
        caps[short] -= 1
        rc, sizes, _ = _raw_select(svs, dm, hub, 24, 200, *caps)
        assert rc == ERR_INVALID and sizes == need, (short, rc, sizes, need)
    rc, sizes, got = _raw_select(svs, dm, hub, 24, 200, *need)
    assert rc == 0 and sizes == need
    _check_selection(got, act, x, cons)
    dm.close()


# ------------------------------------------------------------------ growth (svs_map_add_keyframe)
def _R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _project(T_me, T_anchor, xyz):
    """Stereo observation of an anchored point in frame T_me (float64, for plausible inputs only)."""
    Ra = _R(T_anchor[:4])
    X = Ra.T @ (xyz - T_anchor[4:])
    x = _R(T_me[:4]) @ X + T_me[4:]
    f, px, py, b = mr.CAM
    u = f * x[0] / x[2] + px
    return np.array([u, f * x[1] / x[2] + py, u - f * b / x[2]])


def test_growth_across_scan_chunks_then_assemble_optimise_absorb(svs, oracle):
    m = mr.make_map(250, 4, track_len=(2, 6), unobserved=0.05, levels=(0, 30), seed=21)
    rng = np.random.default_rng(3)
    dm, ba = svs.DeviceMap(), svs.BundleAdjuster()
    _load(dm, m)
    for step, (n_new, n_track) in enumerate([(30, 120), (1020, 0), (0, 0), (0, 40)]):
        V, Np = len(m["poses"]), len(m["point_anchor"])
        oldkey = V - 1
        Np2 = Np + n_new
        if step == 0:
            assert mr.scan_chunks(Np) == 1 < mr.scan_chunks(Np2) == 2
        if step == 1:
            assert mr.scan_chunks(Np) == 2 < mr.scan_chunks(Np2) == 3
        T = np.array([0, 0, 0, 1, -0.05, 0, 0.0])
        newT = oracle.se3_mul(T, m["poses"][oldkey])
        unobs = np.nonzero(np.diff(m["vis_ptr"]) == 0)[0]
        recent = np.nonzero(m["point_anchor"] >= V - 5)[0]
        tp = np.unique(np.concatenate([rng.choice(recent, min(n_track, len(recent)), replace=False), unobs[:5] if n_track else []]))
        tp = rng.permutation(tp).astype(np.int32)
        if n_track:
            assert (np.diff(m["vis_ptr"])[tp] == 0).any()                # tracked points that had no observation
        na = rng.integers(max(V - 3, 0), V, n_new).astype(np.int32)
        nx = np.stack([rng.uniform(-1, 1, n_new), rng.uniform(-1, 1, n_new), rng.uniform(4, 9, n_new)], 1)
        kw = dict(new_anchor=na, new_xyz=nx,
                  new_anchor_center=np.array([_project(m["poses"][a], m["poses"][a], x) for a, x in zip(na, nx)]).reshape(-1, 3),
                  new_anchor_level=rng.integers(0, 31, n_new), new_center=np.array(
                      [_project(newT, m["poses"][a], x) for a, x in zip(na, nx)]).reshape(-1, 3),
                  new_level=rng.integers(0, 31, n_new), track_point=tp,
                  track_center=np.array([_project(newT, m["poses"][m["point_anchor"][p]], m["xyz_anchor"][p]) for p in tp]).reshape(-1, 3),
                  track_level=rng.integers(0, 31, len(tp)))
        assert dm.add_keyframe(oldkey, T, **kw) == (V, Np)
        with pytest.raises(svs.SvsError) as e:                          # the pose graph went with the growth
            dm.select_window(V, 2, 6)
        assert e.value.rc == ERR_STATE
        Tm, xm = dm.get()
        np.testing.assert_array_equal(Tm[:V], m["poses"][:V])
        np.testing.assert_allclose(Tm[V], newT, rtol=0, atol=1e-15)
        m = mr.add_keyframe(m, oldkey, Tm[V], **kw)
        np.testing.assert_array_equal(xm, m["xyz_anchor"])
        graph = mr.chain_graph(V + 1, seed=step)
        dm.set_graph(*graph)
        w, pushes, act, x, ext, cons = _restated_selection(m, graph, V, 3, 8)
        got = dm.select_window(V, 3, 8)
        _check_selection(got, act, x, cons)
        fixed = (got["inner"] == 0).astype(np.uint8)
        E = dm.set_problem(ba, got["window_vertex"], got["active_point"], mr.CAM, fixed=fixed, c_i=got["c_i"], c_j=got["c_j"],
                           c_T=got["c_T"], c_Lambda=got["c_Lambda"])
        _assert_edges(dm, E, mr.copy_data_to_g2o(m, got["window_vertex"], got["active_point"]))
        ba.optimize(2)
        poses, psi = ba.poses(), ba.points()
        dm.absorb(ba)
        m["poses"] = m["poses"].copy(); m["xyz_anchor"] = m["xyz_anchor"].copy()
        m["poses"][got["window_vertex"]] = poses
        m["xyz_anchor"][got["active_point"]] = np.stack([psi[:, 0] / psi[:, 2], psi[:, 1] / psi[:, 2], 1.0 / psi[:, 2]], 1)
        Tm, xm = dm.get()
        np.testing.assert_array_equal(Tm, m["poses"]); np.testing.assert_array_equal(xm, m["xyz_anchor"])
    dm.close(); ba.close()


# ------------------------------------------------------------------ constraints (svs_computeConstraint_batch)
BAR = 1e-12
_WORST = {}


def _check_constraints(svs, g, v1, v2, name):
    cb = svs.ConstraintBuilder()
    T_g, L_g, n_g = cb.compute(g["poses"], g["feat_ptr"], g["feat_point"], g["point_anchor"], g["xyz_anchor"], v1, v2)
    cb.close()
    pairs = sorted(set(zip(np.asarray(v1).tolist(), np.asarray(v2).tolist())))
    ref = dict(zip(pairs, zip(*mr.compute_constraints(g["poses"], g["feat_ptr"], g["feat_point"], g["point_anchor"],
                                                       g["xyz_anchor"], [p[0] for p in pairs], [p[1] for p in pairs]))))
    T, L, n, cT, cL = (np.array([ref[(a, b)][k] for a, b in zip(v1, v2)]) for k in range(5))
    np.testing.assert_array_equal(n_g, n)
    rT, rL = mr.constraint_ratio(T_g, T, cT), mr.constraint_ratio(L_g, L, cL)
    _WORST[name] = (rT, rL)
    print(f"constraint ratios {name}: T {rT:.2e} Lambda {rL:.2e}")
    assert rT <= BAR and rL <= BAR, (rT, rL)
    return T_g, L_g, n_g


def test_constraint_shared_counts_around_the_thread_stride(svs):
    rng = np.random.default_rng(1)
    base = np.arange(0, 4000, 2)                                        # frame 0: even ids
    counts = [0, 1, 2, 3, 127, 128, 129]
    tables = [base] + [np.concatenate([rng.choice(base, k, replace=False), 1 + 2 * rng.choice(2000, 50, replace=False)])
                       for k in counts]
    g = mr.constraint_tables(len(tables), tables, 4000, seed=2, anchor=rng.integers(0, len(tables), 4000))
    v1 = [0] * len(counts); v2 = list(range(1, len(tables)))
    assert np.all(mr.constraint_route(g["feat_ptr"], v1, v2)[0])
    _, L, n = _check_constraints(svs, g, v1, v2, "shared counts 0..129")
    assert list(n) == counts and not L[0].any()


def test_constraint_smem_scratch_boundary_and_mixed_batch(svs):
    rng = np.random.default_rng(2)
    N = 3000
    full = np.arange(N)
    t2048, t2049, t2500 = np.sort(rng.choice(N, 2048, replace=False)), np.sort(rng.choice(N, 2049, replace=False)), \
        np.sort(rng.choice(N, 2500, replace=False))
    # frames: 0,1 = the same 2048 points; 2,3 = the same 2049; 4,5 = all 3000; 6 = 2500 of them; 7 = 100 of them
    tables = [t2048, t2048, t2049, t2049, full, full, t2500, full[:100]]
    g = mr.constraint_tables(len(tables), tables, N, seed=3, anchor=rng.integers(0, len(tables), N))
    g["poses"][5] = g["poses"][4]; g["poses"][5, 6] += 1e-7           # nearly equal poses far from the origin
    g["poses"][4, 4:] += 40.0; g["poses"][5, 4:] += 40.0
    v1 = [0, 2, 4, 4, 5, 4, 0, 2, 6, 4, 5, 7, 4] * 8 + [7]
    v2 = [1, 3, 5, 6, 4, 4, 4, 4, 4, 7, 6, 4, 5] * 8 + [4]
    in_smem, stride = mr.constraint_route(g["feat_ptr"], v1, v2)
    assert stride == N
    assert list(in_smem[:3]) == [True, False, False] and in_smem.any() and (~in_smem).any()
    full_rows = [k for k in range(len(v1) - 1) if not in_smem[k] and not in_smem[k + 1]]
    assert full_rows                                                    # adjacent scratch rows
    T_g, L_g, n = _check_constraints(svs, g, v1, v2, "2048 / 2049 and mixed")
    assert n[0] == 2048 and n[1] == 2049 and n[2] == N and n[3] == 2500
    # (a, b) against (b, a): inverse relative poses
    for a, b in [(2, 4), (3, 8), (9, 11)]:                               # (4, 5) / (5, 4), (4, 6) / (6, 4), (4, 7) / (7, 4)
        assert (v1[a], v2[a]) == (v2[b], v1[b])
        Tab, Tba = T_g[a], T_g[b]
        I = mr._se3_mul(Tab.astype(mr.LD), Tba.astype(mr.LD))
        assert np.abs(I[:3]).max() < 1e-14 and np.abs(I[4:]).max() < 1e-12


def test_constraint_median_ties_self_pairs_and_a_large_batch(svs):
    rng = np.random.default_rng(4)
    N = 400
    vals = np.array([[0, 0, 5.0], [3, 0, 4.0], [0, 0, 6.0], [0, 0, 9.0], [0, 0, 5.5]])
    xyz = vals[rng.integers(0, len(vals), N)]                         # five distances only: ties at every rank
    tables = [np.arange(200), np.arange(201), np.arange(200), np.arange(201), np.arange(N), np.arange(7)]
    poses = np.zeros((len(tables), 7)); poses[:, 3] = 1
    poses[:, 4:] = rng.normal(0, 0.5, (len(tables), 3))
    poses[0] = poses[4]; poses[1] = poses[4]                           # so that the distances in frame 0 / 1 are the table's
    g = mr.constraint_tables(len(tables), tables, N, poses=poses, xyz=xyz, anchor=np.full(N, 4))
    v1 = [0, 1, 0, 1, 4, 2, 5, 4]
    v2 = [2, 3, 4, 4, 4, 2, 5, 5]
    _, _, n = _check_constraints(svs, g, v1, v2, "median ties")
    assert list(n[:4]) == [200, 201, 200, 201]
    d = np.sort(np.linalg.norm(xyz[:201], axis=1))
    assert d[99] == d[100] and d[100] == d[101]                        # ties at r_lo / r_hi (even) and the middle (odd)
    # more than 65 535 pairs in one launch
    big1 = np.tile(np.array(v1 + [0, 2, 3]), 9000)[:70001]
    big2 = np.tile(np.array(v2 + [5, 0, 1]), 9000)[:70001]
    assert len(big1) > 65535
    _check_constraints(svs, g, big1, big2, "70001 pairs")


# ------------------------------------------------------------------ svs_map_absorb refuses a window it no longer holds
def _absorb_setup(svs, seed=31):
    m = mr.make_map(40, 30, track_len=(2, 6), levels=(0, 2), seed=seed)
    win = np.arange(10, 30, dtype=np.int32)
    act = np.nonzero((m["point_anchor"] >= 10) & (m["point_anchor"] < 30))[0].astype(np.int32)
    dm, ba = svs.DeviceMap(), svs.BundleAdjuster()
    _load(dm, m)
    fixed = np.zeros(len(win), np.uint8); fixed[0] = 1
    dm.set_problem(ba, win, act, mr.CAM, fixed=fixed)
    ba.optimize(2)
    return m, win, act, fixed, dm, ba


def _assert_refused(svs, dm, ba, before):
    with pytest.raises(svs.SvsError) as e:
        dm.absorb(ba)
    assert e.value.rc == ERR_STATE
    T, x = dm.get()
    np.testing.assert_array_equal(T, before[0]); np.testing.assert_array_equal(x, before[1])


def test_absorb_refused_after_the_map_is_reloaded(svs):
    m, win, act, fixed, dm, ba = _absorb_setup(svs)
    m2 = mr.make_map(40, 30, track_len=(2, 6), levels=(0, 2), seed=32)   # same V and Np, other values
    assert len(m2["poses"]) == len(m["poses"]) and len(m2["point_anchor"]) == len(m["point_anchor"])
    _load(dm, m2)
    _assert_refused(svs, dm, ba, (m2["poses"], m2["xyz_anchor"]))
    dm.set_problem(ba, win, act, mr.CAM, fixed=fixed)                   # a fresh assembly is absorbed again
    ba.optimize(1)
    dm.absorb(ba)
    assert not np.array_equal(dm.get()[0][win], m2["poses"][win])
    dm.close(); ba.close()


def test_absorb_refused_after_a_refused_assembly(svs):
    m, win, act, fixed, dm, ba = _absorb_setup(svs)
    before = dm.get()
    # the same P and L (the work arena does not grow), one window vertex swapped for one outside it that anchors no
    # active point: the anchors of the points of vertex 10 are now outside the window
    win2 = win.copy(); win2[0] = 35
    act2 = act[::-1].copy()
    with pytest.raises(svs.SvsError) as e:
        dm.set_problem(ba, win2, act2, mr.CAM, fixed=fixed)
    assert e.value.rc == ERR_INVALID
    _assert_refused(svs, dm, ba, before)
    dm.close(); ba.close()


@pytest.mark.parametrize("how", ["svs_ba_set_problem", "another map"])
def test_absorb_refused_after_the_handle_holds_another_problem(svs, how):
    m, win, act, fixed, dm, ba = _absorb_setup(svs)
    before = dm.get()
    g = mr.copy_data_to_g2o(m, win, act)
    if how == "svs_ba_set_problem":
        pb = _problem(g, fixed)
        pb = dataclasses.replace(pb, pose_qt=pb.pose_qt.copy(), psi=pb.psi * 1.01)
        pb.pose_qt[:, 4] += 0.01
        ba.set_problem(pb)                                              # same P, L, even the same structure
        assert (ba.P, ba.L) == (len(win), len(act))
    else:
        m2 = mr.make_map(40, 30, track_len=(2, 6), levels=(0, 2), seed=33)
        win2 = np.arange(5, 25, dtype=np.int32)
        act2 = np.nonzero((m2["point_anchor"] >= 5) & (m2["point_anchor"] < 25))[0][:len(act)].astype(np.int32)
        assert len(act2) == len(act)
        dm2 = svs.DeviceMap()
        _load(dm2, m2)
        dm2.set_problem(ba, win2, act2, mr.CAM, fixed=fixed)
        ba.optimize(1)
    _assert_refused(svs, dm, ba, before)
    if how == "another map":
        dm2.absorb(ba)                                                  # the map that assembled it takes it
        assert not np.array_equal(dm2.get()[0][win2], m2["poses"][win2])
        dm2.close()
    dm.close(); ba.close()
