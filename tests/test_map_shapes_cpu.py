"""CPU checks of tests/map_reference.py: the vectorised restatements equal the plain-Python ones of oracle/pyoracle.py
bit for bit on small maps and on every graph shape the GPU cases use, the long-double computeConstraint equals the C
oracle to 1e-13 of its magnitude companion, the launch-rule restatement is pinned by hand-worked cases, and the
generator is deterministic."""
import numpy as np
import pytest

import map_reference as mr
from scavislam_b200 import synth_graph


def _small_map(seed=0, **kw):
    args = dict(V=24, per_kf=6, track_len=(1, 6), long_tracks=0.1, unobserved=0.1, levels=(0, 30), seed=seed)
    args.update(kw)
    return mr.make_map(**args)


def test_generator_is_deterministic_and_shaped_as_asked():
    m = mr.make_map(12, 5, track_len=(2, 4), long_tracks=0.2, unobserved=0.2, levels=(0, 30), seed=3)
    assert mr.map_digest(m) == mr.map_digest(mr.make_map(12, 5, track_len=(2, 4), long_tracks=0.2, unobserved=0.2,
                                                         levels=(0, 30), seed=3))
    assert mr.map_digest(m) == "fcd23efa927a4d5009ef526498db157376a31e3944611bdc259b3d43b27619e4"
    big = mr.make_map(60, 20, track_len=(2, 6), long_tracks=0.1, unobserved=0.05, levels=(0, 30), seed=1)
    n = np.diff(big["vis_ptr"])
    assert n.max() > 32 and (n == 0).any()
    assert big["feat_level"].min() == 0 and big["feat_level"].max() == 30
    for p in np.nonzero(n)[0][:200]:                            # runs of consecutive keyframes from the anchor on
        vs = big["vis_pose"][big["vis_ptr"][p]:big["vis_ptr"][p + 1]]
        assert vs[0] == big["point_anchor"][p] and np.all(np.diff(vs) == 1)


def test_covisibility_graph_equals_synth_graph():
    m = _small_map(seed=2)
    ptr, ids, _, _ = mr.covisibility_graph(m, max_neighbours=4, with_constraints=False)
    p0, i0, _, _ = synth_graph.make_pose_graph(m, max_neighbours=4, with_constraints=False)
    np.testing.assert_array_equal(ptr, p0); np.testing.assert_array_equal(ids, i0)


def _graphs(m):
    V = len(m["poses"])
    cov = mr.covisibility_graph(m, max_neighbours=4, hubs=(5,), hub_degree=15, seed=1)
    yield "covisibility+hub", cov
    yield "no T/Lambda", cov[:2] + (None, None)
    yield "complete", mr.complete_graph(V)
    yield "chain", mr.chain_graph(V)
    yield "disconnected piece", mr.cut_graph(cov, range(0, 8))
    yield "isolated root", mr.cut_graph(cov, [3])


@pytest.mark.parametrize("seed", [0, 1])
def test_vectorised_restatements_equal_pyoracle(oracle, seed):
    m = _small_map(seed=seed)
    V, Np = len(m["poses"]), len(m["point_anchor"])
    rng = np.random.default_rng(seed)
    for name, (ptr, ids, T, Lm) in _graphs(m):
        for root, inner, dbl in [(3, 0, 1), (3, 2, 5), (0, 7, 8), (5, 6, V + 4), (11, 3, V)]:
            w0 = oracle.compute_double_window(ptr, ids, root, inner, dbl)
            w, pushes = mr.compute_double_window(ptr, ids, root, inner, dbl)
            assert w == w0 and list(w) == list(w0), name
            assert pushes <= mr.bfs_queue_capacity(len(ids))
            a0, x0 = oracle.compute_active_points(m, ptr, ids, w)
            a, x, ext = mr.compute_active_points(m, ptr, ids, w)
            np.testing.assert_array_equal(a, a0); assert x == x0, name
            assert set(ext) == set(x) - set(w)
            if T is not None:
                c0 = oracle.select_constraints(ptr, ids, T, Lm, x)
                c = mr.select_constraints(ptr, ids, T, Lm, x)
                for u, v in zip(c, c0):
                    np.testing.assert_array_equal(u, v)
            else:
                ci, cj, cT, cL = mr.select_constraints(ptr, ids, None, None, x)
                c0 = oracle.select_constraints(ptr, ids, np.zeros((len(ids), 7)), np.zeros((len(ids), 36)), x)
                np.testing.assert_array_equal(ci, c0[0]); np.testing.assert_array_equal(cj, c0[1])
                assert np.all(cT == [0, 0, 0, 1, 0, 0, 0]) and not cL.any()
            if len(a):
                win = np.array(sorted(x), np.int32)
                perm = rng.permutation(a)                       # the caller's order, not sorted
                g0 = oracle.copy_data_to_g2o(m, win, perm)
                g = mr.copy_data_to_g2o(m, win, perm)
                for k in g0:
                    np.testing.assert_array_equal(g[k], g0[k], err_msg=f"{name}: {k}")
    # an isolated root is a window of one; a window larger than the root's component holds the whole component
    iso = mr.cut_graph(mr.covisibility_graph(m, 4, seed=1), [3])
    assert mr.compute_double_window(iso[0], iso[1], 3, 1, 10)[0] == {3: 1}
    piece = mr.cut_graph(mr.chain_graph(V), range(0, 8))
    assert sorted(mr.compute_double_window(piece[0], piece[1], 2, 2, 50)[0]) == list(range(8))


def test_add_keyframe_equals_pyoracle(oracle):
    m = _small_map(seed=4)
    rng = np.random.default_rng(0)
    for n_new, n_track in [(7, 11), (0, 5), (4, 0), (0, 0)]:
        V, Np = len(m["poses"]), len(m["point_anchor"])
        T = oracle.se3_exp(rng.normal(0, 0.1, 6))
        unobs = np.nonzero(np.diff(m["vis_ptr"]) == 0)[0]
        tp = np.unique(np.concatenate([rng.choice(Np, n_track, replace=False), unobs[:2] if n_track else []])).astype(np.int32)
        kw = dict(new_anchor=rng.integers(0, V, n_new), new_xyz=rng.uniform(1, 5, (n_new, 3)),
                  new_anchor_center=rng.uniform(0, 600, (n_new, 3)), new_anchor_level=rng.integers(0, 31, n_new),
                  new_center=rng.uniform(0, 600, (n_new, 3)), new_level=rng.integers(0, 31, n_new),
                  track_point=tp, track_center=rng.uniform(0, 600, (len(tp), 3)), track_level=rng.integers(0, 31, len(tp)))
        m0 = oracle.add_keyframe(m, 3, T, **kw)
        m1 = mr.add_keyframe(m, 3, m0["poses"][-1], **kw)
        for k in m0:
            np.testing.assert_array_equal(m1[k], m0[k], err_msg=k)
        m = m1


def test_long_double_constraint_equals_the_c_oracle(oracle):
    rng = np.random.default_rng(7)
    P, Npt = 6, 400
    tables = [rng.choice(Npt, int(k), replace=False) for k in (300, 250, 1, 2, 3, 100)]
    tables[2] = tables[0][:1]; tables[3] = tables[0][:2]; tables[4] = tables[0][:3]; tables[5] = tables[0][:100]
    g = mr.constraint_tables(P, tables, Npt, seed=1, anchor=rng.integers(0, P, Npt))
    g["poses"][5] = g["poses"][0]; g["poses"][5, 4] += 1e-9         # nearly equal poses: |t12| << |t1|
    g["poses"][5, 4:] += 30.0; g["poses"][0, 4:] += 30.0
    pairs = [(0, 1), (1, 0), (0, 2), (0, 3), (0, 4), (2, 4), (0, 5), (5, 0), (1, 1), (5, 5)]
    v1, v2 = [p[0] for p in pairs], [p[1] for p in pairs]
    T_o, L_o, n_o = oracle.compute_constraints(g["poses"], g["feat_ptr"], g["feat_point"], g["point_anchor"], g["xyz_anchor"], v1, v2)
    T, L, n, cT, cL = mr.compute_constraints(g["poses"], g["feat_ptr"], g["feat_point"], g["point_anchor"], g["xyz_anchor"], v1, v2)
    np.testing.assert_array_equal(n, n_o)
    assert list(n[2:5]) == [1, 2, 3]
    assert mr.constraint_ratio(T_o, T, cT) <= 1e-13
    assert mr.constraint_ratio(L_o, L, cL) <= 1e-13
    # the companion matters: for the nearly equal pair a flat relative bar on Lambda would need to be loose
    k = pairs.index((0, 5))
    rel = float(np.abs(L_o[k, 0, 0] - L[k, 0, 0]) / L[k, 0, 0])
    assert cL[k, 0, 0] > 1e6 * L[k, 0, 0] and rel < 1e-3


def test_median_ties_and_even_odd():
    # distances 5, 5, 5, 7 (even: ranks 1, 2 tie) and 5, 5, 7 (odd)
    xyz = np.array([[0, 0, 5.0], [0, 0, 5.0], [3, 0, 4.0], [0, 0, 7.0]])
    poses = np.zeros((3, 7)); poses[:, 3] = 1; poses[1, 4] = 2.0; poses[2, 4] = 2.0
    g = mr.constraint_tables(3, [[0, 1, 2, 3], [0, 1, 2, 3], [0, 2, 3]], 4, poses=poses, xyz=xyz)
    _, L, n, _, _ = mr.compute_constraints(g["poses"], g["feat_ptr"], g["feat_point"], g["point_anchor"], g["xyz_anchor"], [0, 0], [1, 2])
    assert list(n) == [4, 3]
    assert L[0, 0, 0] == 4 * (350 * 2 / np.longdouble(5)) ** 2 and L[1, 0, 0] == 3 * (350 * 2 / np.longdouble(5)) ** 2


def test_launch_rules_hand_worked():
    assert [mr.scan_chunks(n) for n in (1, 1023, 1024, 1025, 2048, 2049)] == [1, 1, 1, 2, 2, 3]
    assert mr.bfs_queue_capacity(0) == 1 and mr.bfs_queue_capacity(12) == 13
    # a complete graph of 5 walked with a double window of 5 pushes the root and all 20 entries: a full queue
    ptr, ids, _, _ = mr.complete_graph(5, with_constraints=False)
    assert mr.compute_double_window(ptr, ids, 0, 2, 5)[1] == 21 == mr.bfs_queue_capacity(len(ids))
    assert mr.compute_double_window(ptr, ids, 0, 2, 4)[1] == 17      # stops once 4 vertices are in
    fp = np.array([0, 2048, 4096, 4096 + 2049, 4096 + 2049 + 3000])
    in_smem, stride = mr.constraint_route(fp, [0, 1, 2, 3, 2], [1, 2, 3, 2, 0])
    assert list(in_smem) == [True, True, False, False, True] and stride == 3000
    assert mr.constraint_route(fp[:3], [0], [1]) == (np.array([True]), 0)
