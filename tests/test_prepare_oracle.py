"""The prepareForOptimization oracle (oracle/prepare_oracle.c: opr_prepare_for_optimization, driven by
oracle/prepare_pyoracle.py) against the literal long-double transcription of tests/prepare_reference.py, on seeded maps
whose pose graphs are chains, hubs and complete graphs, over sequences of prepares whose windows move by one keyframe or
jump, with loop at -1, at the root, inside and outside the window, and across the P < 2 exit."""
import numpy as np
import pytest

import map_reference as mr
import prepare_reference as pr
from oracle import prepare_pyoracle as ppo

BAR = 1e-12
POSE_TOL = 1e-11   # a re-posed vertex is a chain of SE3 products from the root: float64 against long double


def _graph(kind, m, seed):
    V = len(m["poses"])
    if kind == "chain":
        ptr, ids, _, _ = mr.chain_graph(V, with_constraints=False)
    elif kind == "complete":
        ptr, ids, _, _ = mr.complete_graph(V, with_constraints=False)
    else:
        ptr, ids, _, _ = mr.covisibility_graph(m, max_neighbours=4, hubs=(V // 2,), hub_degree=V // 2, with_constraints=False)
    T, L = pr.consistent_graph(ptr, ids, np.random.default_rng(seed))
    st = np.zeros(len(ids), np.int32)
    return dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=st, nbr_T=T, nbr_Lambda=L)


def _step(state, m, root, loop, inner, dbl):
    g, mg, old = state
    out = ppo.prepare_for_optimization(g, mg, old, m, root, loop, inner, dbl)
    poses, E, moved = pr.prepare(g, mg, old, out["window_type"], m, root, loop)
    mrg, rew, rows = pr.directed(g, E)
    np.testing.assert_array_equal(out["marginalized"], mrg)
    np.testing.assert_array_equal(out["rewritten"], rew)
    assert np.abs(out["poses"] - np.asarray(poses, np.float64)).max() <= POSE_TOL
    still = [v for v in range(len(m["poses"])) if v not in moved]
    np.testing.assert_array_equal(out["poses"][still], m["poses"][still])       # nothing else moves
    worst = 0.0
    for i, (T, L, cT, cL) in rows.items():
        worst = max(worst, mr.constraint_ratio(out["graph"]["nbr_T"][i], T, cT), mr.constraint_ratio(out["graph"]["nbr_Lambda"][i], L, cL))
    assert worst <= BAR, worst
    np.testing.assert_array_equal(out["graph"]["nbr_T"][~rew], g["nbr_T"][~rew])
    np.testing.assert_array_equal(out["graph"]["nbr_Lambda"][~rew], g["nbr_Lambda"][~rew])
    # step 5 computed once per edge as (max, min) equals the literal double write
    _, E1, _ = pr.prepare(g, mg, old, out["window_type"], m, root, loop, once=True)
    for k, e in E.items():
        assert e["mrg"] == E1[k]["mrg"]
        for f in ("T", "L12", "L21"):
            np.testing.assert_array_equal(np.asarray(e[f]), np.asarray(E1[k][f]))
    m2 = dict(m, poses=out["poses"])
    return (out["graph"], out["marginalized"], out["window_type"].astype(np.int32)), m2, out, moved, rew


def _start(m, kind, seed):
    g = _graph(kind, m, seed)
    return (g, np.ones(len(g["nbr_id"]), np.uint8), np.zeros(len(m["poses"]), np.int32))


@pytest.mark.parametrize("kind", ["chain", "hubs", "complete"])
def test_sliding_window_matches_transcription(kind):
    """root = the newest keyframe, one keyframe further at each call: edges leave the inner window and are re-marginalised,
    new vertices are placed from their parents."""
    m = mr.make_map(24, 20, seed=3)
    state = _start(m, kind, 5)
    n_rew = n_moved = 0
    for root in range(4, 24):
        state, m, out, moved, rew = _step(state, m, root, -1, 3, 8)
        n_rew += rew.sum(); n_moved += len(moved)
        assert out["do_optimization"]
    assert n_rew > 0 and n_moved > 0


@pytest.mark.parametrize("kind", ["chain", "hubs", "complete"])
def test_jumps_and_loops(kind):
    """Windows that jump across the map, and loop at -1, at root, inside the window and outside it."""
    m = mr.make_map(30, 15, seed=7)
    state = _start(m, kind, 8)
    rng = np.random.default_rng(11)
    for root in [5, 6, 20, 21, 2, 29, 28, 12]:
        state, m, out, _, _ = _step(state, m, root, -1, 4, 10)
        for loop in (root, int(out["window_vertex"][-1]), -1):
            state, m, out, moved, _ = _step(state, m, root, loop, 4, 10)
            if loop == root:        # every other window vertex is reachable from root, and is re-posed
                assert set(moved) == set(out["window_vertex"].tolist()) - {root}
        outside = [v for v in range(30) if v not in set(out["window_vertex"].tolist())]
        state, m, _, _, _ = _step(state, m, root, int(rng.choice(outside)), 4, 10)


def test_short_window_then_a_further_call():
    """P < 2 keeps the new window and the reinitialised poses but skips steps 4 and 5; the next call's old window is the
    short one."""
    m = mr.make_map(12, 10, seed=2)
    state = _start(m, "chain", 1)
    state, m, out, _, _ = _step(state, m, 6, -1, 2, 6)
    assert out["do_optimization"]
    g0, mg0 = state[0], state[1]
    state, m, out, moved, rew = _step(state, m, 7, -1, 0, 1)
    assert not out["do_optimization"] and list(out["window_vertex"]) == [7]
    assert not rew.any() and not moved
    np.testing.assert_array_equal(state[1], mg0)
    state, m, out, moved, rew = _step(state, m, 8, -1, 2, 6)
    assert out["do_optimization"]
    assert not rew.any()      # nothing was INNER in the short window: no edge leaves the inner window


def test_loop_outside_the_window_marks_nothing():
    m = mr.make_map(20, 12, seed=4)
    a = _start(m, "hubs", 2)
    a, m, out, _, _ = _step(a, m, 10, -1, 3, 7)
    r1 = ppo.prepare_for_optimization(*a, m, 11, -1, 3, 7)
    outside = [v for v in range(20) if v not in set(r1["window_vertex"].tolist())]
    r2 = ppo.prepare_for_optimization(*a, m, 11, outside[0], 3, 7)
    np.testing.assert_array_equal(r1["poses"], r2["poses"])
    np.testing.assert_array_equal(r1["marginalized"], r2["marginalized"])
