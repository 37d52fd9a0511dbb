"""The long-double reference of the Schur build (tests/build_reference.py) against the oracle, its window builder, and
its restatement of the routing rules of the host set-up, pinned by hand-worked cases.  Runs without a GPU.

Measured (x86-64, 80-bit long double): the reference and oracle.reduced_system differ by at most 9e-16 of M per block,
the skip-self variant and the Schur complement of gauss_newton's H by 6e-16, and the one-step state and
oracle.optimize(pb, 1, max_trials=1) by 5e-14 of the step."""
import numpy as np
import pytest

import ba_grad_reference as gref
import build_reference as br

T = br.Track


def _mixed(fixed=(), C=12, unobserved=2, seed=1):
    """Self-only tracks (k = 1, K = 1), anchorless tracks, a padded track with the anchor inside its span, 9-32 and
    more than 32 slots; frame 2 anchors a track of each kernel and frame 5 observes one of each."""
    tracks = [T(0, (), True, 3), T(2, (3, 4, 5), True, 4), T(4, (5, 6, 8), False, 3), T(10, (8, 9, 11, 13), True, 2),
              T(2, tuple(range(3, 14)), True, 2), T(6, tuple(range(1, 6)) + tuple(range(7, 20)), False, 2),
              T(2, tuple(range(3, 40)), True, 1), T(3, tuple(range(4, 38)), False, 1), T(7, (), True, 2)]
    return br.make_tracks_window(42, tracks, seed=seed, fixed=fixed, C=C, unobserved=unobserved)


WINDOWS = {
    "mixed": lambda: _mixed(),
    "fixed_anchor": lambda: _mixed(fixed=(2,)),
    "fixed_observer": lambda: _mixed(fixed=(5,)),
    "no_constraints": lambda: _mixed(C=0, unobserved=0, seed=3),
}


def test_builder_emits_exactly_the_tracks():
    tracks = [T(0, (), True, 3), T(1, (2, 3), False, 2), T(5, (3, 4, 6), True, 1), T(0, tuple(range(1, 100)), False, 1),
              T(99, tuple(range(0, 99)), True, 1)]
    pb = br.make_tracks_window(100, tracks, seed=4, unobserved=5)
    got, un = br.tracks_of(pb)
    assert got == {(t.anchor, tuple(t.observers), t.self_edge): t.count for t in tracks}
    assert un == 5 and pb.L == sum(t.count for t in tracks) + 5
    has =np.zeros(pb.L, bool); has[pb.e_point] = True
    assert not has[0] and not has[-1] and not has.all()         # the unobserved landmarks are interleaved
    # positive depth and disparity at the state the builder hands out, and Huber takes both branches at delta = 1
    from oracle import pyoracle as po
    e2 = np.array([np.sum(pb.e_info[e] * po.edge_error(pb.cam, pb.pose_qt[pb.e_pose[e]], pb.pose_qt[pb.e_anchor[e]],
                                                      pb.psi[pb.e_point[e]], pb.e_obs[e]) ** 2) for e in range(pb.E)])
    assert (e2 > 1).any() and (e2 <= 1).any()


@pytest.mark.parametrize("name", sorted(WINDOWS))
@pytest.mark.parametrize("robust,delta,lam", [(True, 1.0, 50.0), (False, 1.0, 1e-4), (True, 0.5, 1e5), (True, 3.0, 1e-4)])
def test_reference_equals_the_oracle(oracle, name, robust, delta, lam):
    pb = WINDOWS[name]()
    ref = br.reduced_system(oracle, pb, robust, delta, lam)
    S, bs, chi = oracle.reduced_system(pb, robust, delta, lam)
    assert br.block_ratio(S, ref, pb.P) <= 1e-13
    assert br.rhs_ratio(bs, ref, pb.P) <= 1e-13
    assert abs(chi - float(ref.chi2)) <= 1e-13 * chi


@pytest.mark.parametrize("name", sorted(WINDOWS))
def test_skip_self_equals_the_schur_complement_of_gauss_newton(oracle, name):
    pb, lam = WINDOWS[name](), 3.0
    H, _ = gref.gauss_newton(oracle, pb, True, 1.0)
    n = 6 * pb.P
    A = H + lam * np.eye(H.shape[0])
    has = np.zeros(pb.L, bool); has[pb.e_point] = True
    keep = np.concatenate([np.ones(n, bool), np.repeat(has, 3)])
    A = A[np.ix_(keep, keep)]
    S = A[:n, :n] - A[:n, n:] @ np.linalg.solve(A[n:, n:], A[n:, :n])
    fx = np.repeat(pb.fixed == 1, 6)
    S[fx, fx] += 1.0
    ref = br.reduced_system(oracle, pb, True, 1.0, lam, skip_self=True)
    assert br.block_ratio(S, ref, pb.P) <= 1e-13
    # and it differs from the default, which keeps g2o's self-anchor term on every anchor with a self edge
    dflt = br.reduced_system(oracle, pb, True, 1.0, lam)
    assert br.block_ratio(dflt.S, ref, pb.P) > 1e-6


@pytest.mark.parametrize("name", sorted(WINDOWS))
@pytest.mark.parametrize("robust,lam", [(True, 50.0), (False, 1e5)])
def test_one_step_equals_the_oracle(oracle, name, robust, lam):
    pb = WINDOWS[name]()
    poses, psi, x, ref = br.one_step(oracle, pb, robust, 1.0, lam)
    po_, ps_, st = oracle.optimize(pb, 1, robust, 1.0, lam, 1)
    assert st["chi2_iter"][0] < st["chi2_init"]                  # the trial was accepted
    assert np.abs(poses - po_).max() <= 1e-9 * np.abs(poses - pb.pose_qt).max()
    assert np.abs(psi - ps_).max() <= 1e-9 * np.abs(psi - pb.psi).max()
    assert (poses[pb.fixed == 1] == pb.pose_qt[pb.fixed == 1]).all()


# ------------------------------------------------------------------------------------------------ route restatement

@pytest.mark.parametrize("m,lo,hi,anchor,want", [
    (1, 11, 11, 10, 0),      # one observer: nothing to complete
    (2, 11, 13, 10, 1),      # np = 1 = max(1, m/2)
    (4, 11, 16, 10, 2),      # np = 2 = m/2, at the limit
    (4, 11, 17, 10, 0),      # np = 3, one past it
    (4, 8, 13, 10, 1),       # anchor inside lo..hi: not one of the frames to add
    (5, 11, 17, 10, 2),      # completed track of exactly 8 slots
    (6, 11, 18, 10, 0),      # would need 9 slots
    (5, 8, 15, 12, 2),       # anchor inside, 1 + span = 8
    (6, 8, 16, 12, 0),       # anchor inside, 1 + span = 9
    (3, 11, 13, 10, 0),      # no gap
])
def test_track_padding(m, lo, hi, anchor, want):
    assert br.track_padding(m, lo, hi, anchor) == want


def test_wave_bounds_and_which_one_binds():
    """nw_max = min(32/k, 40/K, 8).  By arithmetic 40/K never binds alone: with a self edge K = k and 32/k <= 40/K;
    without one K = k + 1 and 40/(k+1) < 32/k only where 8 is smaller still (k <= 3), so it ties at K = 5, 6, 7."""
    table = {}
    for K in range(1, 9):
        for self_edge in (True, False):
            if K == 1 and not self_edge:
                continue
            k = K if self_edge else K - 1
            a, b, c = br.nw_bounds(k, K)
            m = min(a, b, c)
            table[(K, self_edge)] = (m, tuple(n for n, v in (("32/k", a), ("40/K", b), ("8", c)) if v == m))
            assert table[(K, self_edge)][1] != ("40/K",)
    assert table[(8, True)] == (4, ("32/k",)) and table[(8, False)] == (4, ("32/k",))
    assert table[(5, False)] == (8, ("32/k", "40/K", "8")) and table[(6, False)] == (6, ("32/k", "40/K"))
    assert table[(7, False)] == (5, ("32/k", "40/K")) and table[(1, True)] == (8, ("8",))
    assert br.task_waves(3, 3, 9) == 2 and br.task_waves(8, 8, 5) == 2 and br.task_waves(1, 1, 8 * 70) == 64


def test_build_chunk():
    assert br.build_chunk(1000, 132) == 4 and br.build_chunk(132 * 11 * 10, 132) == 10
    assert br.build_chunk(10 ** 6, 132) == 32
    assert br.build_chunk(1000, 132, "1") == 1 and br.build_chunk(1000, 132, "0") == 1 and br.build_chunk(10, 132, "57") == 57


def test_route_of_a_hand_worked_window():
    tracks = [T(0, (1, 2), True, 3), T(0, (1, 2), False, 2), T(1, tuple(range(2, 12)), True, 1),
              T(2, tuple(range(3, 37)), False, 1)]
    pb = br.make_tracks_window(40, tracks, seed=5, unobserved=1)
    # labels: the unobserved landmark takes label 0, the others follow in track order
    r = br.route(pb, 132, "2")
    assert r.chunk == 2
    assert r.order == [1, 2, 3, 4, 5, 6, 7, 0]
    assert r.tasks == [(0, 2), (2, 1), (3, 2)]                 # runs of the self-edge shape, then the anchorless one
    assert [r.task_shape(t) for t in range(3)] == [(3, 3, True, 2), (3, 3, True, 1), (2, 3, False, 2)]
    assert r.gen == [5, 7] and r.K[5] == 11 and r.k[7] == 0    # 11 slots, and the unobserved landmark last
    assert r.long == [6] and r.K[6] == 35 and r.k[6] == 34
    assert r.launches_per_trial(0) == 5
    r = br.route(pb, 132)
    assert r.chunk == 4 and r.tasks == [(0, 3), (3, 2)]


def test_route_orders_by_locality_key_and_sorts_tasks_by_waves():
    tracks = [T(5, (6, 7), True, 1), T(5, (6,), True, 1), T(5, (4, 6), False, 1), T(5, (6, 7), False, 1)]
    r = br.route(br.make_tracks_window(10, tracks, seed=6), 132)
    assert r.order == [1, 0, 2, 3]                             # self edge first, then by K, first and last observer
    tracks = [T(0, (1, 2), True, 3), T(1, (2, 3), True, 9)]
    r = br.route(br.make_tracks_window(10, tracks, seed=7), 132, "32")
    assert r.tasks == [(3, 9), (0, 3)]                         # two waves before one
    # a padded track takes the slot list of its complete neighbours and joins their run
    tracks = [T(3, (4, 5, 6, 7), True, 2), T(3, (4, 5, 7), True, 1), T(3, (4, 5, 6, 7), True, 2)]
    r = br.route(br.make_tracks_window(10, tracks, seed=8), 132, "32")
    assert r.npad == [0, 0, 1, 0, 0] and r.tasks == [(0, 5)]
    r = br.route(br.make_tracks_window(10, tracks, seed=8), 132, "32", pad=False)
    assert len(r.tasks) == 2


def test_persistent_threshold():
    assert br.wave_smem_bytes() == 113408
    assert br.persistent_threshold_tasks(132) == 1056
