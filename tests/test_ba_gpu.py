"""GPU parity tests of the BA path: CUDA (through the C ABI) vs the CPU oracle.

Tolerances: north_star asks 1e-6 relative on pose parameters; intermediate
quantities (chi2, reduced system, solve) are checked much tighter because both
sides are FP64 and differ only in summation order.
"""
import numpy as np
import pytest

from scavislam_b200 import synth

pytestmark = pytest.mark.gpu

POSE_RTOL = 1e-6


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture(scope="module")
def c1():
    return synth.make_config("C1")


@pytest.fixture(scope="module")
def ba(svs):
    b = svs.BundleAdjuster()
    yield b
    b.close()


def test_device_is_hopper(svs):
    info = svs.device_info()
    assert "sm_90" in info, info


def test_chi2_matches_oracle(ba, oracle, c1):
    ba.set_problem(c1)
    for robust in (True, False):
        g = ba.chi2(robust, 1.0)
        o = oracle.chi2(c1, robust, 1.0)
        assert abs(g - o) <= 1e-11 * abs(o), (robust, g, o)


@pytest.mark.parametrize("lam", [50.0, 1e-3])
def test_reduced_system_matches_oracle(ba, oracle, c1, lam):
    ba.set_problem(c1)
    S, bs, chi = ba.reduced_system(True, 1.0, lam)
    So, bso, chio = oracle.reduced_system(c1, True, 1.0, lam)
    assert abs(chi - chio) <= 1e-11 * abs(chio)
    assert _rel(S, So) < 1e-11
    assert _rel(bs, bso) < 1e-10
    assert np.abs(S - S.T).max() <= 1e-9 * np.abs(S).max()


def test_reduced_solve_matches_numpy(ba, c1):
    ba.set_problem(c1)
    S, bs, _ = ba.reduced_system(True, 1.0, 50.0)
    x, failed = ba.solve_reduced(True, 1.0, 50.0)
    assert failed == 0
    xr = np.linalg.solve(S, bs)
    assert _rel(x, xr) < 1e-9


def test_one_iteration_c1(ba, oracle, c1):
    """BASELINE config C1: 10 KF / 500 pt, single GN iteration."""
    ba.set_problem(c1)
    it, st = ba.optimize(1)
    po, pso, sto = oracle.optimize(c1, 1)
    assert it == sto["iterations"] == 1
    assert st["trials_iter"] == sto["trials_iter"]
    assert abs(st["chi2_init"] - sto["chi2_init"]) <= 1e-10 * sto["chi2_init"]
    assert abs(st["chi2_final"] - sto["chi2_final"]) <= 1e-8 * sto["chi2_final"]
    assert _rel(ba.poses(), po) < POSE_RTOL
    assert _rel(ba.points(), pso) < POSE_RTOL


@pytest.mark.parametrize("iters,lam0", [(5, 50.0), (10, 1e-4), (6, 1e5)])
def test_multi_iteration_c1(ba, oracle, c1, iters, lam0):
    ba.set_problem(c1)
    it, st = ba.optimize(iters, True, 1.0, lam0, 5)
    po, pso, sto = oracle.optimize(c1, iters, True, 1.0, lam0, 5)
    assert it == sto["iterations"]
    assert st["trials_iter"] == sto["trials_iter"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    np.testing.assert_allclose(st["lambda_iter"], sto["lambda_iter"], rtol=1e-6)
    assert _rel(ba.poses(), po) < POSE_RTOL
    assert _rel(ba.points(), pso) < POSE_RTOL


def test_rejected_trials_path(ba, oracle):
    """Large perturbation + small lambda0: an iteration with 6 rejected Levenberg trials."""
    pb = synth.make_window(12, 400, seed=100, pose_noise=(0.5, 0.15), depth_noise=0.6)
    ba.set_problem(pb)
    it, st = ba.optimize(8, False, 1.0, 1e-2, 10)
    po, pso, sto = oracle.optimize(pb, 8, False, 1.0, 1e-2, 10)
    assert sum(sto["trials_iter"]) > sto["iterations"], "case does not exercise rejections"
    assert it == sto["iterations"]
    assert st["trials_iter"] == sto["trials_iter"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-6)
    np.testing.assert_allclose(st["lambda_iter"], sto["lambda_iter"], rtol=1e-6)
    assert _rel(ba.poses(), po) < POSE_RTOL


def test_non_robust_and_fixed_pose(ba, oracle, c1):
    pb = c1.copy()
    pb.fixed[0] = 1
    pb.fixed[4] = 1
    ba.set_problem(pb)
    it, st = ba.optimize(3, False, 1.0, 50.0, 5)
    po, pso, sto = oracle.optimize(pb, 3, False, 1.0, 50.0, 5)
    assert it == sto["iterations"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    g = ba.poses()
    assert np.array_equal(g[0], pb.pose_qt[0]) and np.array_equal(g[4], pb.pose_qt[4])
    assert _rel(g, po) < POSE_RTOL


def test_one_call_api_and_reset(ba, oracle, c1):
    it, poses, psi, st = ba.optimise_inner_and_outer_window(c1, 2)
    po, pso, sto = oracle.optimize(c1, 2)
    assert it == 2
    assert _rel(poses, po) < POSE_RTOL and _rel(psi, pso) < POSE_RTOL
    ba.reset_state()
    assert np.array_equal(ba.poses(), c1.pose_qt)
    assert np.array_equal(ba.points(), c1.psi)
    it2, st2 = ba.optimize(2)
    assert _rel(ba.poses(), po) < POSE_RTOL


def test_empty_and_degenerate(ba, svs):
    pb = synth.make_window(4, 0, seed=5)   # no landmarks, no edges
    ba.set_problem(pb)
    it, st = ba.optimize(2)
    assert it == 1          # rho == 0 -> Terminate after the first iteration, like g2o
    assert np.allclose(ba.poses(), pb.pose_qt)
    pb0 = synth.make_window(0, 0, seed=5)
    ba.set_problem(pb0)
    it, _ = ba.optimize(2)
    assert it == -1   # g2o: 0 vertices to optimize


def test_invalid_inputs_rejected(ba, svs, c1):
    pb = c1.copy()
    pb.e_pose[3] = 10_000
    with pytest.raises(svs.SvsError):
        ba.set_problem(pb)
    pb = c1.copy()
    pb.e_anchor[0] = (pb.e_anchor[0] + 1) % pb.P   # two anchors for one point
    with pytest.raises(svs.SvsError):
        ba.set_problem(pb)


def test_c2_full_size_parity(ba, oracle):
    """BASELINE config C2: 200 KF / 20k pt, 10 iterations (oracle takes ~0.5 s)."""
    pb = synth.make_config("C2")
    ba.set_problem(pb)
    it, st = ba.optimize(10)
    po, pso, sto = oracle.optimize(pb, 10)
    assert it == sto["iterations"] == 10
    assert st["trials_iter"] == sto["trials_iter"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    assert _rel(ba.poses(), po) < POSE_RTOL
    assert _rel(ba.points(), pso) < POSE_RTOL
    # size-independent property: chi2 decreases monotonically over accepted iterations
    assert all(a >= b for a, b in zip([st["chi2_init"]] + st["chi2_iter"][:-1], st["chi2_iter"]))


# ---------------------------------------------------------------- structure variety (generic code paths)

def _add_constraints(pb, pairs, seed=0):
    """Extra pose-pose constraints (e.g. loop closures) with the measurement taken from the truth."""
    from oracle import pyoracle as po
    rng = np.random.default_rng(seed)
    ci, cj, cT, cL = list(pb.c_i), list(pb.c_j), list(pb.c_T), list(pb.c_Lambda)
    for (i, j) in pairs:
        T = po.se3_mul(po.se3_exp(rng.normal(0, 1e-3, 6)), po.se3_mul(pb.truth_pose_qt[j], po.se3_inv(pb.truth_pose_qt[i])))
        lam = np.diag([4e4] * 3 + [1e5] * 3).reshape(36)
        ci.append(i); cj.append(j); cT.append(T); cL.append(lam)
    pb.c_i = np.asarray(ci, np.int32); pb.c_j = np.asarray(cj, np.int32)
    pb.c_T = np.asarray(cT, np.float64).reshape(-1, 7); pb.c_Lambda = np.asarray(cL, np.float64).reshape(-1, 36)
    pb.C = len(ci)
    return pb


def _check_against_oracle(ba, oracle, pb, iters=4):
    ba.set_problem(pb)
    it, st = ba.optimize(iters)
    po_, ps_, sto = oracle.optimize(pb, iters)
    assert it == sto["iterations"] and st["trials_iter"] == sto["trials_iter"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    assert _rel(ba.poses(), po_) < POSE_RTOL and _rel(ba.points(), ps_) < POSE_RTOL
    return st


def test_long_tracks_use_the_generic_build_kernel(ba, oracle):
    """Tracks of up to 14 frames (> 8): one-warp-per-landmark path of the fused kernel."""
    pb = synth.make_window(30, 1500, seed=31, T=14)
    st = _check_against_oracle(ba, oracle, pb)
    assert st["max_track"] > 8


def test_tracks_longer_than_32_frames(ba, oracle):
    """A slowly moving camera: tracks of up to 50 frames + anchor.  The reference adds one edge per in-window
    frame of vis_set without any cap (slam_graph.cpp:1001-1027): the streaming kernel k_build_long takes them."""
    pb = synth.make_window(70, 900, seed=36, T=50)
    ba.set_problem(pb)
    S, bs, chi = ba.reduced_system(True, 1.0, 50.0)
    So, bso, chio = oracle.reduced_system(pb, True, 1.0, 50.0)
    assert abs(chi - chio) <= 1e-11 * abs(chio)
    assert _rel(S, So) < 1e-11 and _rel(bs, bso) < 1e-10
    x, failed = ba.solve_reduced(True, 1.0, 50.0)
    assert failed == 0 and _rel(x, np.linalg.solve(S, bs)) < 1e-9
    st = _check_against_oracle(ba, oracle, pb)
    assert st["max_track"] > 33


def test_loop_closures_break_the_band(ba, oracle):
    """Constraints between far-apart keyframes: no two-ended split, minimum-degree order with fill."""
    pb = _add_constraints(synth.make_window(60, 3000, seed=32), [(0, 59), (59, 0), (5, 40), (12, 55), (20, 58)])
    st = _check_against_oracle(ba, oracle, pb)
    assert st["nnzb_L"] > st["nnzb_S"]          # fill-in happened


def test_dense_reduced_system_uses_the_general_solver(ba, oracle):
    """All-to-all pose constraints: every factor column is wider than the shared-memory ring share."""
    P = 140
    pb = synth.make_window(P, 1400, seed=33)
    pairs = [(i, j) for i in range(P) for j in range(i + 1, P) if (i * 7 + j * 3) % 5 == 0 or j - i > 100]
    pb = _add_constraints(pb, pairs)
    st = _check_against_oracle(ba, oracle, pb, iters=3)
    assert st["nnzb_L"] > 0.8 * P * (P + 1) / 2


def test_two_ended_split_is_used_and_equals_the_chain(ba, oracle, svs):
    import os
    pb = synth.make_window(90, 4000, seed=34)
    ba.set_problem(pb)
    it, st = ba.optimize(3)
    poses = ba.poses()
    os.environ["SVS_SOLVE_CHAIN"] = "1"
    try:
        b2 = svs.BundleAdjuster()
        b2.set_problem(pb)
        it2, st2 = b2.optimize(3)
        assert _rel(b2.poses(), poses) < 1e-9
        np.testing.assert_allclose(st2["chi2_iter"], st["chi2_iter"], rtol=1e-10)
        b2.close()
    finally:
        del os.environ["SVS_SOLVE_CHAIN"]


# ---------------------------------------------------------------- tracks with holes: zero-weight padding (set_problem)

def test_tracks_with_holes_are_completed_without_changing_any_sum(ba, oracle, svs):
    """set_problem completes a track with a few drop-outs with zero-weight edges so that it shares the slot list of its
    neighbours (ba_host.cu, 'Track padding').  The reduced system, chi2 and the LM trajectory must not move: against
    the oracle (which knows nothing of the padding) and against the same library with SVS_BUILD_NO_PAD=1."""
    import os
    pb = synth.with_dropouts(synth.make_window(40, 3000, seed=41), 0.2, seed=3)
    ba.set_problem(pb)
    S, bs, chi = ba.reduced_system(True, 1.0, 50.0)
    So, bso, chio = oracle.reduced_system(pb, True, 1.0, 50.0)
    assert abs(chi - chio) <= 1e-11 * abs(chio)
    assert _rel(S, So) < 1e-11 and _rel(bs, bso) < 1e-10
    st = _check_against_oracle(ba, oracle, pb, iters=5)
    assert st["num_point_edges"] == pb.E          # the caller's count, not the padded one
    poses = ba.poses()
    os.environ["SVS_BUILD_NO_PAD"] = "1"
    try:
        b2 = svs.BundleAdjuster()
        b2.set_problem(pb)
        S2, bs2, chi2 = b2.reduced_system(True, 1.0, 50.0)
        it2, st2 = b2.optimize(5)
        assert _rel(S, S2) < 1e-12 and _rel(bs, bs2) < 1e-11 and abs(chi - chi2) <= 1e-12 * abs(chi2)
        assert _rel(b2.poses(), poses) < 1e-9
        b2.close()
    finally:
        del os.environ["SVS_BUILD_NO_PAD"]


def test_padding_edges_never_evaluate_their_projection(ba, oracle):
    """A padding edge names a frame that never saw the point.  Here that frame looks the other way (every point is
    BEHIND it, depth <= 0 in its coordinates): evaluating the projection would put inf/NaN into the sums."""
    pb = synth.make_window(12, 600, seed=43)
    hole = 5
    keep = (pb.e_pose != hole) & (pb.e_anchor != hole)     # frame 5 observes nothing and anchors nothing that is observed
    out = pb.copy()
    for k in ("e_point", "e_pose", "e_anchor", "e_obs", "e_info"):
        setattr(out, k, np.ascontiguousarray(getattr(pb, k)[keep]))
    out.E = int(keep.sum())
    # turn frame 5 by 180 degrees about its y axis: T' = Ry(pi) T  (q' = (0,1,0,0) * q, t' = Ry t), and fix it
    q, t = out.pose_qt[hole, :4].copy(), out.pose_qt[hole, 4:].copy()
    x, y, z, w = q
    out.pose_qt[hole, :4] = np.array([z, w, -x, -y])        # (0,1,0,0) * (x,y,z,w)
    out.pose_qt[hole, 4:] = np.array([-t[0], t[1], -t[2]])
    out.fixed = out.fixed.copy()
    out.fixed[hole] = 1
    ck = (out.c_i != hole) & (out.c_j != hole)               # its pose-pose constraints go too
    out.c_i, out.c_j, out.c_T, out.c_Lambda = out.c_i[ck].copy(), out.c_j[ck].copy(), out.c_T[ck].copy(), out.c_Lambda[ck].copy()
    out.C = int(ck.sum())
    spans = 0
    for l in range(out.L):
        fr = np.sort(out.e_pose[(out.e_point == l) & (out.e_pose != out.e_anchor)])
        spans += int(fr.size >= 2 and fr[0] < hole < fr[-1])
    assert spans > 20                                        # tracks that do span the hole exist
    ba.set_problem(out)
    S, bs, chi = ba.reduced_system(True, 1.0, 50.0)
    So, bso, chio = oracle.reduced_system(out, True, 1.0, 50.0)
    assert np.isfinite(S).all() and np.isfinite(bs).all() and np.isfinite(chi)
    assert abs(chi - chio) <= 1e-11 * abs(chio) and _rel(S, So) < 1e-11 and _rel(bs, bso) < 1e-10
    _check_against_oracle(ba, oracle, out, iters=3)


# ---------------------------------------------------------------- C2-sized structure variants (bench extras)

def test_c2_with_visibility_dropouts_full_size(ba, oracle):
    """C2 with 20 % of the observations missing at random: tracks with holes, chunk-of-one tasks."""
    pb = synth.with_dropouts(synth.make_config("C2"), 0.2, seed=1)
    _check_against_oracle(ba, oracle, pb, iters=10)


def test_c2_with_loop_closures_full_size(ba, oracle):
    """C2 plus 10 loop-closure constraints between far-apart keyframes: the band is broken."""
    pb = synth.with_loop_closures(synth.make_config("C2"), 10, seed=1)
    st = _check_against_oracle(ba, oracle, pb, iters=10)
    assert st["nnzb_L"] > st["nnzb_S"]
