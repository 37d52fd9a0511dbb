"""svs_ba_covariance (marginal covariances of the BA window) against the dense inverse of the oracle's full
Gauss-Newton system at the device's accepted state.

The reference: oracle.full_system(pb, robust, delta) = H over (poses, landmarks) with pb's state replaced by
ba.poses() / ba.points(); lambda I added to the whole diagonal; the rows and columns of fixed poses (and of landmarks
without edges) dropped; np.linalg.inv.  Pose blocks, pose pairs and landmark blocks are each compared to <= 1e-8 of the
largest entry of their kind.  Every full H stays below about 5 000 rows.

The reduced system is summed with FP64 atomics by the build kernels, so two builds of one state agree only to the last
bits; checks of repeated calls use a tolerance instead of bit equality for that reason.
"""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest

from scavislam_b200 import synth, synth_graph

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-8


@pytest.fixture(scope="module")
def ba(svs):
    b = svs.BundleAdjuster()
    yield b
    b.close()


def _fixed(pb, *poses):
    out = pb.copy()
    out.fixed = np.zeros(pb.P, np.uint8)
    for p in poses:
        out.fixed[p] = 1
    return out


def _dense_reference(oracle, ba, pb, robust, lam, pairs=()):
    """(pose blocks [P,6,6], pair blocks [n,6,6], landmark blocks [L,3,3]) of the dense inverse; zero where the
    variable is not free."""
    st = pb.copy()
    st.pose_qt = ba.poses()
    st.psi = ba.points()
    H, _, _ = oracle.full_system(st, robust, 1.0)
    P, L = pb.P, pb.L
    H = H + lam * np.eye(H.shape[0])
    has_edges = np.zeros(L, bool)
    has_edges[pb.e_point] = True
    free_pose = pb.fixed == 0
    keep = np.concatenate([np.repeat(free_pose, 6), np.repeat(has_edges, 3)])
    Hinv = np.zeros_like(H)
    Hinv[np.ix_(keep, keep)] = np.linalg.inv(H[np.ix_(keep, keep)])
    pose = np.array([Hinv[6 * p:6 * p + 6, 6 * p:6 * p + 6] for p in range(P)])
    pair = np.array([Hinv[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs]).reshape(-1, 6, 6)
    o = 6 * P
    point = np.array([Hinv[o + 3 * l:o + 3 * l + 3, o + 3 * l:o + 3 * l + 3] for l in range(L)]).reshape(-1, 3, 3)
    return pose, pair, point


def _close(got, ref, what):
    scale = max(np.abs(ref).max(), 1e-300)
    err = np.abs(got - ref).max() / scale
    assert err <= TOL, f"{what}: {err:.3e} of the largest entry"


def _check(ba, oracle, pb, robust=True, lam=0.0, pairs=(), iters=0):
    ba.set_problem(pb)
    if iters:
        ba.optimize(iters, robust)
    pose, pair, point, rc, st = ba.covariance(robust, 1.0, lam, pairs)
    assert rc == 0
    rp, rq, rl = _dense_reference(oracle, ba, pb, robust, lam, pairs)
    _close(pose, rp, "pose blocks")
    if len(pairs):
        _close(pair, rq, "pose pairs")
    _close(point, rl, "landmark blocks")
    assert np.array_equal(point, point.transpose(0, 2, 1))
    for p in np.nonzero(pb.fixed)[0]:
        assert not pose[p].any()
    assert st["P"] == pb.P and st["L"] == pb.L
    return pose, pair, point, st


@pytest.mark.parametrize("robust", [True, False])
def test_c1_optimised_with_a_fixed_pose(ba, oracle, robust):
    _check(ba, oracle, _fixed(synth.make_config("C1"), 0), robust=robust, iters=4)


def test_c1_without_fixed_pose_damped(ba, oracle):
    _check(ba, oracle, synth.make_config("C1"), lam=1e-3)


def test_pose_pairs_inside_and_outside_the_pattern(ba, oracle):
    pb = _fixed(synth.make_window(40, 1200, seed=51), 0, 17)
    pairs = [(5, 6), (6, 5), (12, 9), (2, 35), (35, 2), (10, 30), (30, 10), (0, 20), (17, 3), (39, 39)]
    pose, pair, point, st = _check(ba, oracle, pb, pairs=pairs, iters=2)
    assert st["n_cols_solved"] > 0 and st["n_pairs_in_pattern"] > 0
    for k, (i, j) in enumerate(pairs):
        if pb.fixed[i] or pb.fixed[j]:
            assert not pair[k].any()
    assert np.array_equal(pair[3], pair[4].T) or np.abs(pair[3] - pair[4].T).max() <= TOL * np.abs(pair).max()
    np.testing.assert_array_equal(pair[9], pose[39])


def test_tracks_of_9_to_32_slots(ba, oracle):
    _check(ba, oracle, _fixed(synth.make_window(30, 1500, seed=31, T=14), 0))


def test_tracks_longer_than_32_slots(ba, oracle):
    pb = _fixed(synth.make_window(70, 900, seed=36, T=50), 0)
    _check(ba, oracle, pb)
    assert ba.lm_stats()["max_track"] > 33


def test_visibility_dropouts(ba, oracle):
    pb = _fixed(synth.with_dropouts(synth.make_window(40, 1200, seed=41), 0.2, seed=3), 0)
    _check(ba, oracle, pb, iters=2)


def test_loop_closures_two_ended_with_separator(ba, oracle):
    pb = _fixed(synth.with_loop_closures(synth.make_window(60, 1000, seed=32), 3, seed=1), 0)
    _, _, _, st = _check(ba, oracle, pb, pairs=[(0, 59), (3, 45)])
    assert st["nbranch"] == 2


def test_dense_pattern_on_the_general_solver(ba, oracle):
    """Pose-pose constraints between all pairs: the factor's columns are wider than k_solve's shared-memory ring."""
    P = 150
    pb = synth.make_window(P, 700, seed=33)
    pairs = [(i, j) for i in range(P) for j in range(i + 1, P)]
    ci, cj, cT, cL = list(pb.c_i), list(pb.c_j), list(pb.c_T), list(pb.c_Lambda)
    lam = np.diag([4e4] * 3 + [1e5] * 3).reshape(36)
    for i, j in pairs:
        ci.append(i); cj.append(j); cT.append(pb.c_T[0]); cL.append(lam)
    pb.c_i, pb.c_j = np.asarray(ci, np.int32), np.asarray(cj, np.int32)
    pb.c_T, pb.c_Lambda = np.asarray(cT).reshape(-1, 7), np.asarray(cL).reshape(-1, 36)
    pb.C = len(ci)
    _, _, _, st = _check(ba, oracle, _fixed(pb, 0), pairs=[(1, 149), (70, 2)])
    assert st["general"] == 1


def test_single_chain_solver(svs, oracle):
    os.environ["SVS_SOLVE_CHAIN"] = "1"
    try:
        b = svs.BundleAdjuster()
        _, _, _, st = _check(b, oracle, _fixed(synth.make_window(60, 1000, seed=34), 0), pairs=[(2, 50)])
        assert st["nbranch"] == 1 and st["general"] == 0
        b.close()
    finally:
        del os.environ["SVS_SOLVE_CHAIN"]


def test_repeated_calls_and_the_lm_state(ba, svs):
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    poses, points, lm = ba.poses(), ba.points(), ba.lm_stats()
    a = ba.covariance(True, 1.0, 0.0, [(1, 8)])
    b = ba.covariance(True, 1.0, 0.0, [(1, 8)])
    for x, y in zip(a[:3], b[:3]):
        assert np.abs(x - y).max() <= 1e-10 * np.abs(x).max()   # FP64 atomics of the build: last bits only
    # the accepted state and the Levenberg control block are left exactly as they were
    assert np.array_equal(ba.poses(), poses) and np.array_equal(ba.points(), points)
    assert ba.lm_stats() == lm
    ba.optimize(2)
    with_cov = ba.poses(), ba.points()
    ba.set_problem(pb)
    ba.optimize(2)
    ba.optimize(2)
    for x, y in zip(with_cov, (ba.poses(), ba.points())):
        assert np.abs(x - y).max() <= 1e-10 * np.abs(y).max()


def test_window_from_the_device_map_gives_the_same_covariances(svs):
    pb = synth.make_window(30, 3000, seed=6)
    m, win, act = synth_graph.make_map(pb, seed=6)
    dm, b1, b2 = svs.DeviceMap(), svs.BundleAdjuster(), svs.BundleAdjuster()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    fixed = np.zeros(len(win), np.uint8)
    fixed[0] = 1
    E = dm.set_problem(b1, win, act, pb.cam, fixed=fixed, c_i=pb.c_i, c_j=pb.c_j, c_T=pb.c_T, c_Lambda=pb.c_Lambda)
    ep, es, ea, obs, info = dm.last_edges(E)
    pa = dataclasses.replace(pb, E=E, pose_qt=b1.poses(), psi=b1.points(), fixed=fixed, e_point=ep, e_pose=es,
                             e_anchor=ea, e_obs=obs, e_info=info)
    b2.set_problem(pa)
    pairs = [(3, 4), (1, 25)]
    r1, r2 = b1.covariance(True, 1.0, 0.0, pairs), b2.covariance(True, 1.0, 0.0, pairs)
    assert r1[3] == r2[3] == 0
    for x, y in zip(r1[:3], r2[:3]):
        assert np.abs(x - y).max() <= 1e-10 * np.abs(y).max()
    for h in (dm, b1, b2):
        h.close()


def test_c2_pose_blocks_against_the_reduced_system(ba):
    pb = _fixed(synth.make_config("C2"), 0)
    ba.set_problem(pb)
    ba.optimize(3)
    lam = 1e-4
    S, _, _ = ba.reduced_system(True, 1.0, lam)
    pose, pair, point, rc, st = ba.covariance(True, 1.0, lam, [(0, 199), (20, 150)])
    assert rc == 0 and st["n_cols_solved"] > 0
    Z = np.linalg.inv(S)
    ref = np.array([Z[6 * p:6 * p + 6, 6 * p:6 * p + 6] for p in range(pb.P)])
    ref[0] = 0
    _close(pose, ref, "C2 pose blocks")
    _close(pair[1], Z[120:126, 900:906], "C2 far pair")
    assert not pair[0].any()
    assert np.isfinite(point).all() and np.array_equal(point, point.transpose(0, 2, 1))
    assert (np.linalg.eigvalsh(point) > 0).all()


def test_errors(ba, svs):
    b = svs.BundleAdjuster()
    with pytest.raises(svs.SvsError) as e:
        b.covariance()
    assert e.value.rc == -4   # SVS_ERR_STATE: no problem set
    b.close()
    pb = synth.make_config("C1")
    ba.set_problem(pb)
    with pytest.raises(svs.SvsError) as e:
        ba.covariance(True, 1.0, 0.0)   # no fixed pose, lambda = 0: H is singular
    assert e.value.rc == -1 and "singular" in str(e.value)
    ba.set_problem(_fixed(pb, 0))
    for bad in ([(0, pb.P)], [(-1, 2)]):
        with pytest.raises(svs.SvsError) as e:
            ba.covariance(True, 1.0, 0.0, bad)
        assert e.value.rc == -1
    with pytest.raises(svs.SvsError):
        ba.covariance(True, 1.0, -1.0)
    one = np.zeros(1, np.int32)
    dp = C.POINTER(C.c_double)
    ip = C.POINTER(C.c_int)
    for pi, pj, out in ((None, one, np.zeros(36)), (one, None, np.zeros(36)), (one, one, None)):
        rc = svs.lib().svs_ba_covariance(ba._h, 1, 1.0, 0.0, None, 1,
                                         pi.ctypes.data_as(ip) if pi is not None else None,
                                         pj.ctypes.data_as(ip) if pj is not None else None,
                                         out.ctypes.data_as(dp) if out is not None else None, None, None)
        assert rc == -1
    assert ba.covariance(True, 1.0, 0.0)[3] == 0   # the handle stays usable


def _write_window(path, pb, iters, robust, lam, pairs):
    xyz = np.stack([pb.psi[:, 0] / pb.psi[:, 2], pb.psi[:, 1] / pb.psi[:, 2], 1.0 / pb.psi[:, 2]], -1)
    pi = np.array([p[0] for p in pairs], np.int32)
    pj = np.array([p[1] for p in pairs], np.int32)
    with open(path, "wb") as f:
        np.array([pb.P, pb.L, pb.E, pb.C, len(pairs), iters, int(robust)], np.int32).tofile(f)
        np.append(np.asarray(pb.cam, np.float64), lam).tofile(f)
        for a, t in ((pb.pose_qt, np.float64), (pb.fixed, np.int32), (xyz, np.float64), (pb.e_point, np.int32),
                     (pb.e_pose, np.int32), (pb.e_anchor, np.int32), (pb.e_obs, np.float64), (pb.e_info, np.float64),
                     (pb.c_i, np.int32), (pb.c_j, np.int32), (pb.c_T, np.float64), (pb.c_Lambda, np.float64),
                     (pi, np.int32), (pj, np.int32)):
            np.ascontiguousarray(a, t).tofile(f)


def test_cpp_compute_marginals_matches_the_c_abi(ba, tmp_path):
    exe = str(tmp_path / "ba_covariance_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ba_covariance_main.cpp"), "-o", exe, "-L", lib_dir,
                           "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    pb = _fixed(synth.make_config("C1"), 0)
    pairs = [(2, 7), (9, 1), (0, 3)]
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    _write_window(inp, pb, 3, True, 0.0, pairs)
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
    got = np.fromfile(out, np.float64)
    P, L, n = pb.P, pb.L, len(pairs)
    g_pose, g_pair, g_point = (got[:36 * P].reshape(P, 6, 6), got[36 * P:36 * (P + n)].reshape(n, 6, 6),
                               got[36 * (P + n):].reshape(L, 3, 3))
    ba.set_problem(pb)
    ba.optimize(3, True, 1.0, 50.0, 5)   # what StereoGraph::optimize runs: lambda0 = 50, 5 trials
    pose, pair, point, rc, _ = ba.covariance(True, 1.0, 0.0, pairs)
    assert rc == 0
    for x, y, what in ((g_pose, pose, "pose"), (g_pair, pair, "pairs"), (g_point, point, "landmarks")):
        assert np.abs(x - y).max() <= 1e-8 * np.abs(y).max(), what
