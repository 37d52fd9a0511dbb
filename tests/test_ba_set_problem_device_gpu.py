"""svs_ba_set_problem_device: a window whose arrays lie in GPU memory is analysed on the device (ba_structure.cu).

Every window goes in twice: as CUDA tensors, with its edges in a random order and its landmarks relabelled so that they
are not sorted by anchor, and as the same numpy arrays through the host analysis of svs_ba_set_problem.  Both must
give the same reduced system, chi2, block counts and Levenberg trajectory (FP64 atomics in the Schur build leave the
last bits free), and the oracle's result to 1e-6 where the other BA tests compare with it."""
import dataclasses

import numpy as np
import pytest

from scavislam_b200 import synth, synth_graph

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300) if np.size(b) else 0.0


def _shuffled(pb, seed=0):
    """The same window with the edges in a random order and the landmarks relabelled at random."""
    rng = np.random.default_rng(seed)
    out = pb.copy()
    if pb.L:
        lp = rng.permutation(pb.L).astype(np.int32)                # old landmark l -> new label lp[l]
        out.psi = np.ascontiguousarray(pb.psi[np.argsort(lp)])
        out.e_point = lp[pb.e_point].astype(np.int32)
    ep = rng.permutation(pb.E)
    for k in ("e_point", "e_pose", "e_anchor", "e_obs", "e_info"):
        setattr(out, k, np.ascontiguousarray(getattr(out, k)[ep]))
    return out


def _cuda(pb):
    """The window as CUDA tensors (int32 indices, uint8 fixed flags, float64 numbers)."""
    kw = {}
    for k, v in pb.__dict__.items():
        kw[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and k not in ("cam", "truth_pose_qt", "truth_psi") else v
    return dataclasses.replace(pb, **kw)


def _add_constraints(pb, pairs, seed=0):
    from oracle import pyoracle as po
    rng = np.random.default_rng(seed)
    ci, cj, cT, cL = list(pb.c_i), list(pb.c_j), list(pb.c_T), list(pb.c_Lambda)
    for (i, j) in pairs:
        T = po.se3_mul(po.se3_exp(rng.normal(0, 1e-3, 6)), po.se3_mul(pb.truth_pose_qt[j], po.se3_inv(pb.truth_pose_qt[i])))
        ci.append(i); cj.append(j); cT.append(T); cL.append(np.diag([4e4] * 3 + [1e5] * 3).reshape(36))
    pb.c_i = np.asarray(ci, np.int32); pb.c_j = np.asarray(cj, np.int32)
    pb.c_T = np.asarray(cT, np.float64).reshape(-1, 7); pb.c_Lambda = np.asarray(cL, np.float64).reshape(-1, 36)
    pb.C = len(ci)
    return pb


def _with_unobserved(pb, n=40, seed=0):
    rng = np.random.default_rng(seed)
    out = pb.copy()
    out.psi = np.concatenate([pb.psi, np.stack([rng.uniform(-.2, .2, n), rng.uniform(-.2, .2, n), rng.uniform(.1, .5, n)], 1)])
    out.L = pb.L + n
    return out


def _fixed(pb, *idx):
    out = pb.copy()
    out.fixed = out.fixed.copy()
    out.fixed[list(idx)] = 1
    return out


def _compare(svs, oracle, pb, iters=4, flags=0, pairs=None, use_oracle=True, seed=0):
    """Device set-up of the shuffled window against the host set-up of the same arrays; returns the device stats."""
    q = _shuffled(pb, seed)
    dev, host = svs.BundleAdjuster(flags=flags), svs.BundleAdjuster(flags=flags)
    try:
        if pairs is not None:
            dev.set_structure(pairs); host.set_structure(pairs)
        dev.set_problem(_cuda(q)); host.set_problem(q)
        if q.P:
            S, b, chi = dev.reduced_system(True, 1.0, 50.0)
            S2, b2, chi2 = host.reduced_system(True, 1.0, 50.0)
            assert np.abs(S - S2).max() <= 1e-12 * np.abs(S2).max()
            assert np.abs(b - b2).max() <= 1e-12 * max(np.abs(b2).max(), 1e-300)
            assert abs(chi - chi2) <= 1e-12 * abs(chi2)
        assert abs(dev.chi2() - host.chi2()) <= 1e-12 * abs(host.chi2())
        dev.reset_state(); host.reset_state()
        it, st = dev.optimize(iters)
        it2, st2 = host.optimize(iters)
        assert it == it2
        for k in ("nnzb_S", "nnzb_L", "max_track", "num_point_edges", "num_points", "num_frames"):
            assert st[k] == st2[k], (k, st[k], st2[k])
        if it <= 0:
            return st
        assert st["trials_iter"] == st2["trials_iter"]
        np.testing.assert_allclose(st["chi2_iter"], st2["chi2_iter"], rtol=1e-10)
        assert _rel(dev.poses(), host.poses()) < 1e-9 and _rel(dev.points(), host.points()) < 1e-9
        if use_oracle:
            po_, ps_, sto = oracle.optimize(q, iters)
            assert it == sto["iterations"] and st["trials_iter"] == sto["trials_iter"]
            assert _rel(dev.poses(), po_) < 1e-6 and _rel(dev.points(), ps_) < 1e-6
        return st
    finally:
        dev.close(); host.close()


WINDOWS = {
    "c1": lambda: synth.make_config("C1"),
    "c1_fixed_pose": lambda: _fixed(synth.make_config("C1"), 3),
    "30_keyframes": lambda: synth.make_window(30, 1500, seed=7),
    "dropouts": lambda: synth.with_dropouts(synth.make_window(40, 3000, seed=41), 0.2, seed=3),
    "tracks_9_to_32": lambda: synth.make_window(30, 1500, seed=31, T=14),
    "tracks_over_32": lambda: synth.make_window(70, 900, seed=36, T=50),
    "loop_closures": lambda: _add_constraints(synth.make_window(60, 3000, seed=32), [(0, 59), (59, 0), (5, 40), (12, 55), (20, 58)]),
    "two_ended_with_separator": lambda: synth.with_loop_closures(synth.make_window(90, 4000, seed=34), 2, seed=2),
    "unobserved_landmarks": lambda: _with_unobserved(synth.make_config("C1")),
    "no_constraints": lambda: dataclasses.replace(synth.make_window(12, 400, seed=9), C=0, c_i=np.zeros(0, np.int32),
                                                  c_j=np.zeros(0, np.int32), c_T=np.zeros((0, 7)), c_Lambda=np.zeros((0, 36))),
}


@pytest.mark.parametrize("name", sorted(WINDOWS))
def test_device_set_up_equals_the_host_set_up(svs, oracle, name):
    st = _compare(svs, oracle, WINDOWS[name]())
    if name == "tracks_9_to_32":
        assert st["max_track"] > 8
    if name == "tracks_over_32":
        assert st["max_track"] > 33
    if name == "loop_closures":
        assert st["nnzb_L"] > st["nnzb_S"]


def test_dense_window_on_the_general_solver(svs, oracle):
    P = 140
    pairs = [(i, j) for i in range(P) for j in range(i + 1, P) if (i * 7 + j * 3) % 5 == 0 or j - i > 100]
    st = _compare(svs, oracle, _add_constraints(synth.make_window(P, 1400, seed=33), pairs), iters=3)
    assert st["nnzb_L"] > 0.8 * P * (P + 1) / 2


@pytest.mark.parametrize("flag", ["SVS_BA_SKIP_SELF_ANCHOR_HESSIAN", "SVS_BA_NATURAL_ORDER"])
def test_flags(svs, oracle, flag):
    _compare(svs, oracle, synth.make_window(30, 1500, seed=8), flags=getattr(svs, flag), use_oracle=False)


def test_prescribed_structure_pairs_switch_padding_off(svs, oracle):
    pb = synth.with_dropouts(synth.make_window(20, 1000, seed=12), 0.2, seed=4)
    pairs = np.array([(0, 19), (3, 15)], np.int32)
    _compare(svs, oracle, pb, pairs=pairs, use_oracle=False)


def test_empty_windows(svs, oracle):
    _compare(svs, oracle, synth.make_window(4, 0, seed=5), iters=2, use_oracle=False)      # E = 0
    _compare(svs, oracle, synth.make_window(0, 0, seed=5), iters=2, use_oracle=False)      # nothing at all
    one = synth.make_window(3, 50, seed=5)                                                  # P = 1: anchors only
    keep = (one.e_pose == 0) & (one.e_anchor == 0)
    one = dataclasses.replace(one, P=1, pose_qt=one.pose_qt[:1].copy(), fixed=one.fixed[:1].copy(), E=int(keep.sum()),
                              e_point=one.e_point[keep].copy(), e_pose=one.e_pose[keep].copy(), e_anchor=one.e_anchor[keep].copy(),
                              e_obs=one.e_obs[keep].copy(), e_info=one.e_info[keep].copy(), C=0, c_i=np.zeros(0, np.int32),
                              c_j=np.zeros(0, np.int32), c_T=np.zeros((0, 7)), c_Lambda=np.zeros((0, 36)))
    _compare(svs, oracle, one, iters=2, use_oracle=False)


@pytest.mark.parametrize("variant", ["plain", "dropouts", "loop_closures"])
def test_c2_full_size(svs, oracle, variant):
    pb = synth.make_config("C2")
    if variant == "dropouts":
        pb = synth.with_dropouts(pb, 0.2, seed=1)
    if variant == "loop_closures":
        pb = synth.with_loop_closures(pb, 10, seed=1)
    _compare(svs, oracle, pb, iters=10, use_oracle=False)


def _run(ba, pb, iters=3):
    ba.set_problem(pb)
    it, st = ba.optimize(iters)
    return it, st, ba.poses(), ba.points()


def _same_result(a, b):
    assert a[0] == b[0] and a[1]["trials_iter"] == b[1]["trials_iter"]
    np.testing.assert_allclose(a[1]["chi2_iter"], b[1]["chi2_iter"], rtol=1e-10)
    assert _rel(a[2], b[2]) < 1e-9 and _rel(a[3], b[3]) < 1e-9


def test_structure_reuse(svs):
    """The same index tensors with new numbers reuse the structure; a different structure on the same handle (same
    pattern, then a new pattern) is analysed afresh."""
    pb = _shuffled(synth.make_window(30, 1500, seed=14), 1)
    moved = pb.copy()
    moved.pose_qt[:, 4:] += 1e-3
    moved.psi[:, 2] *= 1.01
    moved.e_obs += 0.05
    same_pattern = synth.with_dropouts(pb, 0.01, seed=2)     # fewer edges; the pose pairs are (almost surely) kept
    new_pattern = _add_constraints(pb.copy(), [(0, 29)])
    ba = svs.BundleAdjuster()
    _run(ba, _cuda(pb))
    for q in (moved, same_pattern, new_pattern, moved):
        got = _run(ba, _cuda(q))
        fresh = svs.BundleAdjuster()
        _same_result(got, _run(fresh, _cuda(q)))
        fresh.close()
    ba.close()


def test_invalid_inputs_get_the_host_codes(svs):
    pb = synth.make_window(10, 300, seed=15)
    bad = []
    q = pb.copy(); q.e_pose[3] = 10_000; bad.append(q)                       # edge index out of range
    q = pb.copy(); q.e_point[5] = -1; bad.append(q)
    q = pb.copy(); q.e_anchor[0] = (q.e_anchor[0] + 1) % q.P; bad.append(q)  # two anchors for one point
    q = pb.copy(); i = int(np.nonzero(q.e_pose != q.e_anchor)[0][0])         # a point observed twice by one frame
    for k in ("e_point", "e_pose", "e_anchor", "e_obs", "e_info"):
        setattr(q, k, np.concatenate([getattr(q, k), getattr(q, k)[i:i + 1]]))
    q.E += 1; bad.append(q)
    if pb.C:
        q = pb.copy(); q.c_j = q.c_j.copy(); q.c_j[0] = q.c_i[0]; bad.append(q)   # pose-pose edge onto itself
    dev, host = svs.BundleAdjuster(), svs.BundleAdjuster()
    for q in bad:
        with pytest.raises(svs.SvsError) as e_host:
            host.set_problem(q)
        with pytest.raises(svs.SvsError) as e_dev:
            dev.set_problem(_cuda(q))
        assert e_dev.value.rc == e_host.value.rc and str(e_dev.value) == str(e_host.value)
    # a host pointer given to the device entry point
    import ctypes as C
    k = svs.BundleAdjuster._arrays(pb)
    args, cam = svs.BundleAdjuster._prob_args(pb, k)
    rc = svs.lib().svs_ba_set_problem_device(dev._h, *[C.cast(a, C.c_void_p) if isinstance(a, C._Pointer) else a for a in args])
    assert rc == -1, rc   # SVS_ERR_INVALID, before anything is enqueued
    # the handle still takes a valid problem
    _same_result(_run(dev, _cuda(pb)), _run(host, pb))
    dev.close(); host.close()


def test_numpy_and_cuda_tensors_give_the_same_result(svs):
    pb = synth.make_config("C1")
    a, b = svs.BundleAdjuster(), svs.BundleAdjuster()
    _same_result(_run(a, _cuda(pb)), _run(b, pb))
    a.close(); b.close()


def _map_window(svs, P, L, seed):
    pb = synth.make_window(P, L, seed=seed)
    m, win, act = synth_graph.make_map(pb, seed=seed)
    dm = svs.DeviceMap()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    return pb, m, win, act, dm


def test_from_map_runs_on_the_device_path(svs, oracle):
    pb, m, win, act, dm = _map_window(svs, 30, 3000, 6)
    g = oracle.copy_data_to_g2o(m, win, act)
    ba, ref = svs.BundleAdjuster(), svs.BundleAdjuster()
    for _ in range(2):                                           # the second assembly reuses the structure
        E = dm.set_problem(ba, win, act, pb.cam, c_i=pb.c_i, c_j=pb.c_j, c_T=pb.c_T, c_Lambda=pb.c_Lambda)
        ep, es, ea, obs, info = dm.last_edges(E)
        np.testing.assert_array_equal(ep, g["e_point"]); np.testing.assert_array_equal(es, g["e_pose"])
        np.testing.assert_array_equal(ea, g["e_anchor"]); np.testing.assert_array_equal(obs, g["e_obs"])
        np.testing.assert_array_equal(ba.poses(), g["pose_qt"]); np.testing.assert_array_equal(ba.points(), g["psi"])
        it, st = ba.optimize(3)
    pa = dataclasses.replace(pb, E=E, pose_qt=g["pose_qt"], psi=g["psi"], e_point=ep, e_pose=es, e_anchor=ea, e_obs=obs, e_info=info)
    got = (it, st, ba.poses(), ba.points())
    _same_result(got, _run(ref, pa))
    dm.absorb(ba)
    T, xyz = dm.get()
    np.testing.assert_array_equal(T[win], got[2])
    for h in (dm, ba, ref):
        h.close()
