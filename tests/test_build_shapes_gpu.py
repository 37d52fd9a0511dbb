"""The Schur build at the track shapes where its three kernels change their mapping, against the long-double reference
of tests/build_reference.py.

Each case builds its window from an explicit list of tracks, asserts from the restatement of the routing rules
(build_reference.route) that it reaches the boundary it is named for, and then, for the host set-up
(svs_ba_set_problem) and the device set-up (svs_ba_set_problem_device) of the same window, compares with the reference:
  * reduced_system: per 6x6 block |S - S_ref| <= 1e-11 max M over the block, each 6-vector of bs likewise, chi2 to
    1e-12 relative;
  * chi2() (k_chi2) to 1e-12 relative;
  * one optimize(1, lambda_init=lambda, max_trials=1): the trial is accepted exactly when the reference's step lowers
    chi2, and otherwise leaves the state unchanged.  An accepted step is compared with the reference's one-step state
    to 1e-9 of the step when S is well conditioned (cond(S) eps <= 1e-11).  Where it is not (lambda = 1e-4 on a window
    without a fixed pose: cond(S) ~ 1e10, so no float64 solve is closer than ~1e-6), the step x = log(T1 T0^-1) the
    device applied must solve the reference's S x = bs to a normwise backward error of 1e-10, and psi must equal the
    reference's back-substitution of that x to 1e-9 of the psi step.  The launch count of the trial is
    2 + (k_build_wave or constraints) + k_build + k_build_long.

Worst measured over all cases and both set-ups on an H100 80GB HBM3 (700 W power limit): S 4.4e-14 of M per block,
bs 2.6e-14, chi2 2.7e-15, step 1.8e-12, backward error 2.8e-13.  All 44 trials were accepted; 32 took the
backward-error path."""
import dataclasses
import os

import numpy as np
import pytest

import build_reference as br

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

T = br.Track
S_BAR, CHI_BAR, STEP_BAR, BERR_BAR = 1e-11, 1e-12, 1e-9, 1e-10


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cuda(pb):
    kw = {}
    for k, v in pb.__dict__.items():
        kw[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and k not in ("cam", "truth_pose_qt", "truth_psi") else v
    return dataclasses.replace(pb, **kw)


def _rel_step(got, ref, start):
    return np.abs(got - ref).max() / np.abs(ref - start).max()


def _backward_error(ref, x):
    x = np.asarray(x, br.LD)
    return float(np.abs(ref.S @ x - ref.bs).max() / ((np.abs(ref.S) @ np.abs(x)).max() + np.abs(ref.bs).max()))


def _check(svs, oracle, pb, robust=True, delta=1.0, lam=50.0, flags=0, expect_accept=None):
    """Both set-ups of `pb` against the reference; returns (route, worst ratios)."""
    rt = br.route(pb, _sms(), os.environ.get("SVS_BUILD_CHUNK"))
    ref = br.reduced_system(oracle, pb, robust, delta, lam, skip_self=bool(flags & 1))
    x = br.pose_step(ref)
    poses_ref, psi_ref = br.apply_step(oracle, pb, x, br.back_substitute(ref, x))
    moved = pb.copy(); moved.pose_qt, moved.psi = poses_ref, psi_ref
    accept = oracle.chi2(moved, robust, delta) < float(ref.chi2)
    if expect_accept is not None:
        assert accept == expect_accept
    chi_ref = float(ref.chi2)
    well_conditioned = np.linalg.cond(ref.S.astype(np.float64)) * np.finfo(np.float64).eps <= 1e-11
    worst = dict(S=0.0, b=0.0, chi=0.0, step=0.0, berr=0.0)
    for device in (False, True):
        ba = svs.BundleAdjuster(flags=flags)
        try:
            ba.set_problem(_cuda(pb) if device else pb)
            S, bs, chi = ba.reduced_system(robust, delta, lam)
            r = dict(S=br.block_ratio(S, ref, pb.P), b=br.rhs_ratio(bs, ref, pb.P), chi=abs(chi - chi_ref) / chi_ref)
            r["chi"] = max(r["chi"], abs(ba.chi2(robust, delta) - chi_ref) / chi_ref)
            it, st = ba.optimize(1, robust, delta, lambda_init=lam, max_trials=1)
            assert it == 1 and st["launches"] == rt.launches_per_trial(pb.C), (st["launches"], rt.launches_per_trial(pb.C))
            poses, psi = ba.poses(), ba.points()
            if accept and well_conditioned:
                r["step"] = max(_rel_step(poses, poses_ref, pb.pose_qt), _rel_step(psi, psi_ref, pb.psi))
            elif accept:
                xg = br.recovered_step(oracle, pb.pose_qt, poses, pb.fixed)
                r["berr"] = _backward_error(ref, xg)
                r["step"] = _rel_step(psi, pb.psi + br.back_substitute(ref, xg).astype(np.float64), pb.psi)
            else:
                assert (poses == pb.pose_qt).all() and (psi == pb.psi).all()
            for k in worst:
                worst[k] = max(worst[k], r.get(k, 0.0))
        finally:
            ba.close()
    print(f"\n  ratios S {worst['S']:.2e} b {worst['b']:.2e} chi {worst['chi']:.2e} step {worst['step']:.2e} "
          f"berr {worst['berr']:.2e} accept {accept} well_conditioned {well_conditioned}")
    assert worst["S"] <= S_BAR and worst["b"] <= S_BAR, worst
    assert worst["chi"] <= CHI_BAR, worst
    assert worst["step"] <= STEP_BAR and worst["berr"] <= BERR_BAR, worst
    return rt, worst


# ------------------------------------------------------------------------------------------------ k_build_wave

WAVE_SHAPES = [(1, True)] + [(K, s) for K in range(2, 9) for s in (True, False)]


def _shape_track(anchor, K, self_edge, count):
    return T(anchor, tuple(range(anchor + 1, anchor + K)), self_edge, count)


@pytest.mark.parametrize("K,self_edge", WAVE_SHAPES, ids=[f"K{K}-{'self' if s else 'anchorless'}" for K, s in WAVE_SHAPES])
def test_wave_tasks_around_nw_max(svs, oracle, monkeypatch, K, self_edge):
    """Tasks of 1, nw_max - 1, nw_max, nw_max + 1 and `chunk` = 32 landmarks of one slot shape."""
    monkeypatch.setenv("SVS_BUILD_CHUNK", "32")
    k = K if self_edge else K - 1
    nw = br.nw_max(k, K)
    counts = [1, nw - 1, nw, nw + 1, 32]
    pb = br.make_tracks_window(52, [_shape_track(10 * i, K, self_edge, c) for i, c in enumerate(counts)], seed=K, C=4)
    rt, _ = _check(svs, oracle, pb)
    assert not rt.gen and not rt.long and rt.launches_per_trial(pb.C) == 3   # wave only: the chained trial
    assert sorted(rt.task_shape(t) for t in range(len(rt.tasks))) == sorted((k, K, self_edge, c) for c in counts)


@pytest.mark.parametrize("chunk", [None, "1", "5", "32"])
def test_wave_chunk(svs, oracle, monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("SVS_BUILD_CHUNK", raising=False)
    else:
        monkeypatch.setenv("SVS_BUILD_CHUNK", chunk)
    pb = br.make_tracks_window(52, [_shape_track(3 * i, K, s, 11) for i, (K, s) in enumerate(WAVE_SHAPES)], seed=11, C=6)
    rt, _ = _check(svs, oracle, pb)
    c = rt.chunk
    assert c == (int(chunk) if chunk else 4)
    want = sorted([c] * (11 // c) + ([11 % c] if 11 % c else [])) * len(WAVE_SHAPES)
    assert sorted(cnt for _, cnt in rt.tasks) == sorted(want)


def test_track_padding(svs, oracle, monkeypatch):
    monkeypatch.setenv("SVS_BUILD_CHUNK", "32")
    tracks = [
        T(10, (11, 12, 14, 16), True, 3),        # np = 2 = m/2, at the limit: padded
        T(10, (11, 12, 13, 14, 15, 16), True, 2),  # ... into the slot list of these complete tracks, one run of 5
        T(20, (21, 23, 25, 27), True, 2),        # np = 3, one past the limit: left as it is
        T(32, (30, 31, 33, 35), True, 2),        # anchor inside lo..hi, self edge
        T(42, (40, 41, 43, 45), False, 2),       # anchor inside lo..hi, anchorless
        T(50, (51, 52, 53, 55, 57), True, 2),    # completed track of exactly 8 slots
        T(60, (61, 62, 63, 64, 66, 68), True, 2),  # would need 9 slots: left at 7
    ]
    pb = br.make_tracks_window(70, tracks, seed=12, C=4)
    rt, _ = _check(svs, oracle, pb)
    by_anchor = {}
    for li, l in enumerate(rt.order):
        a = int(pb.e_anchor[pb.e_point == l][0])
        by_anchor.setdefault(a, set()).add((rt.npad[li], rt.K[li]))
    assert by_anchor[10] == {(2, 7), (0, 7)}
    assert by_anchor[20] == {(0, 5)} and by_anchor[32] == {(1, 6)} and by_anchor[42] == {(1, 6)}
    assert by_anchor[50] == {(2, 8)} and by_anchor[60] == {(0, 7)}
    assert sorted(cnt for _, cnt in rt.tasks) == [2] * 5 + [5]
    assert not rt.gen and not rt.long


# ------------------------------------------------------------------------------------------------ grid shape

@pytest.mark.parametrize("mode", ["one_task_per_warp", "persistent"])
@pytest.mark.parametrize("C", [1, 128, 129, 257])
def test_wave_grid_and_constraint_ctas(svs, oracle, monkeypatch, mode, C):
    """Constraint CTAs (128 constraints each, the last one partial for C = 1, 129, 257) trail a grid of one task per
    warp and lead a persistent grid.  The task counts stay clear of the persistent threshold (resident CTAs x 4 warps):
    a quarter of it, and more than twice it."""
    monkeypatch.setenv("SVS_BUILD_CHUNK", "1")
    thr = br.persistent_threshold_tasks(_sms())
    n = thr // 4 if mode == "one_task_per_warp" else 2 * thr + 64
    P = 40
    tracks = [T(a, (a + 1,) if a % 2 else (a + 1, a + 2), a % 3 != 0, 0) for a in range(P - 2)]
    tracks = [dataclasses.replace(t, count=n // len(tracks) + (1 if i < n % len(tracks) else 0)) for i, t in enumerate(tracks)]
    pb = br.make_tracks_window(P, tracks, seed=13, C=C)
    rt, _ = _check(svs, oracle, pb)
    assert len(rt.tasks) == n and pb.L <= 4096
    assert (len(rt.tasks) + 3) // 4 > 2 * _sms() if mode == "persistent" else (len(rt.tasks) + 3) // 4 <= 2 * _sms()


# ------------------------------------------------------------------------------------------------ k_build, k_build_long

def test_generic_kernel_shapes(svs, oracle):
    """k_build: K = 9 with and without a self edge, K = 32 with a self edge (k = 32, every lane) and without (k = 31),
    other K in the same launch (shared memory sized for the largest), unobserved landmarks interleaved."""
    tracks = [T(0, tuple(range(1, 9)), True, 2), T(1, tuple(range(2, 10)), False, 2),
              T(2, tuple(range(3, 34)), True, 2), T(3, tuple(range(4, 35)), False, 2),
              T(4, tuple(range(5, 17)), True, 1), T(5, tuple(range(6, 26)), False, 1), T(6, (7, 8), True, 3)]
    pb = br.make_tracks_window(40, tracks, seed=14, C=8, unobserved=5)
    rt, _ = _check(svs, oracle, pb)
    shapes = {(rt.k[li], rt.K[li], bool(rt.self_[li])) for li in rt.gen}
    assert {(9, 9, True), (8, 9, False), (32, 32, True), (31, 32, False), (0, 0, False)} <= shapes
    assert max(rt.K[li] for li in rt.gen) == 32 and not rt.long and len(rt.tasks) == 1


def test_long_kernel_shapes(svs, oracle):
    """k_build_long: K = 33 without a self edge (k = 32: exactly one pass-A round) and with one (k = 33); k = 64, 65
    (anchorless) and 97."""
    tracks = [T(0, tuple(range(1, 33)), False, 2), T(1, tuple(range(2, 34)), True, 2),
              T(2, tuple(range(3, 66)), True, 1), T(3, tuple(range(4, 69)), False, 1), T(0, tuple(range(1, 97)), True, 1)]
    pb = br.make_tracks_window(100, tracks, seed=15, C=6)
    rt, _ = _check(svs, oracle, pb)
    shapes = {(rt.k[li], rt.K[li], bool(rt.self_[li])) for li in rt.long}
    assert shapes == {(32, 33, False), (33, 33, True), (64, 64, True), (65, 66, False), (97, 97, True)}
    assert not rt.gen and not rt.tasks


def _three_kernels(fixed=()):
    """Frame 2 anchors a track of every kernel (with a self edge) and frame 5 observes them; frame 8 anchors an
    anchorless track of every kernel."""
    tracks = [T(2, (3, 4, 5), True, 5), T(2, tuple(range(3, 15)), True, 2), T(2, tuple(range(3, 41)), True, 1),
              T(8, (9, 10), False, 4), T(8, tuple(range(9, 21)), False, 2), T(8, tuple(range(9, 46)), False, 1),
              T(0, (), True, 3), T(12, (13, 14, 16), True, 4)]
    return br.make_tracks_window(50, tracks, seed=16, C=10, unobserved=3, fixed=fixed)


EVERY = [(False, 1.0, 1e-4), (False, 1.0, 1e5), (True, 0.5, 1e-4), (True, 0.5, 1e5), (True, 1.0, 1e-4), (True, 1.0, 1e5),
         (True, 3.0, 1e-4), (True, 3.0, 1e5)]


@pytest.mark.parametrize("robust,delta,lam", EVERY, ids=[f"{'huber' + str(d) if r else 'plain'}-lam{l:g}" for r, d, l in EVERY])
def test_every_kernel(svs, oracle, robust, delta, lam):
    pb = _three_kernels()
    rt, _ = _check(svs, oracle, pb, robust, delta, lam)
    assert rt.tasks and rt.gen and rt.long and rt.launches_per_trial(pb.C) == 5


@pytest.mark.parametrize("variant", ["skip_self", "fixed_anchor", "fixed_observer"])
def test_every_kernel_flags_and_fixed_poses(svs, oracle, variant):
    pb = _three_kernels(fixed={"fixed_anchor": (2,), "fixed_observer": (5,)}.get(variant, ()))
    flags = svs.SVS_BA_SKIP_SELF_ANCHOR_HESSIAN if variant == "skip_self" else 0
    rt, _ = _check(svs, oracle, pb, flags=flags)
    kinds = set()
    for li in range(len(rt.order)):
        l = rt.order[li]
        m = pb.e_point == l
        if m.any() and (int(pb.e_anchor[m][0]) == 2 if variant != "fixed_observer" else 5 in pb.e_pose[m]):
            kinds.add("long" if li in rt.long else "gen" if li in rt.gen else "wave")
    assert kinds == {"wave", "gen", "long"}


# ------------------------------------------------------------------------------------------------ k_update

@pytest.mark.parametrize("rem", [0, 1, 31])
def test_update_track_lengths_and_landmark_counts(svs, oracle, rem):
    """k_update gives each landmark 8 lanes, four landmarks per warp and 32 per CTA: slots and edges across 8/9,
    16/17 and 32/33, and L mod 32 in {0, 1, 31}."""
    tracks = [T(0, tuple(range(1, 8)), True, 1), T(0, tuple(range(1, 9)), True, 1), T(1, tuple(range(2, 10)), False, 1),
              T(2, tuple(range(3, 18)), True, 1), T(2, tuple(range(3, 19)), True, 1), T(3, tuple(range(4, 20)), False, 1),
              T(4, tuple(range(5, 36)), True, 1), T(4, tuple(range(5, 37)), True, 1), T(5, tuple(range(6, 38)), False, 1)]
    base = sum(t.count for t in tracks)
    extra = (rem - base) % 32 + 64
    tracks.append(T(6, (7, 8), True, extra))
    pb = br.make_tracks_window(40, tracks, seed=17 + rem, C=4)
    assert pb.L % 32 == rem
    rt, w = _check(svs, oracle, pb, expect_accept=True)
    Ks = {(rt.k[li], rt.K[li]) for li in range(len(rt.order))}
    assert {(8, 8), (9, 9), (8, 9), (16, 16), (17, 17), (16, 17), (32, 32), (33, 33), (32, 33)} <= Ks
