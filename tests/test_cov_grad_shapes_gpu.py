"""svs_ba_covariance (k_ba_point_cov, k_chol6_selinv, k_chol6_inv_cols) and svs_ba_window_grad /
svs_ba_observation_grad (k_grad_rhs, k_grad_edges, k_grad_cam, k_grad_constraints) at the track shapes and grid sizes
where their lane mapping changes, against the long-double reference of tests/cov_grad_reference.py.

Each window comes from an explicit list of tracks and asserts through build_reference.route that it reaches the
boundary it is named for (the windows and their checks live in cov_grad_reference.py, which
test_cov_grad_shapes_cpu.py also runs).  Every case runs the host set-up (svs_ba_set_problem) and the device set-up
(torch CUDA tensors, svs_ba_set_problem_device) of one window at one state, not optimised:
  * covariance in a handle without and with SVS_BA_SKIP_SELF_ANCHOR_HESSIAN against reduced_system(skip_self = the
    flag): pose blocks, pose pairs inside and outside the factor's pattern, landmark blocks;
  * window_grad (every output) and observation_grad in handles without and with the flag, against the one skip-self
    reference (the gradient's H never holds the self-anchor term).  In the device set-up the inputs are CUDA tensors
    and every output is pre-filled with NaN inside a NaN guard row on each side: every caller edge and constraint must
    be written, and nothing outside them.
Bars are per block (landmark, pose block, pair, edge, constraint, the camera) against the reference's magnitude
companion.  Landmark blocks: 1e-10; every gradient output: 1e-11 (the gradient's companions are loose, because J v
cancels its pose and landmark terms, so a looser bar would let one dropped edge of 32 through).  Pose blocks and pairs, which carry the factor's own
rounding: max(1e-10, 10 kappa(S) eps) with kappa(S) from the long-double inverse; every window here has kappa(S) ~ 3e6
to 1e8 (the pose Hessians reach ~1e7; lambda = 0 with fixed poses, lambda = 1 without), so that bar is 7e-9 to 3e-7.

Sensitivity: for each shape group (device slot count K and self flag, K >= 2) the reference is perturbed as a lane
group one round short would be (covariance: the pairs of the last round of LANES dropped, or the last pair when they
fit one round; gradient: the slots, and separately the edges, of the last round, or the last one) and with the pair
(K-1, K-1) counted twice; each perturbed reference must miss the bar by 100x against the device output.  (K = 1 is left
out: its only slot is the anchor's self slot, whose Hpl block is zero to rounding.)

Worst measured over all cases, both set-ups and both flags on an H100 80GB HBM3 (700 W power limit): landmark blocks
4.5e-14 of their companion, pose blocks and pairs 9.7e-11 (5.2e-3 of their bar), dL/dz 5.8e-15, dL/domega 5.2e-14,
dL/d delta_c 4.4e-16, dL/dLambda_c 1.1e-16, dL/dcam 8.7e-19.  The perturbed references missed their bar by at least
300x.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import build_reference as br
import cov_grad_reference as cr

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SENSE = 100.0


def _cuda(pb):
    kw = {}
    for k, v in pb.__dict__.items():
        kw[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and k not in ("cam", "truth_pose_qt", "truth_psi") else v
    return dataclasses.replace(pb, **kw)


def _with_fixed(pb, fixed):
    pb = pb.copy()
    pb.fixed = np.zeros(pb.P, np.uint8)
    pb.fixed[list(fixed)] = 1
    return pb


def _groups(pb, rt):
    """{(K, self): user labels} over the observed landmarks with at least two slots, and per label its lane count."""
    groups, lanes = {}, np.zeros(pb.L, np.int64)
    for li, l in enumerate(rt.order):
        lanes[l] = 8 if rt.K[li] <= 8 else 32
        if rt.k[li] and rt.K[li] >= 2:
            groups.setdefault((rt.K[li], bool(rt.self_[li])), []).append(l)
    return groups, lanes


def _last_round(n, lanes):
    """keep[i] of n items of a lane group one round short: the items of the last round dropped (the last item when
    they all fit one round)."""
    keep = np.ones(n, bool)
    if n > lanes:
        keep[lanes * ((n - 1) // lanes):] = False
    elif n:
        keep[n - 1] = False
    return keep


def _pair_short(lanes):
    def f(l, K):
        iu = np.triu_indices(K)                      # a-major pairs a <= b
        m = np.zeros((K, K))
        m[iu] = _last_round(len(iu[0]), lanes[l])
        return m
    return f


def _pair_double(l, K):
    m = np.triu(np.ones((K, K)))
    m[K - 1, K - 1] = 2
    return m


def _sensitivity(groups, got, pert, comp, b, what, index=None):
    """Per shape group, the perturbed reference must miss the bar by SENSE x against the device output."""
    worst = np.inf
    for key, labels in groups.items():
        idx = np.asarray(labels) if index is None else np.concatenate([index[l] for l in labels])
        r = cr.block_ratio(got[idx], pert[idx], comp[idx], tuple(range(1, got.ndim)))
        assert r >= SENSE * b, f"{what}: shape {key} misses the bar by only {r / b:.1f}x"
        worst = min(worst, r / b)
    return worst


# ------------------------------------------------------------------------------------------------ covariance

def _check_covariance(svs, oracle, pb, rt, lam, pairs, want_outside):
    groups, lanes = _groups(pb, rt)
    worst, margin = {}, np.inf
    for flags in (0, svs.SVS_BA_SKIP_SELF_ANCHOR_HESSIAN):
        ref = br.reduced_system(oracle, pb, True, 1.0, lam, skip_self=bool(flags))
        Z, kappa = cr.inverse_ld(ref.S)
        cov = cr.covariance(ref, pb, pairs, Z, kappa)
        bz, b = cr.pose_bar(kappa), cr.BLOCK_BAR
        for device in (False, True):
            ba = svs.BundleAdjuster(flags=flags)
            try:
                ba.set_problem(_cuda(pb) if device else pb)
                pose, pair, point, rc, st = ba.covariance(True, 1.0, lam, pairs)
            finally:
                ba.close()
            assert rc == 0
            r = dict(pose=cr.block_ratio(pose, cov.pose, cov.pose_m, (1, 2)),
                     pair=cr.block_ratio(pair, cov.pair, cov.pair_m, (1, 2)),
                     point=cr.block_ratio(point, cov.point, cov.point_m, (1, 2)))
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
            assert r["pose"] <= bz and r["pair"] <= bz and r["point"] <= b, (flags, device, r, bz, b)
            assert np.array_equal(point, point.transpose(0, 2, 1))
            assert st["n_pairs_in_pattern"] > 0 and (st["n_cols_solved"] > 0 or not want_outside), st
        slots = cr.slot_lists(ref, pb)
        for mult, what in ((_pair_short(lanes), "one round short"), (_pair_double, "diagonal pair twice")):
            pert, _ = cr.landmark_blocks(ref, pb, Z, slots, mult)
            margin = min(margin, _sensitivity(groups, point, pert, cov.point_m, b, f"covariance {what}"))
    print(f"\n  covariance kappa {kappa:.2e} pose bar {bz:.1e}: worst {worst}; perturbations miss by >= {margin:.1e} x")


# ------------------------------------------------------------------------------------------------ gradient

def _guarded(rows, width):
    """A NaN-filled CUDA buffer of rows + 2 rows and its inner view (the guard rows stay outside the call)."""
    buf = torch.full((rows + 2, width), float("nan"), dtype=torch.float64, device="cuda")
    return buf, buf[1:rows + 1]


def _device_grads(svs, ba, pb, gp, gl, lam):
    """window_grad and observation_grad through the C ABI with NaN-filled CUDA outputs in NaN guard rows."""
    lib = svs.lib()
    tgp, tgl = torch.from_numpy(gp).cuda(), torch.from_numpy(gl).cuda()
    bufs = {k: _guarded(n, w) for k, (n, w) in
            dict(obs=(pb.E, 3), info=(pb.E, 3), cT=(pb.C, 6), cLambda=(pb.C, 36), cam=(1, 4)).items()}
    out = svs.SvsBaGradOut()
    for k, (_, v) in bufs.items():
        setattr(out, svs.BundleAdjuster._GRAD_OUT[k][0], v.data_ptr() if v.numel() else None)
    st = svs.SvsBaGradStats()
    torch.cuda.synchronize()
    rc = lib.svs_ba_window_grad(ba._h, 1, 1.0, float(lam), tgp.data_ptr(), tgl.data_ptr(), C.byref(out), 1, C.byref(st))
    assert rc == 0
    ob, obs = _guarded(pb.E, 3)
    ib, info = _guarded(pb.E, 3)
    rc = lib.svs_ba_observation_grad(ba._h, 1, 1.0, float(lam), tgp.data_ptr(), tgl.data_ptr(), obs.data_ptr(),
                                     info.data_ptr(), 1, C.byref(st))
    assert rc == 0
    torch.cuda.synchronize()
    for k, (buf, v) in list(bufs.items()) + [("obs2", (ob, obs)), ("info2", (ib, info))]:
        b = buf.cpu().numpy()
        assert np.isnan(b[0]).all() and np.isnan(b[-1]).all(), f"{k}: written outside its rows"
        assert not np.isnan(b[1:-1]).any(), f"{k}: a row left unwritten"
    res = {k: v.cpu().numpy() for k, (_, v) in bufs.items()}
    res["cam"] = res["cam"][0]
    return res, obs.cpu().numpy(), info.cpu().numpy()


def _check_gradient(svs, oracle, pb, rt, lam, seed=0, sensitivity=True):
    groups, lanes = _groups(pb, rt)
    rng = np.random.default_rng(seed)
    gp, gl = rng.normal(size=(pb.P, 6)), rng.normal(size=(pb.L, 3))
    ref = br.reduced_system(oracle, pb, True, 1.0, lam, skip_self=True)
    Z, kappa = cr.inverse_ld(ref.S)
    g = cr.adjoint(oracle, pb, gp, gl, True, 1.0, lam, ref, Z, kappa)
    b = cr.GRAD_BAR
    worst = {}
    got_obs = None
    for flags in (0, svs.SVS_BA_SKIP_SELF_ANCHOR_HESSIAN):
        for device in (False, True):
            ba = svs.BundleAdjuster(flags=flags)
            try:
                ba.set_problem(_cuda(pb) if device else pb)
                if device:
                    res, obs, info = _device_grads(svs, ba, pb, gp, gl, lam)
                else:
                    res, rc, st = ba.window_grad(gp, gl, True, 1.0, lam)
                    assert rc == 0 and st["E"] == pb.E
                    obs, info, rc, _ = ba.observation_grad(gp, gl, True, 1.0, lam)
                    assert rc == 0
            finally:
                ba.close()
            r = dict(obs=cr.block_ratio(res["obs"], g.obs, g.obs_m, 1), info=cr.block_ratio(res["info"], g.info, g.info_m, 1),
                     obs_grad=max(cr.block_ratio(obs, g.obs, g.obs_m, 1), cr.block_ratio(info, g.info, g.info_m, 1)),
                     cT=cr.block_ratio(res["cT"], g.cT, g.cT_m, 1), cLambda=cr.block_ratio(res["cLambda"], g.cLambda, g.cLambda_m, 1),
                     cam=cr.block_ratio(res["cam"][None], g.cam[None], g.cam_m[None], 1))
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
            assert max(r.values()) <= b, (flags, device, r, b)
            got_obs = res["obs"]
    margin = np.inf
    if sensitivity:
        ep = np.asarray(pb.e_point)
        edges_of = {l: np.nonzero(ep == l)[0] for l in range(pb.L)}
        for kw, what in ((dict(slot_keep=lambda l, K: _last_round(K, lanes[l])), "slots one round short"),
                         (dict(edge_keep=lambda l, k: _last_round(k, lanes[l])), "edges one round short")):
            pert = cr.adjoint(oracle, pb, gp, gl, True, 1.0, lam, ref, Z, kappa, **kw)
            margin = min(margin, _sensitivity(groups, got_obs, pert.obs, g.obs_m, b, f"gradient {what}", edges_of))
    print(f"\n  gradient kappa {kappa:.2e}: worst {worst}; perturbations miss by >= {margin:.1e} x")


# ------------------------------------------------------------------------------------------------ cases

CFG = [("lam0-fixed", 0.0, True), ("lam1-free", 1.0, False)]


@pytest.mark.parametrize("cfg", CFG, ids=[c[0] for c in CFG])
@pytest.mark.parametrize("rem", [0, 1, 31])
def test_eight_lane_tracks(svs, oracle, rem, cfg):
    """K = 1 .. 8 with and without a self edge, padded tracks, a zero-weight edge, L = rem mod 32; pose pairs inside
    the band of short tracks and far outside it."""
    _, lam, fix = cfg
    pb = cr.lanes8_window(rem)
    rt = br.route(pb, cr.H100_SMS)
    cr.check_lanes8(pb, rt, rem)
    pb = _with_fixed(pb, (5,) if fix else ())
    pairs = [(3, 4), (4, 3), (12, 12), (0, 29), (29, 1), (5, 20)]
    _check_covariance(svs, oracle, pb, rt, lam, pairs, want_outside=True)
    _check_gradient(svs, oracle, pb, rt, lam, seed=rem)


@pytest.mark.parametrize("cfg", CFG, ids=[c[0] for c in CFG])
@pytest.mark.parametrize("rem", [0, 1, 7])
def test_warp_tracks(svs, oracle, rem, cfg):
    """gen_lm (K = 9 .. 32, landmarks without edges) and long_lm (K = 33 .. 65, 97 for rem = 0), ngen = nlong = rem
    mod 8; at lambda = 0 the anchor of one long track and an observer of another are fixed."""
    _, lam, fix = cfg
    pb = cr.warp_window(rem)
    rt = br.route(pb, cr.H100_SMS)
    cr.check_warps(pb, rt, rem)
    pb = _with_fixed(pb, cr.WARP_FIXED if fix else ())
    pairs = [(4, 60), (60, 4), (7, 30), (6, 40), (0, pb.P - 1)]
    _check_covariance(svs, oracle, pb, rt, lam, pairs, want_outside=False)
    _check_gradient(svs, oracle, pb, rt, lam, seed=10 + rem)


@pytest.mark.parametrize("P,L,C,boundary", cr.GRID, ids=[f"P{p}-L{l}-C{c}-{b}" for p, l, c, b in cr.GRID])
def test_gradient_grids(svs, oracle, P, L, C, boundary):
    """k_grad_rhs at L + 6P next to a multiple of 256, k_grad_cam at L < 256 and L = 256 m + 1, k_grad_constraints at
    C = 0, 1, 255, 256, 257 with frames 0 and 1 fixed (constraints joining both, one or neither), at lambda = 1."""
    pb = cr.grid_window(P, L, C)
    rt = br.route(pb, cr.H100_SMS)
    cr.check_grid(pb, P, L, C, boundary)
    _check_gradient(svs, oracle, _with_fixed(pb, (0, 1)), rt, 1.0, seed=L)
