"""The long-double reference of the covariance and gradient kernels (tests/cov_grad_reference.py) against the float64
dense references, and the routes of the windows test_cov_grad_shapes_gpu.py runs.  Runs without a GPU.

Measured (x86-64, 80-bit long double), as a ratio per block to the block's magnitude companion: against the dense
float64 inverse of oracle.full_system, pose blocks 6.6e-14, pose pairs 1.0e-14, landmark blocks 2.0e-16; against
ba_grad_reference.observation_grad and ba_window_grad_reference.window_grad, every gradient output at most 1.6e-15
(kappa(S) ~ 6e5-4e6 here, so the float64 references carry errors of ~kappa eps of their own)."""
import numpy as np
import pytest

import ba_grad_reference as gref
import ba_window_grad_reference as wref
import build_reference as br
import cov_grad_reference as cr

T = br.Track
AGREE = 1e-11


def _small(fixed=(), C=6):
    """Every kind of track the kernels tell apart, on a window small enough for a dense float64 inverse."""
    tracks = [T(0, (), True, 2), T(1, (2, 3), False, 2), T(2, (3, 4, 5), True, 2), T(6, (4, 5, 7, 9), True, 1),
              T(1, tuple(range(2, 12)), True, 1), T(0, tuple(range(1, 14)), False, 1)] + cr._chain(14)
    return cr._with_zero_weight_edge(br.make_tracks_window(14, tracks, seed=7, fixed=fixed, C=C, unobserved=2))


def _dense_cov(oracle, pb, lam, pairs):
    H, _, _ = oracle.full_system(pb, True, 1.0)
    H = H + lam * np.eye(len(H))
    has = np.zeros(pb.L, bool)
    has[pb.e_point] = True
    keep = np.concatenate([np.repeat(pb.fixed == 0, 6), np.repeat(has, 3)])
    Z = np.zeros_like(H)
    Z[np.ix_(keep, keep)] = np.linalg.inv(H[np.ix_(keep, keep)])
    o = 6 * pb.P
    pose = np.array([Z[6 * p:6 * p + 6, 6 * p:6 * p + 6] for p in range(pb.P)])
    pair = np.array([Z[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs])
    point = np.array([Z[o + 3 * l:o + 3 * l + 3, o + 3 * l:o + 3 * l + 3] for l in range(pb.L)])
    return pose, pair, point


@pytest.mark.parametrize("lam,fixed", [(0.0, (3,)), (1.0, ())])
def test_covariance_equals_the_dense_inverse(oracle, lam, fixed):
    pb = _small(fixed)
    pairs = [(1, 2), (12, 0), (5, 5)] + ([(3, 7)] if fixed else [])
    ref = br.reduced_system(oracle, pb, True, 1.0, lam)
    cov = cr.covariance(ref, pb, pairs)
    pose, pair, point = _dense_cov(oracle, pb, lam, pairs)
    r = dict(pose=cr.block_ratio(pose, cov.pose, cov.pose_m, (1, 2)),
             pair=cr.block_ratio(pair, cov.pair, cov.pair_m, (1, 2)),
             point=cr.block_ratio(point, cov.point, cov.point_m, (1, 2)))
    print(f"\n  kappa {cov.kappa:.2e} ratios {r}")
    assert max(r.values()) <= AGREE, r
    assert not cov.point[~ref.has_edges].any() and not cov.pose[list(fixed)].any()


@pytest.mark.parametrize("lam,fixed", [(0.0, (3,)), (1.0, ())])
def test_adjoint_equals_the_dense_references(oracle, lam, fixed):
    pb = _small(fixed)
    rng = np.random.default_rng(3)
    gp, gl = rng.normal(size=(pb.P, 6)), rng.normal(size=(pb.L, 3))
    g = cr.adjoint(oracle, pb, gp, gl, True, 1.0, lam)
    dobs, dinfo = gref.observation_grad(oracle, pb, gp, gl, True, 1.0, lam)
    want = wref.window_grad(oracle, pb, gp, gl, True, 1.0, lam)
    r = dict(obs=cr.block_ratio(dobs, g.obs, g.obs_m, 1), info=cr.block_ratio(dinfo, g.info, g.info_m, 1),
             cT=cr.block_ratio(want["cT"], g.cT, g.cT_m, 1), cLambda=cr.block_ratio(want["cLambda"], g.cLambda, g.cLambda_m, 1),
             cam=cr.block_ratio(want["cam"][None], g.cam[None], g.cam_m[None], 1))
    r["window_obs"] = cr.block_ratio(want["obs"], g.obs, g.obs_m, 1)
    print(f"\n  kappa {g.kappa:.2e} ratios {r}")
    assert max(r.values()) <= AGREE, r
    zero = ~np.asarray(pb.e_info).any(1)
    assert zero.sum() == 1 and not g.obs[zero].any() and not g.info[zero].any()


def test_inverse_ld_refines_to_long_double():
    rng = np.random.default_rng(0)
    A = rng.normal(size=(60, 60))
    S = (A @ A.T + 1e-3 * np.eye(60)).astype(cr.LD)
    Z, kappa = cr.inverse_ld(S)
    Z64 = np.linalg.inv(S.astype(np.float64))
    res = float(np.abs(np.eye(60, dtype=cr.LD) - S @ Z).max())
    res64 = float(np.abs(np.eye(60) - S.astype(np.float64) @ Z64).max())
    assert res < res64 / 100 and kappa > 1e3


# ------------------------------------------------------------------------------------------------ routes

@pytest.mark.parametrize("rem", [0, 1, 31])
def test_lanes8_windows_reach_their_boundaries(rem):
    pb = cr.lanes8_window(rem)
    cr.check_lanes8(pb, br.route(pb, cr.H100_SMS), rem)


@pytest.mark.parametrize("rem", [0, 1, 7])
def test_warp_windows_reach_their_boundaries(rem):
    pb = cr.warp_window(rem)
    cr.check_warps(pb, br.route(pb, cr.H100_SMS), rem)


@pytest.mark.parametrize("P,L,C,boundary", cr.GRID, ids=[f"P{p}-L{l}-C{c}-{b}" for p, l, c, b in cr.GRID])
def test_grid_windows_reach_their_boundaries(P, L, C, boundary):
    cr.check_grid(cr.grid_window(P, L, C), P, L, C, boundary)


def test_grid_list_covers_every_constraint_boundary():
    assert {c for _, _, c, _ in cr.GRID} == {0, 1, 255, 256, 257}
    assert {b for _, _, _, b in cr.GRID} == {"rhs-", "rhs+", "cam"}
    assert any(l < 256 for _, l, _, _ in cr.GRID)
