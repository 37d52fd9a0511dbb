"""svs_ba_observation_grad (gradients of the optimised window with respect to its observations and weights) against
the dense reference of ba_grad_reference.py at the device's accepted state, each output to <= 1e-8 of its largest
entry.  The upstream gradient is seeded random and includes fixed poses, whose entries must not matter.

The build kernels sum the reduced system with FP64 atomics, so two builds of one state agree only to the last bits;
checks of repeated calls and of an optimize after a call use a tolerance instead of bit equality for that reason.
"""
import dataclasses
import os

import numpy as np
import pytest

import ba_grad_reference as ref
from scavislam_b200 import synth, synth_graph

pytestmark = pytest.mark.gpu

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


def _upstream(pb, seed=0):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(pb.P, 6)), rng.normal(size=(pb.L, 3))


def _close(got, want, what):
    scale = max(np.abs(want).max(), 1e-300)
    err = np.abs(got - want).max() / scale
    assert err <= TOL, f"{what}: {err:.3e} of the largest entry"


def _check(ba, oracle, pb, robust=True, lam=0.0, iters=0, seed=0):
    ba.set_problem(pb)
    if iters:
        ba.optimize(iters, robust)
    gp, gl = _upstream(pb, seed)
    dobs, dinfo, rc, st = ba.observation_grad(gp, gl, robust, 1.0, lam)
    assert rc == 0
    state = dataclasses.replace(pb, pose_qt=ba.poses(), psi=ba.points())
    r_obs, r_info = ref.observation_grad(oracle, state, gp, gl, robust, 1.0, lam)
    _close(dobs, r_obs, "dL/dobs")
    _close(dinfo, r_info, "dL/dinfo")
    # the fixed poses' entries of g do not matter
    gp2 = gp.copy()
    gp2[np.asarray(pb.fixed) != 0] = 1e3
    d2, i2, _, _ = ba.observation_grad(gp2, gl, robust, 1.0, lam)
    _close(d2, r_obs, "dL/dobs with other fixed-pose gradients")
    assert st["P"] == pb.P and st["L"] == pb.L and st["E"] == pb.E
    return dobs, dinfo, st


@pytest.mark.parametrize("robust", [True, False])
def test_c1_optimised_with_a_fixed_pose(ba, oracle, robust):
    _check(ba, oracle, _fixed(synth.make_config("C1"), 0), robust=robust, iters=4)


def test_c1_without_fixed_pose_damped(ba, oracle):
    """No fixed pose: only lambda removes the gauge freedom, and J v cancels v's large gauge component, so the output's
    rounding error grows like 1/lambda (3.6e-8 of the largest entry at lambda = 1e-3 on an H100).  lambda = 1."""
    _check(ba, oracle, synth.make_config("C1"), lam=1.0, iters=2)


def test_tracks_of_9_to_32_slots(ba, oracle):
    _check(ba, oracle, _fixed(synth.make_window(30, 1500, seed=31, T=14), 0), iters=2)


def test_tracks_longer_than_32_slots(ba, oracle):
    _check(ba, oracle, _fixed(synth.make_window(70, 900, seed=36, T=50), 0), iters=1)
    assert ba.lm_stats()["max_track"] > 33


def test_visibility_dropouts_write_every_caller_edge(ba, oracle):
    pb = _fixed(synth.with_dropouts(synth.make_window(40, 1200, seed=41), 0.2, seed=3), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    gp, gl = _upstream(pb)
    import torch
    nan = torch.full((pb.E, 3), float("nan"), dtype=torch.float64, device="cuda")
    outs = [nan.clone(), nan.clone()]
    from scavislam_b200 import capi
    import ctypes as C
    st = capi.SvsBaGradStats()
    tg = [torch.as_tensor(a, device="cuda") for a in (gp, gl)]
    rc = capi.lib().svs_ba_observation_grad(ba._h, 1, 1.0, 0.0, tg[0].data_ptr(), tg[1].data_ptr(), outs[0].data_ptr(),
                                            outs[1].data_ptr(), 1, C.byref(st))
    assert rc == 0 and st.E == pb.E
    for o in outs:   # every caller edge written, nothing beyond (padding edges produce no output)
        assert torch.isfinite(o).all()
    state = dataclasses.replace(pb, pose_qt=ba.poses(), psi=ba.points())
    r_obs, r_info = ref.observation_grad(oracle, state, gp, gl, True, 1.0, 0.0)
    _close(outs[0].cpu().numpy(), r_obs, "dL/dobs")
    _close(outs[1].cpu().numpy(), r_info, "dL/dinfo")


def test_loop_closures_two_ended_with_separator(ba, oracle):
    pb = _fixed(synth.with_loop_closures(synth.make_window(60, 1000, seed=32), 3, seed=1), 0)
    _, _, st = _check(ba, oracle, pb, iters=2)
    assert st["nbranch"] == 2


def test_dense_pattern_on_the_general_solver(ba, oracle):
    P = 150
    pb = synth.make_window(P, 700, seed=33)
    ci, cj, cT, cL = list(pb.c_i), list(pb.c_j), list(pb.c_T), list(pb.c_Lambda)
    lam = np.diag([4e4] * 3 + [1e5] * 3).reshape(36)
    for i in range(P):
        for j in range(i + 1, P):
            ci.append(i); cj.append(j); cT.append(pb.c_T[0]); cL.append(lam)
    pb.c_i, pb.c_j = np.asarray(ci, np.int32), np.asarray(cj, np.int32)
    pb.c_T, pb.c_Lambda = np.asarray(cT).reshape(-1, 7), np.asarray(cL).reshape(-1, 36)
    pb.C = len(ci)
    _, _, st = _check(ba, oracle, _fixed(pb, 0))
    assert st["general"] == 1


def test_single_chain_solver(svs, oracle):
    os.environ["SVS_SOLVE_CHAIN"] = "1"
    try:
        b = svs.BundleAdjuster()
        _, _, st = _check(b, oracle, _fixed(synth.make_window(60, 1000, seed=34), 0), iters=1)
        assert st["nbranch"] == 1 and st["general"] == 0
        b.close()
    finally:
        del os.environ["SVS_SOLVE_CHAIN"]


def test_landmarks_without_edges_and_a_zero_weight_edge(ba, oracle):
    pb = _fixed(synth.make_config("C1"), 0)
    keep = np.isin(pb.e_point, np.arange(0, pb.L, 7), invert=True)   # every 7th landmark loses its edges
    pb = dataclasses.replace(pb, E=int(keep.sum()), e_point=pb.e_point[keep], e_pose=pb.e_pose[keep],
                             e_anchor=pb.e_anchor[keep], e_obs=pb.e_obs[keep], e_info=pb.e_info[keep].copy())
    pb.e_info[5] = 0.0
    dobs, dinfo, _ = _check(ba, oracle, pb, iters=2)
    assert not dobs[5].any() and not dinfo[5].any()


def test_self_anchor_term_never_enters(svs, oracle):
    """One window and one state, not optimised, in handles with and without SVS_BA_SKIP_SELF_ANCHOR_HESSIAN."""
    pb = _fixed(synth.make_config("C1"), 0)
    gp, gl = _upstream(pb, 4)
    a, b = svs.BundleAdjuster(), svs.BundleAdjuster(flags=svs.SVS_BA_SKIP_SELF_ANCHOR_HESSIAN)
    ra, rb = [], []
    for h, out in ((a, ra), (b, rb)):
        h.set_problem(pb)
        out.extend(h.observation_grad(gp, gl)[:2])
    for x, y in zip(ra, rb):
        assert np.abs(x - y).max() <= 1e-10 * np.abs(y).max()
    r_obs, _ = ref.observation_grad(oracle, pb, gp, gl)
    _close(ra[0], r_obs, "dL/dobs")
    a.close(); b.close()


def test_host_and_cuda_tensor_arrays_agree(ba):
    import torch
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    gp, gl = _upstream(pb, 6)
    h_obs, h_info, rc, _ = ba.observation_grad(gp, gl)
    t_obs, t_info, rc2, _ = ba.observation_grad(torch.as_tensor(gp, device="cuda"), torch.as_tensor(gl, device="cuda"))
    assert rc == rc2 == 0 and t_obs.is_cuda and t_info.is_cuda
    for x, y in ((h_obs, t_obs), (h_info, t_info)):
        assert np.abs(x - y.cpu().numpy()).max() <= 1e-10 * np.abs(x).max()
    o_obs, _, _, _ = ba.observation_grad(None, gl)          # None = 0
    p_obs, _, _, _ = ba.observation_grad(np.zeros_like(gp), gl)
    assert np.abs(o_obs - p_obs).max() <= 1e-10 * np.abs(p_obs).max()


def test_window_from_the_device_map_uses_last_edges_order(svs, oracle):
    pb = synth.make_window(30, 3000, seed=6)
    m, win, act = synth_graph.make_map(pb, seed=6)
    dm, b1 = svs.DeviceMap(), svs.BundleAdjuster()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    fixed = np.zeros(len(win), np.uint8)
    fixed[0] = 1
    E = dm.set_problem(b1, win, act, pb.cam, fixed=fixed, c_i=pb.c_i, c_j=pb.c_j, c_T=pb.c_T, c_Lambda=pb.c_Lambda)
    ep, es, ea, obs, info = dm.last_edges(E)
    pa = dataclasses.replace(pb, E=E, L=len(act), pose_qt=b1.poses(), psi=b1.points(), fixed=fixed, e_point=ep,
                             e_pose=es, e_anchor=ea, e_obs=obs, e_info=info)
    gp, gl = _upstream(pa, 8)
    dobs, dinfo, rc, _ = b1.observation_grad(gp, gl)
    assert rc == 0
    r_obs, r_info = ref.observation_grad(oracle, pa, gp, gl)
    _close(dobs, r_obs, "dL/dobs")
    _close(dinfo, r_info, "dL/dinfo")
    dm.close(); b1.close()


def test_optimize_after_the_call_is_unchanged(ba):
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    poses, points, lm = ba.poses(), ba.points(), ba.lm_stats()
    ba.observation_grad(*_upstream(pb))
    assert np.array_equal(ba.poses(), poses) and np.array_equal(ba.points(), points)
    assert ba.lm_stats() == lm
    ba.optimize(2)
    with_grad = ba.poses(), ba.points()
    ba.set_problem(pb)
    ba.optimize(2)
    ba.optimize(2)
    for x, y in zip(with_grad, (ba.poses(), ba.points())):
        assert np.abs(x - y).max() <= 1e-10 * np.abs(y).max()   # FP64 atomics of the build: last bits only


def test_errors(ba, svs):
    b = svs.BundleAdjuster()
    with pytest.raises(svs.SvsError) as e:
        b.observation_grad()
    assert e.value.rc == -4   # SVS_ERR_STATE: no problem set
    b.close()
    pb = synth.make_config("C1")
    ba.set_problem(pb)
    with pytest.raises(svs.SvsError) as e:
        ba.observation_grad(lam=0.0)   # no fixed pose, lambda = 0: H is singular
    assert e.value.rc == -1 and "singular" in str(e.value)
    ba.set_problem(_fixed(pb, 0))
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(svs.SvsError) as e:
            ba.observation_grad(lam=bad)
        assert e.value.rc == -1
    assert ba.observation_grad()[2] == 0   # the handle stays usable


def test_sharded_handle_is_unsupported(svs):
    b = svs.BundleAdjuster()
    b.comm_init(1, 0, svs.comm_unique_id())
    pb = _fixed(synth.make_config("C1"), 0)
    b.set_problem_sharded(pb)
    with pytest.raises(svs.SvsError) as e:
        b.observation_grad()
    assert e.value.rc == -3   # SVS_ERR_UNSUPPORTED
    b.close()


@pytest.mark.parametrize("on_cuda", [True, False])
def test_autograd_backward_is_observation_grad(ba, on_cuda):
    import torch
    from scavislam_b200.autograd import optimise_window, pose_grad_to_tangent
    dev = "cuda" if on_cuda else "cpu"
    pb = _fixed(synth.make_config("C1"), 0)
    e_obs = torch.as_tensor(pb.e_obs, device=dev).requires_grad_()
    e_info = torch.as_tensor(pb.e_info, device=dev).requires_grad_()
    poses, psi = optimise_window(ba, pb, e_obs, e_info, 6)
    assert poses.shape == (pb.P, 7) and psi.shape == (pb.L, 3) and poses.device.type == dev
    rng = np.random.default_rng(9)
    wq = torch.as_tensor(rng.normal(size=(pb.P, 7)), device=dev)
    wl = torch.as_tensor(rng.normal(size=(pb.L, 3)), device=dev)
    loss = (wq * poses).sum() + (wl * psi).sum()
    loss.backward()
    g_delta = pose_grad_to_tangent(poses.detach().cpu(), wq.cpu()).numpy()
    dobs, dinfo, rc, _ = ba.observation_grad(g_delta, wl.cpu().numpy())
    assert rc == 0
    for got, want in ((e_obs.grad, dobs), (e_info.grad, dinfo)):
        assert got.device.type == dev
        assert np.abs(got.cpu().numpy() - want).max() <= 1e-10 * np.abs(want).max()
