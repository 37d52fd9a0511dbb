"""svs_ba_window_grad (gradients of the optimised window with respect to its observations, weights, pose-pose
constraints and stereo camera) against the dense reference of ba_window_grad_reference.py at the device's accepted
state, each output to <= 1e-8 of its largest entry, on the windows test_ba_grad_gpu.py covers.  The upstream gradient is
seeded random and includes fixed poses, whose entries must not matter.

The build kernels sum the reduced system with FP64 atomics, so two builds of one state agree only to the last bits; the
outputs of two calls are compared with a tolerance instead of bit equality for that reason.
"""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

import ba_window_grad_reference as wref
from scavislam_b200 import synth, synth_graph

pytestmark = pytest.mark.gpu

TOL = 1e-8
NAMES = ("obs", "info", "cT", "cLambda", "cam")


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


def _rel(got, want):
    return np.abs(np.asarray(got) - np.asarray(want)).max() / max(np.abs(want).max(), 1e-300)


def _close(got, want, what, tol=TOL):
    err = _rel(got, want)
    assert err <= tol, f"{what}: {err:.3e} of the largest entry"


def _check(ba, oracle, pb, robust=True, lam=0.0, iters=0, seed=0, same_tol=1e-12):
    ba.set_problem(pb)
    if iters:
        ba.optimize(iters, robust)
    gp, gl = _upstream(pb, seed)
    res, rc, st = ba.window_grad(gp, gl, robust, 1.0, lam)
    assert rc == 0 and set(res) == set(NAMES)
    assert res["cT"].shape == (pb.C, 6) and res["cLambda"].shape == (pb.C, 36) and res["cam"].shape == (4,)
    state = dataclasses.replace(pb, pose_qt=ba.poses(), psi=ba.points())
    want = wref.window_grad(oracle, state, gp, gl, robust, 1.0, lam)
    for k in NAMES:
        _close(res[k], want[k], f"dL/d{k}")
    # the observation outputs are svs_ba_observation_grad's (another build: the last bits may differ)
    dobs, dinfo, rc2, _ = ba.observation_grad(gp, gl, robust, 1.0, lam)
    assert rc2 == 0
    _close(res["obs"], dobs, "dL/dobs against observation_grad", same_tol)
    _close(res["info"], dinfo, "dL/dinfo against observation_grad", same_tol)
    # the fixed poses' entries of g do not matter
    gp2 = gp.copy()
    gp2[np.asarray(pb.fixed) != 0] = 1e3
    res2, _, _ = ba.window_grad(gp2, gl, robust, 1.0, lam, want=("cT", "cLambda", "cam"))
    for k in ("cT", "cLambda", "cam"):
        _close(res2[k], want[k], f"dL/d{k} with other fixed-pose gradients")
    assert st["P"] == pb.P and st["L"] == pb.L and st["E"] == pb.E
    return res, st, state


@pytest.mark.parametrize("robust", [True, False])
def test_c1_optimised_with_a_fixed_pose(ba, oracle, robust):
    res, _, state = _check(ba, oracle, _fixed(synth.make_config("C1"), 0), robust=robust, iters=4)
    # dL/dcam is the contraction of the same call's dL/dobs with de/dcam
    host = sum(wref.camera_jacobian(oracle, state, e).T @ res["obs"][e] for e in range(state.E))
    _close(res["cam"], host, "dL/dcam against the contraction of dL/dobs", 1e-12)
    assert np.array_equal(res["cLambda"].reshape(-1, 6, 6), np.transpose(res["cLambda"].reshape(-1, 6, 6), (0, 2, 1)))


def test_c1_without_fixed_pose_damped(ba, oracle):
    """No fixed pose: lambda = 1, as in test_ba_grad_gpu.py (the gauge direction's rounding error grows like 1/lambda).
    The same amplification applies to the last-bit differences between two builds: against observation_grad's call the
    observation outputs differed by 5.6e-12 of the largest entry on an H100, so that comparison is held to 1e-10 here
    (1e-12 on the windows with a fixed pose)."""
    _check(ba, oracle, synth.make_config("C1"), lam=1.0, iters=2, same_tol=1e-10)


def test_tracks_of_9_to_32_slots(ba, oracle):
    _check(ba, oracle, _fixed(synth.make_window(30, 1500, seed=31, T=14), 0), iters=2)


def test_tracks_longer_than_32_slots(ba, oracle):
    _check(ba, oracle, _fixed(synth.make_window(70, 900, seed=36, T=50), 0), iters=1)
    assert ba.lm_stats()["max_track"] > 33


def test_visibility_dropouts(ba, oracle):
    _check(ba, oracle, _fixed(synth.with_dropouts(synth.make_window(40, 1200, seed=41), 0.2, seed=3), 0), iters=2)


def test_loop_closures_two_ended_with_separator(ba, oracle):
    pb = _fixed(synth.with_loop_closures(synth.make_window(60, 1000, seed=32), 3, seed=1), 0)
    _, st, _ = _check(ba, oracle, pb, iters=2)
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
    _, st, _ = _check(ba, oracle, _fixed(pb, 0))
    assert st["general"] == 1


def test_single_chain_solver(svs, oracle):
    os.environ["SVS_SOLVE_CHAIN"] = "1"
    try:
        b = svs.BundleAdjuster()
        _, st, _ = _check(b, oracle, _fixed(synth.make_window(60, 1000, seed=34), 0), iters=1)
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
    res, _, _ = _check(ba, oracle, pb, iters=2)
    assert not res["obs"][5].any() and not res["info"][5].any()


def test_constraint_between_two_fixed_poses_gets_exactly_zero(ba, oracle):
    pb = _fixed(synth.make_config("C1"), 2, 3)
    both = (np.isin(pb.c_i, [2, 3]) & np.isin(pb.c_j, [2, 3]))
    assert both.sum() == 2   # (2, 3) and (3, 2)
    res, _, _ = _check(ba, oracle, pb, iters=2)
    assert np.all(res["cT"][both] == 0) and np.all(res["cLambda"][both] == 0)
    assert np.abs(res["cT"][~both]).max() > 0


def test_host_and_cuda_tensor_arrays_agree(ba):
    import torch
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    gp, gl = _upstream(pb, 6)
    h, rc, _ = ba.window_grad(gp, gl)
    t, rc2, _ = ba.window_grad(torch.as_tensor(gp, device="cuda"), torch.as_tensor(gl, device="cuda"))
    assert rc == rc2 == 0
    for k in NAMES:
        assert t[k].is_cuda
        _close(t[k].cpu().numpy(), h[k], f"dL/d{k} CUDA against host", 1e-10)


@pytest.mark.parametrize("on_cuda", [True, False])
def test_null_outputs_are_left_untouched(ba, svs, on_cuda):
    """Each output alone, with every other member NULL: the others keep their sentinel, and the requested one equals
    the all-outputs call."""
    import torch
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    gp, gl = _upstream(pb, 7)
    full, _, _ = ba.window_grad(gp, gl)
    dev = "cuda" if on_cuda else "cpu"
    shapes = {k: tuple(np.shape(full[k])) for k in NAMES}
    g = [torch.as_tensor(a, device=dev) for a in (gp, gl)]
    for only in NAMES:
        bufs = {k: torch.full(shapes[k], float("nan"), dtype=torch.float64, device=dev) for k in NAMES}
        out = svs.SvsBaGradOut()
        setattr(out, svs.BundleAdjuster._GRAD_OUT[only][0], bufs[only].data_ptr())
        st = svs.SvsBaGradStats()
        torch.cuda.synchronize()
        rc = svs.lib().svs_ba_window_grad(ba._h, 1, 1.0, 0.0, g[0].data_ptr(), g[1].data_ptr(), C.byref(out),
                                          int(on_cuda), C.byref(st))
        assert rc == 0
        for k in NAMES:
            if k == only:
                _close(bufs[k].cpu().numpy(), full[k], f"dL/d{k} alone", 1e-10)
            else:
                assert torch.isnan(bufs[k]).all(), f"{k} was written when only {only} was requested"
    # no outputs at all: a valid call
    assert svs.lib().svs_ba_window_grad(ba._h, 1, 1.0, 0.0, None, None, None, 0, None) == 0


def test_optimize_after_the_call_is_unchanged(ba):
    pb = _fixed(synth.make_config("C1"), 0)
    ba.set_problem(pb)
    ba.optimize(2)
    poses, points, lm = ba.poses(), ba.points(), ba.lm_stats()
    ba.window_grad(*_upstream(pb))
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
    import torch
    b = svs.BundleAdjuster()
    with pytest.raises(svs.SvsError) as e:
        b.window_grad()
    assert e.value.rc == -4   # SVS_ERR_STATE: no problem set
    b.close()
    pb = synth.make_config("C1")
    ba.set_problem(pb)
    with pytest.raises(svs.SvsError) as e:
        ba.window_grad(lam=0.0)   # no fixed pose, lambda = 0: H is singular
    assert e.value.rc == -1 and "singular" in str(e.value) and "svs_ba_window_grad" in str(e.value)
    ba.set_problem(_fixed(pb, 0))
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(svs.SvsError) as e:
            ba.window_grad(lam=bad)
        assert e.value.rc == -1
    # on_device with a host array as an output: refused before anything is enqueued
    host = np.full((pb.C, 6), 7.0)
    dev = torch.zeros((pb.C, 36), dtype=torch.float64, device="cuda")
    out = svs.SvsBaGradOut()
    out.dL_dcT, out.dL_dcLambda = host.ctypes.data, dev.data_ptr()
    rc = svs.lib().svs_ba_window_grad(ba._h, 1, 1.0, 0.0, None, None, C.byref(out), 1, None)
    assert rc == -1 and "device memory" in svs.lib().svs_last_error(ba._h).decode()
    assert (host == 7.0).all()
    with pytest.raises(ValueError):
        ba.window_grad(want=("cT", "nope"))
    assert ba.window_grad()[1] == 0   # the handle stays usable


def test_sharded_handle_is_unsupported(svs):
    b = svs.BundleAdjuster()
    b.comm_init(1, 0, svs.comm_unique_id())
    pb = _fixed(synth.make_config("C1"), 0)
    b.set_problem_sharded(pb)
    with pytest.raises(svs.SvsError) as e:
        b.window_grad()
    assert e.value.rc == -3   # SVS_ERR_UNSUPPORTED
    b.close()


def test_window_from_the_device_map_keeps_the_constraint_order(svs, oracle):
    """The constraints go to set_problem_from_map in a shuffled order; their gradients come back in that order."""
    pb = synth.make_window(30, 3000, seed=6)
    m, win, act = synth_graph.make_map(pb, seed=6)
    dm, b1 = svs.DeviceMap(), svs.BundleAdjuster()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    fixed = np.zeros(len(win), np.uint8)
    fixed[0] = 1
    perm = np.random.default_rng(3).permutation(pb.C)
    ci, cj, cT, cL = pb.c_i[perm], pb.c_j[perm], pb.c_T[perm], pb.c_Lambda[perm]
    E = dm.set_problem(b1, win, act, pb.cam, fixed=fixed, c_i=ci, c_j=cj, c_T=cT, c_Lambda=cL)
    ep, es, ea, obs, info = dm.last_edges(E)
    pa = dataclasses.replace(pb, E=E, L=len(act), pose_qt=b1.poses(), psi=b1.points(), fixed=fixed, e_point=ep,
                             e_pose=es, e_anchor=ea, e_obs=obs, e_info=info, c_i=ci, c_j=cj, c_T=cT, c_Lambda=cL)
    gp, gl = _upstream(pa, 8)
    res, rc, _ = b1.window_grad(gp, gl)
    assert rc == 0
    want = wref.window_grad(oracle, pa, gp, gl)
    for k in NAMES:
        _close(res[k], want[k], f"dL/d{k}")
    dm.close(); b1.close()


@pytest.mark.parametrize("on_cuda", [True, False])
def test_autograd_backward_fills_constraint_and_camera_grads(ba, on_cuda):
    import torch
    from scavislam_b200.autograd import optimise_window, pose_grad_to_tangent, tangent_grad_to_pose
    dev = "cuda" if on_cuda else "cpu"
    pb = _fixed(synth.make_config("C1"), 0)
    leaf = lambda a: torch.as_tensor(np.array(a, np.float64), device=dev).requires_grad_()
    e_obs, e_info = leaf(pb.e_obs), leaf(pb.e_info)
    c_T, c_Lambda, cam = leaf(pb.c_T), leaf(pb.c_Lambda.reshape(-1, 6, 6)), leaf(pb.cam)
    poses, psi = optimise_window(ba, pb, e_obs, e_info, 6, c_T=c_T, c_Lambda=c_Lambda, cam=cam)
    assert poses.device.type == dev
    rng = np.random.default_rng(9)
    wq = torch.as_tensor(rng.normal(size=(pb.P, 7)), device=dev)
    wl = torch.as_tensor(rng.normal(size=(pb.L, 3)), device=dev)
    ((wq * poses).sum() + (wl * psi).sum()).backward()
    g_delta = pose_grad_to_tangent(poses.detach().cpu(), wq.cpu()).numpy()
    res, rc, _ = ba.window_grad(g_delta, wl.cpu().numpy())
    assert rc == 0
    want = dict(obs=res["obs"], info=res["info"], cLambda=res["cLambda"].reshape(-1, 6, 6), cam=res["cam"],
                cT=tangent_grad_to_pose(torch.as_tensor(pb.c_T), torch.as_tensor(res["cT"])).numpy())
    for k, t in (("obs", e_obs), ("info", e_info), ("cT", c_T), ("cLambda", c_Lambda), ("cam", cam)):
        assert t.grad is not None and t.grad.device.type == dev and t.grad.shape == t.shape, k
        _close(t.grad.cpu().numpy(), want[k], f"{k}.grad", 1e-10)


def test_autograd_without_them_is_observation_grad(ba):
    import torch
    from scavislam_b200.autograd import optimise_window, pose_grad_to_tangent
    pb = _fixed(synth.make_config("C1"), 0)
    e_obs = torch.as_tensor(pb.e_obs, device="cuda").requires_grad_()
    e_info = torch.as_tensor(pb.e_info, device="cuda").requires_grad_()
    poses, psi = optimise_window(ba, pb, e_obs, e_info, 6)
    rng = np.random.default_rng(10)
    wq = torch.as_tensor(rng.normal(size=(pb.P, 7)), device="cuda")
    wl = torch.as_tensor(rng.normal(size=(pb.L, 3)), device="cuda")
    ((wq * poses).sum() + (wl * psi).sum()).backward()
    dobs, dinfo, rc, _ = ba.observation_grad(pose_grad_to_tangent(poses.detach().cpu(), wq.cpu()).numpy(),
                                             wl.cpu().numpy())
    assert rc == 0
    _close(e_obs.grad.cpu().numpy(), dobs, "e_obs.grad", 1e-10)
    _close(e_info.grad.cpu().numpy(), dinfo, "e_info.grad", 1e-10)
