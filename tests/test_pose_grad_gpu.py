"""svs_pose_grad and svs_calcFastMotionOnly_device on the GPU: the device gradient against the dense reference of
pose_grad_reference.py at the device's own returned pose, central differences of the device forward, bit-identity
(repeated calls, host against CUDA-tensor input, the forward after a gradient call), the error codes and
scavislam_b200.autograd.track_pose."""
import ctypes as C

import numpy as np
import pytest

import pose_grad_reference as ref
from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth_images as si
from scavislam_b200 import synth_pose as sp

pytestmark = pytest.mark.gpu
I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
KERNEL = 2.0   # PoseOptimizerParams(true, 2, 15), the front end's setting


def _forward(po, tr, robust=True, iters=50, torch_dev=None):
    args = (tr["pid"], tr["obs"], tr["xyz"])
    if torch_dev is not None:
        import torch
        args = tuple(torch.as_tensor(a, device=torch_dev) for a in args)
    return po.calc_fast_motion_only(*args, tr["cam"], tr["T_init"], robust, KERNEL, iters)


def _rel(got, want):
    return np.abs(np.asarray(got) - want).max() / max(np.abs(want).max(), 1e-300)


# (n, seed, outlier_frac, shared_points, lambda, the launch shape it takes)
SHAPES = [
    (20, 1, 0.0, False, 0.0, "one CTA"),
    (333, 2, 0.1, False, 0.0, "one CTA"),
    (512, 3, 0.1, False, 0.0, "one CTA, the largest n it takes"),
    (513, 4, 0.1, False, 0.0, "8-CTA cluster, the smallest n it takes"),
    (1800, 5, 0.15, True, 0.0, "8-CTA cluster, shared points"),
    (5000, 6, 0.1, False, 0.0, "8-CTA cluster, outliers"),
    (1, 7, 0.0, False, 10.0, "one CTA; n = 1: H has rank 3, lambda > 0"),
]


@pytest.mark.parametrize("n,seed,out,shared,lam,shape", SHAPES, ids=[f"n{s[0]}" for s in SHAPES])
def test_matches_reference(svs, oracle, n, seed, out, shared, lam, shape):
    tr = sp.make_track(n, seed=seed, outlier_frac=out, shared_points=shared)
    po = svs.PoseOptimizer()
    T, st = _forward(po, tr)
    assert st["num_obs"] == n
    g = np.random.default_rng(seed).normal(size=6)
    res, rc, gst = po.grad(g, lam)
    assert rc == 0 and (gst["num_obs"], gst["npoints"]) == (n, len(tr["xyz"]))
    dobs, dxyz, dcam, _ = ref.pose_grad(oracle, tr["pid"], tr["obs"], tr["xyz"], tr["cam"], T, g, lam, True, KERNEL)
    if shared:
        assert np.bincount(tr["pid"]).min() >= 2   # every point's gradient is a sum
    for name, want in (("obs", dobs), ("xyz", dxyz), ("cam", dcam)):
        assert _rel(res[name], want) <= 1e-10, (name, shape, _rel(res[name], want))
    po.close()


@pytest.mark.parametrize("n,seed", [(333, 11), (1800, 12)])
def test_central_differences_of_the_device_forward(svs, n, seed):
    """Outlier-free tracks, robust off: the LM reaches its root to ~1e-15, so the device forward itself can be
    differentiated.  Tolerances as in test_pose_grad_cpu.py (Gauss-Newton error of 0.3 px residuals)."""
    tr = sp.make_track(n, seed=seed, shared_points=n > 1000)
    po = svs.PoseOptimizer()
    T, _ = _forward(po, tr, robust=False)
    g = np.random.default_rng(seed).normal(size=6)
    res, rc, _ = po.grad(g)
    assert rc == 0
    from oracle import pyoracle as oracle

    def loss(**kw):
        t = dict(tr, **kw)
        Tp, _ = po.calc_fast_motion_only(t["pid"], t["obs"], t["xyz"], t["cam"], tr["T_init"], False, KERNEL, 50)
        return float(g @ ref.tangent(oracle, Tp, T))

    def cd(name, idx, h):
        vals = []
        for s in (1, -1):
            a = np.array(tr[name], np.float64)
            a[idx] += s * h
            vals.append(loss(**{name: a}))
        return (vals[0] - vals[1]) / (2 * h)

    rng = np.random.default_rng(3)
    obs_i = rng.choice(n, 3, replace=False)
    e_obs = max(abs(cd("obs", (i, k), 1e-3) - res["obs"][i, k]) for i in obs_i for k in range(3))
    e_xyz = max(abs(cd("xyz", (int(tr["pid"][i]), k), 1e-5) - res["xyz"][tr["pid"][i], k]) for i in obs_i for k in range(3))
    e_cam = max(abs(cd("cam", k, h) - res["cam"][k]) for k, h in enumerate((1e-3, 1e-3, 1e-3, 1e-6)))
    errs = (e_obs / np.abs(res["obs"]).max(), e_xyz / np.abs(res["xyz"]).max(), e_cam / np.abs(res["cam"]).max())
    assert all(e <= t for e, t in zip(errs, (1e-3, 1e-2, 5e-3))), errs
    po.close()


@pytest.mark.parametrize("n", [333, 1800])
def test_bit_identical_repeats_and_device_input(svs, n):
    import torch
    tr = sp.make_track(n, seed=21, outlier_frac=0.1, shared_points=n > 1000)
    g = np.random.default_rng(2).normal(size=6)
    po = svs.PoseOptimizer()
    T_h, st_h = _forward(po, tr)
    a, rc_a, _ = po.grad(g)
    b, rc_b, _ = po.grad(g)
    assert rc_a == rc_b == 0
    for k in a:
        assert np.array_equal(a[k], b[k]), k                                   # two calls
    T_d, st_d = _forward(po, tr, torch_dev="cuda:0")                           # svs_calcFastMotionOnly_device
    assert np.array_equal(T_d, T_h)
    assert {k: st_d[k] for k in st_d if k != "ms"} == {k: st_h[k] for k in st_h if k != "ms"}
    d, rc_d, _ = po.grad(torch.as_tensor(g, device="cuda:0"))                  # every array on the device
    assert rc_d == 0
    for k in a:
        assert isinstance(d[k], torch.Tensor) and d[k].is_cuda
        assert np.array_equal(d[k].cpu().numpy(), a[k]), k
    po.close()


def test_requested_outputs_only(svs):
    """A NULL output is neither computed nor written; each requested one equals the full call's bits."""
    import torch
    tr = sp.make_track(700, seed=31, outlier_frac=0.1, shared_points=True)
    g = np.random.default_rng(4).normal(size=6)
    po = svs.PoseOptimizer()
    _forward(po, tr)
    full, _, _ = po.grad(g)
    for w in ("obs", "xyz", "cam"):
        part, rc, _ = po.grad(g, want=(w,))
        assert rc == 0 and list(part) == [w] and np.array_equal(part[w], full[w])
    res, rc, _ = po.grad(g, want=())
    assert rc == 0 and res == {}
    # device outputs: sentinels around the one requested output stay as they were
    buf = torch.full((3 * 700 + 8,), 7.0, dtype=torch.float64, device="cuda:0")
    gd = torch.as_tensor(g, device="cuda:0")
    torch.cuda.synchronize()
    rc = svs.lib().svs_pose_grad(po._h, 0.0, gd.data_ptr(), buf[4:].data_ptr(), None, None, 1, None)
    assert rc == 0
    out = buf.cpu().numpy()
    assert (out[:4] == 7.0).all() and (out[4 + 3 * 700:] == 7.0).all()
    assert np.array_equal(out[4:4 + 3 * 700].reshape(700, 3), full["obs"])
    po.close()


def test_forward_after_gradient_is_unchanged(svs):
    tr = sp.make_track(900, seed=41, outlier_frac=0.1)
    tr2 = sp.make_track(300, seed=42, outlier_frac=0.1)
    po, fresh = svs.PoseOptimizer(), svs.PoseOptimizer()
    T1, s1 = _forward(po, tr)
    po.grad(np.ones(6))
    T2, s2 = _forward(po, tr)
    assert np.array_equal(T1, T2) and s1["chi2"] == s2["chi2"] and s1["trials"] == s2["trials"]
    po.grad(np.ones(6))
    T3, _ = _forward(po, tr2)                      # another track on the same handle
    T4, _ = _forward(fresh, tr2)
    assert np.array_equal(T3, T4)
    po.close(); fresh.close()


def _matcher_run(svs, po):
    """One successful svs_calcFastMotionOnly_matched (as tests/test_pose_gpu.py drives it)."""
    seq = si.sequence(2)
    cams = fi.level_cams()
    cam = (cams[0][0], cams[0][1], cams[0][2], cams[0][3])
    lv2 = [(640 >> l, 480 >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(2)]
    fg = svs.FastGrid(640, 480, 222, 74, 25, 3, 3)
    fg.set_image(seq[0]["img"])
    kxy, _ = fg.detect_adaptively(5)
    fg.set_image(seq[1]["img"])
    xy, off = fg.detect_adaptively(5)
    m = svs.GuidedMatcher(lv2)
    m.set_keyframe(0, I7, fi.uint8_pyramid(seq[0]["img"], 2))
    m.set_current(fi.uint8_pyramid(seq[1]["img"], 2), seq[1]["disp"])
    m.set_features(0, xy, np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(9)]).astype(np.int32))
    m.set_features(1, np.zeros((0, 2), np.int32), np.zeros(0, np.int32))
    d = seq[0]["disp"][kxy[:, 1], kxy[:, 0]]
    kxy, d = kxy[d > 0], d[d > 0]
    z = cam[0] * cam[3] / d
    pts = np.zeros(len(kxy), svs.MATCH_POINT_DTYPE)
    pts["xyz_anchor"] = np.stack([(kxy[:, 0] - cam[1]) / cam[0] * z, (kxy[:, 1] - cam[2]) / cam[0] * z, z], 1)
    pts["anchor_obs_pyr"] = kxy
    m.match(I7, I7, pts, 4, 22, 10)
    po.calc_fast_motion_only_matched(m, cam, I7, True, 2.0, 15)
    m.close(); fg.close()


def test_error_codes(svs):
    import torch
    L = svs.lib()
    tr = sp.make_track(50, seed=51)
    po = svs.PoseOptimizer(max_obs=64)
    g = np.zeros(6)
    with pytest.raises(svs.SvsError) as e:                 # before any forward call
        po.grad(g)
    assert e.value.rc == -4
    _forward(po, tr)
    for lam in (-1.0, float("nan"), float("inf")):
        with pytest.raises(svs.SvsError) as e:
            po.grad(g, lam)
        assert e.value.rc == -1
    # on_device = 1 with a host array: refused before anything is enqueued
    out = np.zeros((50, 3))
    assert L.svs_pose_grad(po._h, 0.0, None, out.ctypes.data, None, None, 1, None) == -1
    assert not out.any()
    assert po.grad(g)[1] == 0                               # the problem is still there
    # a failed forward call leaves nothing to differentiate: point_id out of range, host and device input
    bad = tr["pid"].copy(); bad[7] = 50
    for dev in (None, "cuda:0"):
        _forward(po, tr)
        t = dict(tr, pid=bad)
        with pytest.raises(svs.SvsError) as e:
            _forward(po, t, torch_dev=dev)
        assert e.value.rc == -1 and "point_id outside point_list" in str(e.value)
        with pytest.raises(svs.SvsError) as e:
            po.grad(g)
        assert e.value.rc == -4
    # device input: a host pointer is refused
    c, p, st = svs.SvsCam(*tr["cam"]), po._params(True, KERNEL, 50, -1.0), svs.SvsPoseStats()
    T = tr["T_init"].copy()
    pid_d = torch.as_tensor(tr["pid"], device="cuda:0")
    xyz_d = torch.as_tensor(tr["xyz"], device="cuda:0")
    obs_h = np.ascontiguousarray(tr["obs"])
    assert L.svs_calcFastMotionOnly_device(po._h, 50, pid_d.data_ptr(), obs_h.ctypes.data, 50, xyz_d.data_ptr(),
                                           C.byref(c), C.byref(p), svs._dp(T), C.byref(st)) == -1
    # the matcher's variant leaves nothing to differentiate either
    pm = svs.PoseOptimizer()
    _forward(pm, tr)
    _matcher_run(svs, pm)
    with pytest.raises(svs.SvsError) as e:
        pm.grad(g)
    assert e.value.rc == -4
    # H + lambda I not positive definite: one observation on the optical axis (its J has a zero column), lambda = 0
    one = dict(pid=np.zeros(1, np.int32), obs=np.array([[321.0, 240.5, 311.0]]), xyz=np.array([[0.0, 0.0, 5.0]]),
               cam=tr["cam"], T_init=I7)
    _forward(po, one, iters=0)
    res, rc, _ = po.grad(np.ones(6), 0.0)
    assert rc == 1 and all(not a.any() for a in res.values())
    res, rc, _ = po.grad(np.ones(6), 1.0)
    assert rc == 0 and res["obs"].any()
    po.close(); pm.close()


@pytest.mark.parametrize("device", ["cpu", "cuda:0"])
def test_track_pose_backward(svs, device):
    import torch
    from scavislam_b200.autograd import pose_grad_to_tangent, track_pose
    tr = sp.make_track(600, seed=61, outlier_frac=0.1, shared_points=True)
    obs = torch.tensor(tr["obs"], device=device, requires_grad=True)
    xyz = torch.tensor(tr["xyz"], device=device, requires_grad=True)
    cam = torch.tensor(tr["cam"], device=device, requires_grad=True)
    po = svs.PoseOptimizer()
    T = track_pose(po, tr["pid"], obs, xyz, cam, tr["T_init"], True, KERNEL, 15)
    assert T.dtype == torch.float64 and T.device == torch.device(device) and T.shape == (7,)
    w = torch.as_tensor(np.random.default_rng(6).normal(size=7), device=device)
    (T * w).sum().backward()
    g = pose_grad_to_tangent(T.detach()[None].cpu(), w[None].cpu())[0].numpy()
    want, rc, _ = po.grad(g)
    assert rc == 0
    for t, name in ((obs, "obs"), (xyz, "xyz"), (cam, "cam")):
        assert t.grad is not None and t.grad.device == torch.device(device)
        assert np.abs(t.grad.cpu().numpy() - want[name]).max() <= 1e-12 * np.abs(want[name]).max(), name
    T_np, _ = po.calc_fast_motion_only(tr["pid"], tr["obs"], tr["xyz"], tr["cam"], tr["T_init"], True, KERNEL, 15)
    assert np.array_equal(T.detach().cpu().numpy(), T_np)
    po.close()
