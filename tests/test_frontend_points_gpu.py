"""GPU parity tests of svs_match_track, svs_processMatchedPoints and svs_addMorePoints against
oracle/frontend_oracle.c: every output bit-identical (counts, flags, order, doubles)."""
import numpy as np
import pytest

from oracle import frontend_pyoracle as fp
from scavislam_b200 import capi
from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth_images as si

pytestmark = pytest.mark.gpu

NLV = 2
I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
SHAPES = {
    "640x480_2": ([(640, 480), (320, 240)], (500., 319.5, 239.5, 0.12)),
    "newcollege": ([(512, 384), (256, 192), (128, 96)], (389.956085, 254.903519, 201.899490, 0.110014)),
    "1241x376": ([(1241, 376), (620, 188)], (718.856, 607.1928, 185.2157, 0.537)),
}


def _features(oracle, pyr):
    feats = []
    for l in range(NLV):
        g = oracle.fast_grid(640 >> l, 480 >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
        xy, off = oracle.fast_detect_adaptively(pyr[l], g, 5)
        content = np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(9)]).astype(np.int32)
        feats.append((xy, content))
    return feats


def _points(oracle, kf_pyr, disp, cams):
    pts = []
    for l in range(NLV):
        g = oracle.fast_grid(640 >> l, 480 >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
        kxy, _ = oracle.fast_detect_adaptively(kf_pyr[l], g, 5)
        d = disp[kxy[:, 1] << l, kxy[:, 0] << l] / (1 << l)
        kxy, d = kxy[d > 0], d[d > 0]
        z = cams[l][0] * cams[l][3] / d
        p = np.zeros(len(kxy), oracle.MATCH_POINT_DTYPE)
        p["anchor_level"] = l
        p["xyz_anchor"] = np.stack([(kxy[:, 0] - cams[l][1]) / cams[l][0] * z, (kxy[:, 1] - cams[l][2]) / cams[l][0] * z, z], 1)
        p["anchor_obs_pyr"] = kxy
        pts.append(p)
    return np.concatenate(pts)


@pytest.fixture(scope="module")
def scene(svs, oracle):
    seq = si.sequence(2)
    cams = fi.level_cams(nlevels=NLV)
    levels = [(640 >> l, 480 >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(NLV)]
    kf_pyr = fi.uint8_pyramid(seq[0]["img"], NLV)
    cur_pyr = fi.uint8_pyramid(seq[1]["img"], NLV)
    feats = _features(oracle, cur_pyr)
    pts = _points(oracle, kf_pyr, seq[0]["disp"], cams)
    T_cur = oracle.se3_exp(np.array([0.001, 0.0, -0.02, 0.0, -0.0035, 0.0]))
    T_key_w = oracle.se3_exp(np.array([0.3, -0.1, 0.2, 0.01, 0.02, -0.01]))
    m = svs.GuidedMatcher(levels)
    m.set_keyframe(0, T_key_w, kf_pyr)
    m.set_current(cur_pyr, seq[1]["disp"])
    for l in range(NLV):
        m.set_features(l, *feats[l])
    cam = tuple(cams[0][:4])
    yield dict(m=m, pts=pts, T_cur=T_cur, T_key_w=T_key_w, cam=cam, disp=seq[1]["disp"], feats=feats)
    m.close()


def _split(pts, sizes):
    ends = np.cumsum(sizes)
    return [pts[a:b] for a, b in zip([0] + list(ends[:-1]), ends)]


def _group_sizes(n):
    return [n // 6, n // 6, n // 6, n // 6, n - 4 * (n // 6)]


@pytest.mark.parametrize("cut", ["before_first", "after_first", "never"])
def test_match_track_budget(scene, cut):
    """The budget cuts before the first neighbour group, after keeping the first, or never; with no cut the results are
    byte-identical to svs_match's and calcFastMotionOnly_matched gives the same bits after either."""
    m, pts = scene["m"], scene["pts"]
    sizes = _group_sizes(len(pts))
    ends = np.cumsum(sizes)
    full = m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10)
    mg = [int(full["matched"][a:b].sum()) for a, b in zip([0] + list(ends[:-1]), ends)]
    assert mg[1] > 0 and mg[2] > 0
    nmax = {"before_first": 2 * mg[0], "after_first": 2 * (mg[0] + mg[1]), "never": 10 ** 6}[cut]
    kept = {"before_first": [1, 0, 0, 0, 1], "after_first": [1, 1, 0, 0, 1], "never": [1] * 5}[cut]
    want, a, b = fp.c_budget(full, ends, nmax)
    res, na, nb = m.match_track(scene["T_cur"], scene["T_key_w"], _split(pts, sizes), nmax, 4, 22, 10)
    assert (na, nb) == (a, b)
    assert np.array_equal(res["matched"], want["matched"])
    got = [int(res["matched"][a:b].sum()) for a, b in zip([0] + list(ends[:-1]), ends)]
    assert got == [g * k for g, k in zip(mg, kept)]
    assert na == sum(got[:-1]) and nb == sum(got)
    keep = res["matched"] == 1
    assert np.array_equal(res[keep].tobytes(), full[keep].tobytes())
    if cut == "never":
        assert res.tobytes() == full.tobytes()
        po = capi.PoseOptimizer()
        T1, _ = po.calc_fast_motion_only_matched(m, scene["cam"], scene["T_cur"])
        m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10)
        T2, _ = po.calc_fast_motion_only_matched(m, scene["cam"], scene["T_cur"])
        assert T1.tobytes() == T2.tobytes()
        po.close()


@pytest.mark.parametrize("n_new_frac", [0.0, 0.5, 1.0])
def test_process_after_match(scene, n_new_frac):
    m, pts, cam = scene["m"], scene["pts"], scene["cam"]
    res = m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10)
    n_new = int(len(pts) * n_new_frac)
    out, st, flags, drop = m.process_matched_points(scene["T_cur"], cam, n_new)
    wout, wst, wflags = fp.c_process(res, pts["anchor_level"], n_new, scene["T_cur"], cam, 640, 480)
    assert out.tobytes() == wout.tobytes()
    d = fp.stats_dict(wst)
    for k in ("num_matched_points", "num_tracked", "num_new"):
        assert st[k] == d[k], k
    assert np.array_equal(st["grid2x2"], d["grid2x2"]) and np.array_equal(st["grid3x3"], d["grid3x3"])
    assert np.array_equal(np.float64(st["av_track_length"]), np.float64(d["av_track_length"]))
    assert np.array_equal(flags.reshape(-1), wflags)
    assert drop == bool(fp.c_drop(wst, scene["T_cur"]))
    assert drop == capi.shall_we_drop_new_keyframe(st, scene["T_cur"])
    # addMorePoints from the processed points
    sizes = [(640, 480), (320, 240)]
    corners = [f[0] for f in scene["feats"]]
    for nmax in (300, 30):
        p = capi.frontend_params(num_max_points=nmax, seed=11)
        pts_g, rows_g, cnt_g = m.add_more_points(0, cam, 2, params=p)
        want = fp.c_seed(sizes, corners, scene["disp"], wout, d["num_matched_points"][:2], wflags, 2, nmax, 11, I7, cam, 2)
        assert pts_g.tobytes() == want[0].tobytes() and rows_g.tobytes() == want[1].tobytes()
        assert list(cnt_g) == list(want[2])


def test_seed_fresh_on_frames(scene):
    m, cam = scene["m"], scene["cam"]
    sizes = [(640, 480), (320, 240)]
    corners = [f[0] for f in scene["feats"]]
    for seed in (0, 3):
        g = m.add_more_points(1, cam, 1, params=capi.frontend_params(seed=seed))
        want = fp.c_seed(sizes, corners, scene["disp"], np.zeros(0, fp.TRACKED_DTYPE), [0, 0], np.ones(9, np.int32), 2,
                         300, seed, I7, cam, 1)
        assert g[0].tobytes() == want[0].tobytes() and g[1].tobytes() == want[1].tobytes()
        assert len(g[0]) > 100


def _seed_case(svs, sizes, cam, corners, disp, nmax=300, R=2, seed=0, T=I7):
    levels = [(w, h, cam[0] / (1 << l), cam[1], cam[2]) for l, (w, h) in enumerate(sizes)]
    m = svs.GuidedMatcher(levels, max_keypoints=max(len(c) for c in corners) + 1)
    m.set_current_disparity(disp)
    for l, c in enumerate(corners):
        m.set_features(l, c, np.zeros(len(c), np.int32))
    g = m.add_more_points(1, cam, 0, T_newkey_from_cur=T,
                          params=svs.frontend_params(num_max_points=nmax, newpoint_clearance=R, seed=seed))
    want = fp.c_seed(sizes, corners, disp, np.zeros(0, fp.TRACKED_DTYPE), [0] * len(sizes), np.ones(9, np.int32), R,
                     nmax, seed, T, cam, 0)
    assert g[0].tobytes() == want[0].tobytes() and g[1].tobytes() == want[1].tobytes()
    assert list(g[2]) == list(want[2])
    m.close()
    return g


@pytest.mark.parametrize("shape", list(SHAPES))
def test_seed_shapes(svs, shape):
    """Random corners with repeated positions, the 1-px border and disparities <= 0; the cap reached mid-depth."""
    sizes, cam = SHAPES[shape]
    rng = np.random.default_rng(21)
    w0, h0 = sizes[0]
    disp = rng.uniform(-2, 40, (h0, w0)).astype(np.float32)
    corners = []
    for l, (w, h) in enumerate(sizes):
        c = np.stack([rng.integers(0, w, 3000 >> l), rng.integers(0, h, 3000 >> l)], 1).astype(np.int32)
        c[-4:] = c[:4]
        c[:4] = [[0, 3], [w - 1, 5], [7, 0], [9, h - 1]]
        corners.append(c)
    T = np.array([0.01, -0.02, 0.005, 1, 0.1, -0.05, 0.2])
    T[:4] /= np.linalg.norm(T[:4])
    g = _seed_case(svs, sizes, cam, corners, disp, T=T)
    assert g[2][0] == 301                                   # level 0 stops at cap + 1, inside a depth of the order
    _seed_case(svs, sizes, cam, corners, disp, nmax=7, R=3, seed=5)


def test_seed_diagonal_chain(svs):
    """A lone diagonal chain of corners 1 px apart: every corner's window holds its neighbours, so each decision waits
    on the ones before it in emission order (the most rounds of the greedy)."""
    sizes, cam = [(512, 512)], (400., 255.5, 255.5, 0.1)
    disp = np.full((512, 512), 8, np.float32)
    chain = np.array([[i + 4, i + 4] for i in range(500)], np.int32)
    for R in (1, 2):
        g = _seed_case(svs, sizes, cam, [chain], disp, nmax=10 ** 6, R=R)
        assert 500 // (2 * R + 1) <= g[2][0] < 500


def test_seed_all_flags_off(svs, scene):
    """add flags all off (every 3x3 cell above min_num_points): nothing is seeded."""
    m, pts, cam = scene["m"], scene["pts"], scene["cam"]
    m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10)
    m.process_matched_points(scene["T_cur"], cam, 0, params=capi.frontend_params(min_num_points=-1))
    g = m.add_more_points(0, cam, 0, params=capi.frontend_params(min_num_points=-1))
    assert len(g[0]) == 0 and list(g[2]) == [0, 0]


def test_process_after_match_track_and_nothing_gated(scene):
    """After svs_match_track the gate sees the budgeted TrackData; a pose far off gates nothing: NaN track length."""
    m, pts, cam = scene["m"], scene["pts"], scene["cam"]
    sizes = _group_sizes(len(pts))
    res, na, nb = m.match_track(scene["T_cur"], scene["T_key_w"], _split(pts, sizes), 200, 4, 22, 10)
    out, st, flags, drop = m.process_matched_points(scene["T_cur"], cam, int(np.cumsum(sizes)[-2]))
    wout, wst, wflags = fp.c_process(res, pts["anchor_level"], int(np.cumsum(sizes)[-2]), scene["T_cur"], cam, 640, 480)
    assert out.tobytes() == wout.tobytes() and np.array_equal(flags.reshape(-1), wflags)
    T_far = np.array([0, 0, 0, 1, 3.0, 0, 0])
    out, st, flags, drop = m.process_matched_points(T_far, cam, 0)
    assert len(out) == 0 and np.isnan(st["av_track_length"]) and drop
    assert flags.reshape(-1).tolist() == [1] * 9


def test_state_errors_and_refusals(svs, scene):
    m, cam, pts = scene["m"], scene["cam"], scene["pts"]
    m2 = svs.GuidedMatcher([(64, 48, 50., 31.5, 23.5)])
    with pytest.raises(svs.SvsError) as e:
        m2.process_matched_points(I7, cam, 0)
    assert e.value.rc == -4
    with pytest.raises(svs.SvsError) as e:
        m2.add_more_points(0, cam, 0)                           # fresh = 0 without processMatchedPoints
    assert e.value.rc == -4
    m2.close()
    res = m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10)
    first = m.process_matched_points(scene["T_cur"], cam, 0)
    with pytest.raises(svs.SvsError) as e:
        m.process_matched_points(scene["T_cur"], cam, len(pts) + 1)
    assert e.value.rc == -1
    with pytest.raises(ValueError):
        m.match_track(scene["T_cur"], scene["T_key_w"], [pts[:5]], 300, 4, 22, 10)
    bad = np.array([len(pts) + 5, 3], np.int32)       # group_end out of order: refused before anything changes
    arr = np.ascontiguousarray(pts, capi.MATCH_POINT_DTYPE)
    a, b = capi.C.c_int(), capi.C.c_int()
    rc = capi.lib().svs_match_track(m._h, capi._dp(np.ascontiguousarray(scene["T_cur"])),
                                    capi._dp(np.ascontiguousarray(scene["T_key_w"])),
                                    arr.ctypes.data_as(capi.C.POINTER(capi.SvsMatchPoint)), len(arr), 2, capi._ip(bad),
                                    300, 4, 22, 10, None, capi.C.byref(a), capi.C.byref(b))
    assert rc == -1
    again = m.process_matched_points(scene["T_cur"], cam, 0)   # the last match's results are still in place
    assert again[0].tobytes() == first[0].tobytes()
    before = m.add_more_points(0, cam, 0)
    for bad_call in (lambda: m.add_more_points(2, cam, 0),
                     lambda: m.add_more_points(0, cam, 0, params=capi.frontend_params(newpoint_clearance=-1)),
                     lambda: m.process_matched_points(scene["T_cur"], cam, -1)):
        with pytest.raises(svs.SvsError) as e:
            bad_call()
        assert e.value.rc == -1
    after = m.add_more_points(0, cam, 0)                        # refusals left the processed points as they were
    assert before[0].tobytes() == after[0].tobytes() and before[1].tobytes() == after[1].tobytes()
    assert m.match(scene["T_cur"], scene["T_key_w"], pts, 4, 22, 10).tobytes() == res.tobytes()
    with pytest.raises(svs.SvsError) as e:                      # a new match: the processed points are gone
        m.add_more_points(0, cam, 0)
    assert e.value.rc == -4
