"""The device StereoBM (svs_stereo) against OpenCV's cv2.StereoBM with the reference's settings, bit for bit: the
1/16-px map (16 x the float output) equals cv2's int16 output element for element at the reference's camera, at
640x480 over the range of numberOfDisparities, at 1241x376 and at an odd size.

Every filtering stage is exercised on purpose.  The inputs are rendered pairs with pasted sparse-dot patches (texture
threshold), flat and low-contrast patches and a periodic texture (uniqueness, left-right check), and each named stage case
first asserts, with cv2 alone, that turning its stage off changes pixels on that input, so that a change of input
cannot silently stop testing a stage.  Then: the three kinds of image pointer give one map, and the device hand-over
into the dense trackers and the matcher gives what the host setters give with the map read back."""
import functools

import cv2
import numpy as np
import pytest

from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth_images as si

pytestmark = pytest.mark.gpu

SVS_ERR_INVALID = -1
I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
NC_CAM = (389.956085, 254.903519, 201.899490, 0.120005)   # data/newcollege.cfg, 512x384
ODD_CAM = (700.0, 620.5, 188.0, 0.12)                      # 1241x376


def cv_bm(left, right, ndisp, **stage_off):
    """cv2.StereoBM as calcDisparityCpu configures it; stage_off = {setter suffix: value} turns a stage off."""
    bm = cv2.StereoBM_create(numDisparities=ndisp, blockSize=7)
    bm.setPreFilterType(cv2.STEREO_BM_PREFILTER_XSOBEL)
    bm.setPreFilterCap(31); bm.setMinDisparity(0); bm.setTextureThreshold(10); bm.setUniquenessRatio(15)
    bm.setSpeckleWindowSize(100); bm.setSpeckleRange(32); bm.setDisp12MaxDiff(1)
    for k, v in stage_off.items():
        getattr(bm, "set" + k)(v)
    return bm.compute(left, right)


STAGE_OFF = dict(texture=("TextureThreshold", 0), uniqueness=("UniquenessRatio", 0),
                 left_right=("Disp12MaxDiff", -1), speckle=("SpeckleWindowSize", 0))


def _paste(left, right, y, x, patch, disp):
    h, w = patch.shape
    left[y:y + h, x:x + w] = patch
    right[y:y + h, x - disp:x - disp + w] = patch


@functools.lru_cache(maxsize=None)
def stress_pair(w, h, cam=None, seed=77):
    """A rendered pair with pasted sparse-dot, flat and low-contrast patches and a periodic texture, each at a known
    disparity, spread over the frame."""
    left, right, _ = si.render_stereo_pair(np.array([0.0, 0.0, 0.0]), 0.0, seed, w, h, cam)
    left, right = left.copy(), right.copy()
    rng = np.random.default_rng(seed)
    dots = np.full((max(h // 8, 16), max(w // 5, 24)), 120, np.uint8)
    dots[2::8, 2::8] += 1      # a lone +1 dot per 8x8 cell: unique matches, most windows below the texture threshold
    _paste(left, right, int(0.03 * h), int(0.3 * w), dots, 7)
    _paste(left, right, int(0.85 * h), int(0.2 * w), dots, 11)
    ph, pw = max(h // 10, 12), max(w // 10, 16)
    for k in range(3):
        y, x = int(h * (0.15 + 0.3 * k)), int(w * (0.3 + 0.2 * k))
        _paste(left, right, y, x, np.full((ph, pw), 90 + 40 * k, np.uint8), 6 + 3 * k)                   # flat
        low = (128 + rng.integers(-1, 2, (ph, pw))).astype(np.uint8)
        _paste(left, right, y, x + pw + 8, low, 9)                                                        # low contrast
        xs = np.arange(pw * 2)
        stripes = np.tile((100 + 70 * ((xs // 3) % 2)).astype(np.uint8), (ph, 1))
        _paste(left, right, min(y + ph + 6, h - ph - 1), x - pw // 2, stripes, 5 + k)                     # periodic
    return left, right


def device_map(svs, left, right, ndisp):
    h, w = left.shape
    sm = svs.StereoMatcher(w, h, ndisp, device=0)
    sm.compute(left, right)
    d = sm.disparity()
    sm.close()
    return d


def assert_bit_exact(d, ref):
    assert d.shape == ref.shape
    d16 = d * 16
    assert np.array_equal(d16, np.round(d16)), "the map is not in 1/16 px"
    bad = d16.astype(np.int32) != ref
    assert not bad.any(), f"{bad.sum()} pixels differ, first at {np.argwhere(bad)[:5].tolist()}"


# ---------------------------------------------------------------- 1. bit-exact with cv2

@pytest.mark.parametrize("ndisp", [16, 32, 64, 160])
def test_640x480_matches_opencv(svs, ndisp):
    left, right = stress_pair(640, 480)
    ref = cv_bm(left, right, ndisp)
    assert (ref > 0).mean() > 0.3
    assert_bit_exact(device_map(svs, left, right, ndisp), ref)


@pytest.mark.parametrize("w,h,cam,ndisp", [(512, 384, NC_CAM, 32), (1241, 376, ODD_CAM, 64),
                                           (639, 479, (570.342, 319.0, 239.0, 0.075), 32)])
def test_other_shapes_match_opencv(svs, w, h, cam, ndisp):
    left, right = stress_pair(w, h, cam)
    ref = cv_bm(left, right, ndisp)
    assert (ref > 0).mean() > 0.3
    assert_bit_exact(device_map(svs, left, right, ndisp), ref)


@pytest.mark.parametrize("ndisp", [16, 64])
def test_narrow_images_are_all_invalid(svs, ndisp):
    rng = np.random.default_rng(3)
    for w in (ndisp - 1, ndisp, ndisp + 3):
        left, right = (rng.integers(0, 256, (40, w), dtype=np.uint8) for _ in range(2))
        d = device_map(svs, left, right, ndisp)
        assert (d == -1).all(), w
        if w < ndisp:   # cv2 fills this map; up to ndisp + 5 columns wide it leaves it unwritten
            assert_bit_exact(d, cv_bm(left, right, ndisp))


# ---------------------------------------------------------------- 2. every stage reached

@pytest.mark.parametrize("stage", sorted(STAGE_OFF))
def test_stage_is_exercised_and_matches_opencv(svs, stage):
    left, right = stress_pair(640, 480)
    ref = cv_bm(left, right, 32)
    name, value = STAGE_OFF[stage]
    changed = (cv_bm(left, right, 32, **{name: value}) != ref).sum()
    assert changed > 50, f"turning the {stage} stage off changes only {changed} pixels on this input"
    assert_bit_exact(device_map(svs, left, right, 32), ref)


# ---------------------------------------------------------------- 3. pointer kinds

def test_host_and_device_images_give_one_map(svs):
    import torch
    left, right = stress_pair(640, 480)
    sm = svs.StereoMatcher(640, 480, 32, device=0)
    sm.compute(left, right)
    host = sm.disparity()
    prep = svs.FramePreprocessor(640, 480, 1, device=0)
    prep.process(left)
    sm.compute(prep.level(0), right)
    assert sm.disparity().tobytes() == host.tobytes()
    tl, tr = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()
    sm.compute(tl, tr)
    assert sm.disparity().tobytes() == host.tobytes()
    sm.compute(tl, tr)
    assert sm.disparity().tobytes() == host.tobytes()
    ptr, stride = sm.device_disparity()
    assert ptr and stride >= 640
    prep.close(); sm.close()


def test_tensor_written_on_a_torch_stream_is_complete(svs):
    """compute() orders its read after the torch stream that writes the image: here a side stream that first sleeps,
    then forms both images with kernels, and the map still equals the host one."""
    import torch
    left, right = stress_pair(640, 480)
    sm = svs.StereoMatcher(640, 480, 32, device=0)
    sm.compute(left, right)
    host = sm.disparity()
    lf, rf = torch.from_numpy(left).cuda().float(), torch.from_numpy(right).cuda().float()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        tl, tr = (lf * 1.0).to(torch.uint8), (rf * 1.0).to(torch.uint8)
        sm.compute(tl, tr)
    assert sm.disparity().tobytes() == host.tobytes()
    sm.close()


def test_images_of_the_wrong_kind_are_refused(svs):
    import torch
    left, right = stress_pair(640, 480)
    sm = svs.StereoMatcher(640, 480, 32, device=0)
    small = svs.FramePreprocessor(320, 240, 1, device=0)
    small.process(left[:240, :320])
    tl = torch.from_numpy(left).cuda()
    for bad in (left[:479], left.astype(np.uint16), small.level(0), tl.float(), tl.to(torch.int8), tl[:, :639],
                tl.t().contiguous()):
        with pytest.raises(svs.SvsError):
            sm.compute(bad, right)
    small.close(); sm.close()


# ---------------------------------------------------------------- 4. hand-over into the consumers

@pytest.fixture(scope="module")
def frames():
    seq = si.sequence(2)
    pairs = [si.render_stereo_pair(f["pos"], f["yaw"]) for f in seq]
    return pairs


def _maps(svs, frames):
    """The device map of each frame, and its read-back, from one handle per frame (kept open for the pointers)."""
    out = []
    for left, right, _ in frames:
        sm = svs.StereoMatcher(640, 480, 32, device=0)
        sm.compute(left, right)
        out.append((sm, sm.disparity()))
    return out


def test_dense_tracker_handover(svs, frames):
    cams = fi.level_cams(nlevels=3)
    maps = _maps(svs, frames)
    sm, host = maps[0]
    clouds = []
    for device in (False, True):
        dt = svs.DenseTracker(640, 480, 3)
        for l in range(3):
            dt.set_intrinsics(l, *cams[l][:3])
        if device:
            dt.set_disparity_device(*sm.device_disparity())
        else:
            dt.set_disparity(host)
        dt.compute_point_cloud(I7, cams)
        clouds.append([dt.get_point_cloud(l) for l in range(3)])
        dt.close()
    for a, b in zip(*clouds):
        assert a.tobytes() == b.tobytes()
    assert np.any(clouds[0][0] != 0)


def test_dense_tracker_cpu_variant_handover(svs, frames):
    cams = fi.level_cams(nlevels=3)
    maps = _maps(svs, frames)
    sm, host = maps[0]
    p8 = fi.uint8_pyramid(frames[0][0], 3)
    cur = fi.float_pyramid(frames[1][0], 3)
    clouds = []
    for device in (False, True):
        t = svs.DenseTrackerCpuVariant(640, 480, 3)
        for l in range(3):
            dx, dy = fi.gradients(cur[l])
            t.set_prev_u8(l, p8[l])
            t.set_cur(l, cur[l], dx, dy)
        if device:
            t.set_disparity_device(*sm.device_disparity())
        else:
            t.set_disparity(host)
        t.compute_point_cloud(I7, cams)
        clouds.append([t.point_cloud(l) for l in range(3)])
        t.close()
    for a, b in zip(*clouds):
        assert a.tobytes() == b.tobytes()


def _corners(img):
    fast = cv2.FastFeatureDetector_create(20)
    xy = np.array([k.pt for k in fast.detect(img)], np.float64).reshape(-1, 2)
    return np.ascontiguousarray(np.rint(xy).astype(np.int32))


def test_matcher_handover(svs, frames):
    cams = fi.level_cams(nlevels=3)
    levels = [(640 >> l, 480 >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(3)]
    maps = _maps(svs, frames)
    (sm0, key_disp), (sm1, cur_host) = maps
    kf_pyr = fi.uint8_pyramid(frames[0][0], 3)
    cur_pyr = fi.uint8_pyramid(frames[1][0], 3)
    kxy = _corners(kf_pyr[0])
    d = key_disp[kxy[:, 1], kxy[:, 0]]
    kxy, d = kxy[d > 0], d[d > 0]
    f, px, py, b = cams[0]
    z = f * b / d
    pts = np.zeros(len(kxy), svs.MATCH_POINT_DTYPE)
    pts["keyframe"] = 0
    pts["xyz_anchor"] = np.stack([(kxy[:, 0] - px) / f * z, (kxy[:, 1] - py) / f * z, z], 1)
    pts["anchor_obs_pyr"] = kxy
    T_cur = np.array([0, 0, 0, 1, 0, 0, -0.02])
    out = []
    for device in (False, True):
        m = svs.GuidedMatcher(levels)
        m.set_keyframe(0, I7, kf_pyr)
        m.set_current(cur_pyr)
        if device:
            m.set_current_disparity_device(*sm1.device_disparity())
        else:
            m.set_current_disparity(cur_host)
        for l in range(3):
            c = _corners(cur_pyr[l])
            m.set_features(l, c, np.zeros(len(c), np.int32))
        res = m.match(T_cur, I7, pts, 4, 22, 10)
        fresh = m.add_more_points(1, cams[0], 1)
        out.append((res, fresh))
        m.close()
    (r0, f0), (r1, f1) = out
    assert r0.tobytes() == r1.tobytes()
    assert r0["matched"].sum() > 50
    for a, b in zip(f0, f1):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    assert len(f0[0]) > 50


# ---------------------------------------------------------------- 5. refusals

def test_refusals_keep_the_previous_map(svs):
    L = svs.lib()
    left, right = stress_pair(640, 480)
    sm = svs.StereoMatcher(640, 480, 32, device=0)
    sm.compute(left, right)
    before = sm.disparity()
    other = np.ascontiguousarray(right[:, ::-1])
    lp, rp = left.ctypes.data, other.ctypes.data
    assert L.svs_stereo_compute(sm._h, lp, 640, 1, rp, 640, 0) == SVS_ERR_INVALID      # host memory flagged as device
    assert L.svs_stereo_compute(sm._h, lp, 640, 0, rp, 640, 1) == SVS_ERR_INVALID
    assert L.svs_stereo_compute(sm._h, lp, 639, 0, rp, 640, 0) == SVS_ERR_INVALID      # pitch < w
    assert L.svs_stereo_compute(sm._h, lp, 640, 0, rp, 600, 0) == SVS_ERR_INVALID
    assert sm.disparity().tobytes() == before.tobytes()
    for nd in (0, 8, 40, 176):
        with pytest.raises(svs.SvsError) as e:
            svs.StereoMatcher(640, 480, nd, device=0)
        assert e.value.rc == SVS_ERR_INVALID
    # the consumers refuse host memory passed as a device map and keep theirs
    cams = fi.level_cams(nlevels=3)
    dt = svs.DenseTracker(640, 480, 3)
    for l in range(3):
        dt.set_intrinsics(l, *cams[l][:3])
    dt.set_disparity_device(*sm.device_disparity())
    dt.compute_point_cloud(I7, cams)
    cloud = dt.get_point_cloud(0)
    junk = np.full((480, 640), 7.0, np.float32)
    for call in (lambda: dt.set_disparity_device(junk.ctypes.data, 640),
                 lambda: dt.set_disparity_device(sm.device_disparity()[0], 600)):
        with pytest.raises(svs.SvsError) as e:
            call()
        assert e.value.rc == SVS_ERR_INVALID
    dt.compute_point_cloud(I7, cams)
    assert dt.get_point_cloud(0).tobytes() == cloud.tobytes()
    t = svs.DenseTrackerCpuVariant(640, 480, 3)
    with pytest.raises(svs.SvsError):
        t.set_disparity_device(junk.ctypes.data, 640)
    m = svs.GuidedMatcher([(640, 480) + tuple(cams[0][:3])])
    with pytest.raises(svs.SvsError):
        m.set_current_disparity_device(junk.ctypes.data, 640)
    with pytest.raises(svs.SvsError):
        m.set_current_disparity_device(sm.device_disparity()[0], 320)
    dt.close(); t.close(); m.close(); sm.close()
