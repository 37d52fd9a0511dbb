"""Front-end kernels (FAST, matcher, dense trackers, preprocessing, motion-only LM) against the CPU oracle and OpenCV
at the image shapes where their launches change, and at the reference's own stereo camera.

All front-end kernels choose their launch from the image size.  Every shape case below restates that choice from
the kernel's constants and asserts that it reaches the launch it is named for, so that a change of constants (or a
card with another SM count) cannot silently move a case off its boundary:
  k_dt_track_level (dt.cu)  min(track_blocks, ceil(w h / 256)) CTAs of 256 threads, track_blocks = 2 x SMs; one pixel
                            per thread and step while w h <= 2 stride (stride = CTAs x 256), batches of kPxBatch = 4
                            strides above; the last CTA sums the partials in kSeg = 18 segments of 9 loads, so a
                            second round starts above 9 kSeg = 162 CTAs.
  k_dtc_level (dtc.cu)      one CTA of 512 threads over (w/4)(h/4) points.
  k_fast_select (fast.cu)   (32 / grid_w) grid_w cells per round; k_fast_scan 32 cells per warp round; 64 cells max.

Bars are those of the per-kernel suites: FAST keypoints, per-cell offsets and threshold trajectories bit-exact;
matcher fields bit-exact; point clouds and residual images bit-exact; dense tracker chi2 / J^T J / J^T r to 1e-11,
identical pass counts and the pose to 1e-9; uint8 pyramids bit-exact with OpenCV, float pyramids bit-exact with a
float32 restatement of the kernel's tap order (and within 2e-7 of OpenCV's vectorised order)."""
import cv2
import numpy as np
import pytest

from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth_images as si

pytestmark = pytest.mark.gpu

I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
T_OFF = np.array([0.004, 0.001, -0.018, 0.0002, -0.0036, 0.0001])    # a pose near the rendered motion
T_FAR = np.array([0.03, 0.01, -0.05, 0.002, -0.02, 0.004])          # some pixels leave the frame

# The reference's stereo configuration, data/newcollege.cfg: 512x384, cam.f, cam.px, cam.py, cam.baseline;
# use_n_levels_in_frontent = 3.
NC_W, NC_H, NC_LEVELS = 512, 384, 3
NC_CAM = (389.956085, 254.903519, 201.899490, 0.120005)
# A 1241x376 camera (the width of a KITTI odometry frame): every pyramid level is odd or not a multiple of 16 wide.
ODD_W, ODD_H, ODD_LEVELS = 1241, 376, 3
ODD_CAM = (700.0, 620.5, 188.0, 0.12)

# launch constants restated from the kernels
DT_THREADS, DT_PX_BATCH, DT_SEG, DT_SEG_LOADS = 256, 4, 18, 9
DTC_THREADS, DTC_NTH = 512, 4
FAST_SEL_CELLS, FAST_SCAN_WARPS, FAST_MAX_CELLS = 32, 32, 64
SVS_ERR_INVALID, SVS_ERR_UNSUPPORTED = -1, -3


def _cam_for(w, h):
    return (0.9 * max(w, h), 0.5 * (w - 1), 0.5 * (h - 1), 0.075)


def _seq(n, w, h, cam):
    return si.sequence(n, w=w, h=h, cam=cam)


def _track_blocks():
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count


def dt_launch(w, h, track_blocks):
    """k_dt_track_level's launch for a w x h level (svs_dt_track, accumulate_pass, the last CTA's partial sums)."""
    npx = w * h
    blocks = min(track_blocks, max(1, -(-npx // DT_THREADS)))
    stride = blocks * DT_THREADS
    batched = npx > 2 * stride
    steps = -(-npx // (DT_PX_BATCH * stride)) if batched else -(-npx // stride)   # pixel-loop iterations of thread 0
    red_rounds = -(-blocks // (DT_SEG * DT_SEG_LOADS))
    return dict(npx=npx, blocks=blocks, stride=stride, batched=batched, steps=steps, red_rounds=red_rounds)


def fast_rounds(grid_w, grid_h):
    """(cells per k_fast_select round, k_fast_select rounds, k_fast_scan warp rounds)."""
    n = grid_w * grid_h
    per_round = (FAST_SEL_CELLS // grid_w) * grid_w
    return per_round, -(-n // per_round), -(-n // FAST_SCAN_WARPS)


def _content(off):
    return np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(len(off) - 1)]).astype(np.int32)


# ---------------------------------------------------------------- dense tracker helpers

def _dt_inputs(oracle, seq, cams, w0, h0, nl, i_prev=0, i_cur=1, T_cloud=I7, disp=None):
    """Per level: the full OpenCV pyramid planes (cv2.pyrDown rounds sizes up) and the oracle's level dict on the
    tracker's (h0 >> l, w0 >> l) window of them."""
    prev_p = fi.float_pyramid(seq[i_prev]["img"], nl)
    cur_p = fi.float_pyramid(seq[i_cur]["img"], nl)
    disp = seq[i_prev]["disp"] if disp is None else disp
    full, lv = [], []
    for l in range(nl):
        dx, dy = fi.gradients(cur_p[l])
        full.append((prev_p[l], cur_p[l], dx, dy))
        w, h = w0 >> l, h0 >> l
        crop = [np.ascontiguousarray(a[:h, :w]) for a in full[-1]]
        lv.append(dict(prev=crop[0], cur=crop[1], dx=crop[2], dy=crop[3], f=cams[l][0], px=cams[l][1], py=cams[l][2],
                       cloud=oracle.dt_point_cloud(T_cloud, cams[l], disp, l, w, h)))
    return full, lv, disp


def _dt_handle(svs, full, cams, disp, w0, h0, flags=0):
    dt = svs.DenseTracker(w0, h0, len(full), flags)
    dt.set_disparity(disp)
    for l, planes in enumerate(full):
        dt.set_intrinsics(l, cams[l][0], cams[l][1], cams[l][2])
        dt.set_images(l, *planes)
    dt.compute_point_cloud(I7, cams)
    return dt


def _check_dt_passes(oracle, dt, lv, flags, levels=None, poses=(I7, T_OFF), min_frac=0.3):
    for l in (range(len(lv)) if levels is None else levels):
        for pose in poses:
            T = pose if len(pose) == 7 else oracle.se3_exp(pose)
            chi_o, H_o, b_o, n = oracle.dt_pass(lv[l], T, exact=bool(flags))
            assert n >= min_frac * lv[l]["prev"].size, (l, n)
            chi = dt.chi2(l, T)
            H, b, chi2 = dt.jacobian_reduction(l, T)
            assert abs(chi - chi_o) <= 1e-11 * chi_o and abs(chi2 - chi_o) <= 1e-11 * chi_o, (l, chi, chi_o)
            np.testing.assert_allclose(H, H_o, rtol=1e-11, atol=1e-11 * np.abs(H_o).max())
            np.testing.assert_allclose(b, b_o, rtol=1e-9, atol=1e-11 * np.abs(b_o).max())


def _check_dt_track(oracle, dt, lv, flags, T0=I7):
    T, st = dt.track(T0)
    To, sto = oracle.dt_track(lv, T0, exact=bool(flags))
    assert st["passes"] == sto["passes"], (st["passes"], sto["passes"])
    np.testing.assert_allclose(st["chi2"], sto["chi2"], rtol=1e-9)
    np.testing.assert_allclose(T, To, rtol=0, atol=1e-9)
    return T, st, sto


# ---------------------------------------------------------------- FAST / matcher helpers

def frontend_grid(w, h, level):
    """FastGrid arguments of the front end for pyramid level `level` of a (w, h) level (stereo_frontend.cpp:71-88)."""
    dim = max(3 - int(level * 0.5), 1)
    inv = 0.5 ** level
    total = int(2000 * inv * inv)
    per_cell = total // (dim * dim)
    return (w, h, per_cell, max(per_cell // 3, 10), 25, dim, dim)


def _grid_args(w, h, gw, gh):
    per_cell = 2000 // (gw * gh)
    return (w, h, per_cell, max(per_cell // 3, 10), 25, gw, gh)


def _check_fast_trajectory(svs, oracle, imgs, args):
    """Same keypoints, per-cell ordinals and thresholds as the oracle over a frame sequence (5 trials on the first
    frame, 6 afterwards, as the front end calls detectAdaptively)."""
    w, h = args[0], args[1]
    fg = svs.FastGrid(*args)
    og = oracle.fast_grid(*args)
    thr_seen = set()
    for it, img in enumerate(imgs):
        trials = 5 if it == 0 else 6
        fg.set_image(np.ascontiguousarray(img[:h, :w]))
        xy, off = fg.detect_adaptively(trials)
        xo, oo = oracle.fast_detect_adaptively(img, og, trials)
        np.testing.assert_array_equal(off, oo)
        np.testing.assert_array_equal(xy, xo)
        thr = [c[4] for c in fg.cell_list()]
        assert thr == [og.cells[k].thr for k in range(fg.ncells)]
        thr_seen.update(thr)
    fg.close()
    assert len(thr_seen) > 1   # the walk moved some cell's threshold


def _kf_points(oracle, kf_pyr, disp, cams, sizes, keyframe=0):
    """Map points anchored on every level: the FAST corners of the keyframe's level l with their disparity."""
    pts = []
    for l, (w, h) in enumerate(sizes):
        g = oracle.fast_grid(*frontend_grid(w, h, l))
        kxy, _ = oracle.fast_detect_adaptively(kf_pyr[l], g, 5)
        d = disp[kxy[:, 1] << l, kxy[:, 0] << l] / (1 << l)
        ok = d > 0
        kxy, d = kxy[ok], d[ok]
        z = cams[l][0] * cams[l][3] / d
        p = np.zeros(len(kxy), oracle.MATCH_POINT_DTYPE)
        p["keyframe"] = keyframe
        p["anchor_level"] = l
        p["xyz_anchor"] = np.stack([(kxy[:, 0] - cams[l][1]) / cams[l][0] * z, (kxy[:, 1] - cams[l][2]) / cams[l][0] * z,
                                    z], 1)
        p["anchor_obs_pyr"] = kxy
        pts.append(p)
    return np.concatenate(pts)


def _cur_features(svs, pyr, sizes):
    feats = []
    for l, (w, h) in enumerate(sizes):
        g = svs.FastGrid(*frontend_grid(w, h, l))
        g.set_image(np.ascontiguousarray(pyr[l][:h, :w]))
        xy, off = g.detect_adaptively(5)
        g.close()
        feats.append((xy, _content(off)))
    return feats


def _assert_same_match(res, ref):
    for f in ("predicted", "textured", "matched", "n_candidates", "index", "min_dist", "uv_pyr", "obs", "xyz_actkey"):
        np.testing.assert_array_equal(res[f], ref[f], err_msg=f)


def _check_matcher(svs, oracle, seq, cams, w0, h0, nl, radii=(4, 10)):
    sizes = [(w0 >> l, h0 >> l) for l in range(nl)]
    levels = [(w, h, cams[l][0], cams[l][1], cams[l][2]) for l, (w, h) in enumerate(sizes)]
    kf_pyr = fi.uint8_pyramid(seq[0]["img"], nl)
    pts = _kf_points(oracle, kf_pyr, seq[0]["disp"], cams, sizes)
    assert all((pts["anchor_level"] == l).sum() > 20 for l in range(nl))
    T_key_w = oracle.se3_exp(np.array([0.3, -0.1, 0.2, 0.01, 0.02, -0.01]))
    for i_cur in range(1, len(seq)):
        cur_pyr = fi.uint8_pyramid(seq[i_cur]["img"], nl)
        feats = _cur_features(svs, cur_pyr, sizes)
        trees = [oracle.QuadTree(w, h, *feats[l]) for l, (w, h) in enumerate(sizes)]
        T_cur = oracle.se3_exp(np.array([0.001, 0.0, -0.02 * i_cur, 0.0, -0.0035 * i_cur, 0.0]))
        m = svs.GuidedMatcher(levels)
        m.set_keyframe(0, T_key_w, kf_pyr)
        m.set_current(cur_pyr, seq[i_cur]["disp"])
        for l in range(nl):
            m.set_features(l, *feats[l])
        for radius in radii:
            res = m.match(T_cur, T_key_w, pts, radius, 22, 10)
            ref = oracle.match(levels, cur_pyr, seq[i_cur]["disp"], trees, [(T_key_w, kf_pyr)], T_cur, T_key_w, pts,
                               radius, 22, 10)
            for l in range(nl):   # matches on every level
                assert ref["matched"][pts["anchor_level"] == l].sum() > 5, (l, radius)
            assert ref["matched"].sum() > 0.3 * len(pts)
            _assert_same_match(res, ref)
        m.close()


# ---------------------------------------------------------------- 1. the reference's camera, end to end

@pytest.fixture(scope="module")
def nc_seq():
    return _seq(3, NC_W, NC_H, NC_CAM)


@pytest.fixture(scope="module")
def nc_cams():
    return fi.level_cams(*NC_CAM, nlevels=NC_LEVELS)


def _reflect101(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def pyrdown_f32(src):
    """5-tap pyrDown in float32, taps summed in the order of OpenCV's scalar loop (c 6 + (l + r) 4 + ll + rr, rows,
    then columns), each operation rounded to float32: what k_pyrdown_f32 computes."""
    h, w = src.shape
    xs, ys = 2 * np.arange((w + 1) // 2), 2 * np.arange((h + 1) // 2)
    c = [src[:, _reflect101(xs - 2 + k, w)] for k in range(5)]
    rows = c[2] * np.float32(6) + (c[1] + c[3]) * np.float32(4) + c[0] + c[4]
    r = [rows[_reflect101(ys - 2 + k, h)] for k in range(5)]
    return (r[2] * np.float32(6) + (r[1] + r[3]) * np.float32(4) + r[0] + r[4]) * np.float32(1.0 / 256.0)


def _check_prep(svs, img, nl):
    """uint8 levels bit-exact with cv2.pyrDown; float levels bit-exact with the float32 restatement of the kernel's
    tap order, and within 2e-7 of cv2.pyrDown (the bar of tests/test_prep_gpu.py), whose vectorised loop sums the
    taps in another order: about half the values differ from the scalar order, by a few ulp."""
    h, w = img.shape
    pp = svs.FramePreprocessor(w, h, nl)
    pp.process(img)
    u8, f32 = img, img.astype(np.float32) * np.float32(1.0 / 255.0)
    mine = f32
    for l in range(nl):
        if l > 0:
            u8, f32, mine = cv2.pyrDown(u8), cv2.pyrDown(f32), pyrdown_f32(mine)
        assert (pp.level(l)["w"], pp.level(l)["h"]) == (u8.shape[1], u8.shape[0])
        np.testing.assert_array_equal(pp.get_u8(l), u8)
        np.testing.assert_array_equal(pp.get_f32(l, 0), mine)
        np.testing.assert_allclose(pp.get_f32(l, 0), f32, rtol=0, atol=2e-7)
        mine = pp.get_f32(l, 0)
        dx, dy = fi.gradients(mine)
        np.testing.assert_array_equal(pp.get_f32(l, 1), dx)
        np.testing.assert_array_equal(pp.get_f32(l, 2), dy)
    pp.close()


def test_newcollege_preprocessing_matches_opencv(svs, nc_seq):
    _check_prep(svs, nc_seq[1]["img"], NC_LEVELS)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_newcollege_fast_frontend_grids(svs, oracle, nc_seq, level):
    """The front end's own grids (3x3, 3x3, 2x2) on levels 0-2, threshold trajectory over a sequence."""
    imgs = [fi.uint8_pyramid(f["img"], NC_LEVELS)[level] for f in nc_seq + nc_seq[::-1]]
    args = frontend_grid(NC_W >> level, NC_H >> level, level)
    assert args[5] == (2 if level == 2 else 3)
    _check_fast_trajectory(svs, oracle, imgs, args)


def test_newcollege_matcher_three_levels(svs, oracle, nc_seq, nc_cams):
    _check_matcher(svs, oracle, nc_seq, nc_cams, NC_W, NC_H, NC_LEVELS)


@pytest.mark.parametrize("flags", [0, 1])
def test_newcollege_dense_tracker(svs, oracle, nc_seq, nc_cams, flags):
    full, lv, disp = _dt_inputs(oracle, nc_seq, nc_cams, NC_W, NC_H, NC_LEVELS)
    dt = _dt_handle(svs, full, nc_cams, disp, NC_W, NC_H, flags)
    for l in range(NC_LEVELS):
        np.testing.assert_array_equal(dt.get_point_cloud(l), lv[l]["cloud"])
    _check_dt_passes(oracle, dt, lv, flags)
    for l in range(NC_LEVELS):
        for pose in (I7, oracle.se3_exp(T_FAR)):
            np.testing.assert_array_equal(dt.residual_image(l, pose), oracle.dt_residual_image(lv[l], pose, exact=bool(flags)))
    T, st, _ = _check_dt_track(oracle, dt, lv, flags)
    assert abs(T[6] + 0.02) < 0.01    # 2 cm forward between the frames
    dt.close()


def _dtc_check(svs, oracle, seq, cams, w0, h0, nl):
    p8 = fi.uint8_pyramid(seq[0]["img"], nl)
    cur = fi.float_pyramid(seq[1]["img"], nl)
    t = svs.DenseTrackerCpuVariant(w0, h0, nl)
    t.set_disparity(seq[0]["disp"])
    lv = []
    for l in range(nl):
        dx, dy = fi.gradients(cur[l])
        h, w = cur[l].shape
        assert (w, h) == (w0 >> l, h0 >> l)
        lv.append(dict(prev_u8=p8[l], cur=cur[l], dx=dx, dy=dy, cam=cams[l],
                       cloud=oracle.dtc_point_cloud(I7, cams[l], seq[0]["disp"], l, w, h)))
        t.set_prev_u8(l, p8[l])
        t.set_cur(l, cur[l], dx, dy)
    t.compute_point_cloud(I7, cams)
    for l in range(nl):
        np.testing.assert_array_equal(t.point_cloud(l), lv[l]["cloud"])
    T_g, sg = t.track(I7, cams)
    T_o, so = oracle.dtc_track(lv, I7)
    t.close()
    assert sg["passes"] == so["passes"]
    np.testing.assert_allclose(sg["chi2"], so["chi2"], rtol=1e-9)
    np.testing.assert_allclose(T_g, T_o, rtol=1e-9, atol=1e-11)
    return T_g, sg, lv


def test_newcollege_dense_tracker_cpu_variant(svs, oracle, nc_seq, nc_cams):
    T, st, _ = _dtc_check(svs, oracle, nc_seq, nc_cams, NC_W, NC_H, NC_LEVELS)
    assert abs(T[6] + 0.02) < 0.01


def _matched_pose(svs, oracle, m, res, cam):
    ok = res["matched"] == 1
    assert ok.sum() >= 20                     # the front end gives up below 20 (stereo_frontend.cpp:1053)
    po = svs.PoseOptimizer()
    T_dev, sd = po.calc_fast_motion_only_matched(m, cam, I7, True, 2.0, 15)
    obs, xyz = np.ascontiguousarray(res["obs"][ok]), np.ascontiguousarray(res["xyz_actkey"][ok])
    T_host, sh = po.calc_fast_motion_only(np.arange(ok.sum()), obs, xyz, cam, I7, True, 2.0, 15)
    T_o, so = oracle.calc_fast_motion_only(np.arange(ok.sum()), obs, xyz, np.array(cam), I7, True, 2.0, 15)
    po.close()
    assert sd["num_obs"] == int(ok.sum()) == sh["num_obs"] == so["num_obs"]
    np.testing.assert_allclose(T_dev, T_host, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(T_dev, T_o, rtol=1e-6, atol=1e-9)
    return T_dev


def test_newcollege_motion_only_on_the_matches(svs, oracle, nc_seq, nc_cams):
    sizes = [(NC_W >> l, NC_H >> l) for l in range(NC_LEVELS)]
    levels = [(w, h, nc_cams[l][0], nc_cams[l][1], nc_cams[l][2]) for l, (w, h) in enumerate(sizes)]
    kf_pyr = fi.uint8_pyramid(nc_seq[0]["img"], NC_LEVELS)
    cur_pyr = fi.uint8_pyramid(nc_seq[1]["img"], NC_LEVELS)
    pts = _kf_points(oracle, kf_pyr, nc_seq[0]["disp"], nc_cams, sizes)
    m = svs.GuidedMatcher(levels)
    m.set_keyframe(0, I7, kf_pyr)
    m.set_current(cur_pyr, nc_seq[1]["disp"])
    for l, f in enumerate(_cur_features(svs, cur_pyr, sizes)):
        m.set_features(l, *f)
    res = m.match(I7, I7, pts, 4, 22, 10)
    T = _matched_pose(svs, oracle, m, res, nc_cams[0])
    assert -0.03 < T[6] < 0                   # forward, as rendered (t_z = -0.02; integer corners, f = 390)
    m.close()


def _device_chain(svs, seq, cams, w0, h0, nl, on_device):
    """prep -> dense tracker, FAST on every level -> matcher -> motion-only LM, with the planes handed over by device
    pointer (on_device) or copied to the host from the same preprocessors."""
    sizes = [(w0 >> l, h0 >> l) for l in range(nl)]
    pa, pb = svs.FramePreprocessor(w0, h0, nl), svs.FramePreprocessor(w0, h0, nl)
    pa.process(seq[0]["img"])
    pb.process(seq[1]["img"])
    dt = svs.DenseTracker(w0, h0, nl)
    dt.set_disparity(seq[0]["disp"])
    for l in range(nl):
        dt.set_intrinsics(l, cams[l][0], cams[l][1], cams[l][2])
        if on_device:
            la, lb = pa.level(l), pb.level(l)
            dt.set_images_device(l, la["f32"], lb["f32"], lb["dx"], lb["dy"], lb["stride_f32"])
        else:
            dt.set_images(l, pa.get_f32(l, 0), pb.get_f32(l, 0), pb.get_f32(l, 1), pb.get_f32(l, 2))
    dt.compute_point_cloud(I7, cams)
    T_dt, st_dt = dt.track(I7)
    levels = [(w, h, cams[l][0], cams[l][1], cams[l][2]) for l, (w, h) in enumerate(sizes)]
    m = svs.GuidedMatcher(levels)
    if on_device:
        m.set_pyramid_device(0, [pa.level(l)["u8"] for l in range(nl)], [pa.level(l)["pitch_u8"] for l in range(nl)], I7)
        m.set_pyramid_device(-1, [pb.level(l)["u8"] for l in range(nl)], [pb.level(l)["pitch_u8"] for l in range(nl)])
        m.set_current_disparity(seq[1]["disp"])
    else:
        m.set_keyframe(0, I7, [pa.get_u8(l) for l in range(nl)])
        m.set_current([pb.get_u8(l) for l in range(nl)], seq[1]["disp"])
    fast = []
    for l, (w, h) in enumerate(sizes):
        g = svs.FastGrid(*frontend_grid(w, h, l))
        if on_device:
            lb = pb.level(l)
            g.set_image_device(lb["u8"], lb["pitch_u8"], w, h)
        else:
            g.set_image(pb.get_u8(l)[:h, :w])
        xy, off = g.detect_adaptively(5)
        fast.append((xy, off))
        if on_device:
            m.set_features_from_fast(l, g)
        else:
            m.set_features(l, xy, _content(off))
        g.close()
    return dict(dt=(T_dt, st_dt), fast=fast, m=m, handles=(pa, pb, dt))


def _check_device_chain(svs, oracle, seq, cams, w0, h0, nl):
    sizes = [(w0 >> l, h0 >> l) for l in range(nl)]
    pts = _kf_points(oracle, fi.uint8_pyramid(seq[0]["img"], nl), seq[0]["disp"], cams, sizes)
    out = []
    for on_device in (False, True):
        r = _device_chain(svs, seq, cams, w0, h0, nl, on_device)
        r["res"] = r["m"].match(I7, I7, pts, 4, 22, 10)
        po = svs.PoseOptimizer()
        r["pose"] = po.calc_fast_motion_only_matched(r["m"], cams[0], I7, True, 2.0, 15)
        po.close()
        r["m"].close()
        for h in r["handles"]:
            h.close()
        out.append(r)
    host, dev = out
    assert dev["dt"][1]["passes"] == host["dt"][1]["passes"] and np.array_equal(dev["dt"][0], host["dt"][0])
    for (xd, od), (xh, oh) in zip(dev["fast"], host["fast"]):
        np.testing.assert_array_equal(od, oh)
        np.testing.assert_array_equal(xd, xh)
    assert host["res"]["matched"].sum() >= 20
    _assert_same_match(dev["res"], host["res"])
    assert np.array_equal(dev["pose"][0], host["pose"][0])
    assert abs(host["dt"][0][6] + 0.02) < 0.01
    return host


def test_newcollege_chain_handed_over_on_the_device(svs, oracle, nc_seq, nc_cams):
    _check_device_chain(svs, oracle, nc_seq, nc_cams, NC_W, NC_H, NC_LEVELS)


# ---------------------------------------------------------------- 2. odd widths

@pytest.fixture(scope="module")
def odd_seq():
    return _seq(3, ODD_W, ODD_H, ODD_CAM)


@pytest.fixture(scope="module")
def odd_cams():
    return fi.level_cams(*ODD_CAM, nlevels=ODD_LEVELS)


def test_odd_width_level_sizes():
    """The tracker's level is w0 >> l (as the reference's pyrFromZero_d); the pyramid rounds up: they differ here."""
    assert [ODD_W >> l for l in range(3)] == [1241, 620, 310]
    assert [(ODD_W + (1 << l) - 1) >> l for l in range(3)] == [1241, 621, 311]
    assert all((ODD_W >> l) % 16 for l in range(3))


def test_odd_width_preprocessing_matches_opencv(svs, odd_seq):
    _check_prep(svs, odd_seq[0]["img"], ODD_LEVELS)


def test_odd_width_tracker_host_device_and_oracle_agree(svs, oracle, odd_seq, odd_cams):
    """The tracker fed by host arrays of the rounded-up pyramid, by device hand-over from the preprocessor, and the
    oracle on the (h0 >> l, w0 >> l) windows of the same planes: all three agree."""
    nl = ODD_LEVELS
    pa, pb = svs.FramePreprocessor(ODD_W, ODD_H, nl), svs.FramePreprocessor(ODD_W, ODD_H, nl)
    pa.process(odd_seq[0]["img"])
    pb.process(odd_seq[1]["img"])
    disp = odd_seq[0]["disp"]
    full = [(pa.get_f32(l, 0), pb.get_f32(l, 0), pb.get_f32(l, 1), pb.get_f32(l, 2)) for l in range(nl)]
    assert [p[0].shape[1] for p in full] == [1241, 621, 311]
    lv = []
    for l in range(nl):
        w, h = ODD_W >> l, ODD_H >> l
        crop = [np.ascontiguousarray(a[:h, :w]) for a in full[l]]
        lv.append(dict(prev=crop[0], cur=crop[1], dx=crop[2], dy=crop[3], f=odd_cams[l][0], px=odd_cams[l][1],
                       py=odd_cams[l][2], cloud=oracle.dt_point_cloud(I7, odd_cams[l], disp, l, w, h)))
    dt_host = _dt_handle(svs, full, odd_cams, disp, ODD_W, ODD_H)
    dt_dev = svs.DenseTracker(ODD_W, ODD_H, nl)
    dt_dev.set_disparity(disp)
    for l in range(nl):
        la, lb = pa.level(l), pb.level(l)
        dt_dev.set_intrinsics(l, *odd_cams[l][:3])
        dt_dev.set_images_device(l, la["f32"], lb["f32"], lb["dx"], lb["dy"], lb["stride_f32"])
    dt_dev.compute_point_cloud(I7, odd_cams)
    for dt in (dt_host, dt_dev):
        _check_dt_passes(oracle, dt, lv, 0)
        for l in range(nl):
            np.testing.assert_array_equal(dt.get_point_cloud(l), lv[l]["cloud"])
            np.testing.assert_array_equal(dt.residual_image(l, oracle.se3_exp(T_OFF)),
                                          oracle.dt_residual_image(lv[l], oracle.se3_exp(T_OFF)))
    T_h, st_h, _ = _check_dt_track(oracle, dt_host, lv, 0)
    T_d, st_d, _ = _check_dt_track(oracle, dt_dev, lv, 0)
    assert st_h["passes"] == st_d["passes"] and np.array_equal(T_h, T_d)
    assert abs(T_h[6] + 0.02) < 0.01
    for h in (pa, pb, dt_host, dt_dev):
        h.close()


def test_odd_width_tracker_rejects_a_narrow_image(svs):
    dt = svs.DenseTracker(ODD_W, ODD_H, 2)
    ok = np.zeros((ODD_H >> 1, 620), np.float32)
    dt.set_images(1, ok, ok, ok, ok)
    for bad in (np.zeros((ODD_H >> 1, 619), np.float32), np.zeros(((ODD_H >> 1) - 1, 621), np.float32)):
        with pytest.raises(svs.SvsError) as e:
            dt.set_images(1, cur=bad)
        assert e.value.rc == SVS_ERR_INVALID
    dt.close()


@pytest.mark.parametrize("level", [0, 1, 2])
def test_odd_width_fast_frontend_grids(svs, oracle, odd_seq, level):
    """Grid of the front end on the camera's (w0 >> l, h0 >> l) level, on the wider rounded-up pyramid level."""
    imgs = [fi.uint8_pyramid(f["img"], ODD_LEVELS)[level] for f in odd_seq + odd_seq[::-1]]
    _check_fast_trajectory(svs, oracle, imgs, frontend_grid(ODD_W >> level, ODD_H >> level, level))


def test_odd_width_matcher_three_levels(svs, oracle, odd_seq, odd_cams):
    _check_matcher(svs, oracle, odd_seq, odd_cams, ODD_W, ODD_H, ODD_LEVELS)


def test_odd_width_chain_handed_over_on_the_device(svs, oracle, odd_seq, odd_cams):
    _check_device_chain(svs, oracle, odd_seq, odd_cams, ODD_W, ODD_H, ODD_LEVELS)


# ---------------------------------------------------------------- 3. k_dt_track_level / k_dt_pass launch sweep

def _sweep_shapes(T):
    """name -> (w, h, check of dt_launch(w, h, T)).  64 columns: a 256-pixel run of a CTA is four image rows, so the
    run that ends an image still has rows inside the window the tracker samples (1 <= v <= h - 2), and "one more" is
    one more run (4 rows)."""
    return {
        "1cta": (16, 16, lambda d: d["blocks"] == 1),
        "162cta": (64, 648, lambda d: d["blocks"] == 162 and d["red_rounds"] == 1),
        "163cta": (64, 652, lambda d: d["blocks"] == 163 and d["red_rounds"] == 2),
        "track_blocks": (64, 4 * T, lambda d: d["blocks"] == T and d["npx"] == d["stride"] and d["steps"] == 1),
        "track_blocks_plus_run": (64, 4 * T + 4, lambda d: -(-d["npx"] // DT_THREADS) == T + 1 and d["blocks"] == T
                                  and not d["batched"] and d["steps"] == 2),
        "2stride": (64, 8 * T, lambda d: d["blocks"] == T and d["npx"] == 2 * d["stride"] and not d["batched"]),
        "2stride_plus_run": (64, 8 * T + 4, lambda d: d["batched"] and d["npx"] == 2 * d["stride"] + DT_THREADS
                             and d["steps"] == 1),
        "over_4stride": (64, 16 * T + 8, lambda d: d["batched"] and d["npx"] > 4 * d["stride"] and d["steps"] == 2),
    }


@pytest.mark.parametrize("name", ["1cta", "162cta", "163cta", "track_blocks", "track_blocks_plus_run", "2stride",
                                  "2stride_plus_run", "over_4stride"])
def test_dt_launch_sweep(svs, oracle, name):
    T = _track_blocks()
    w, h, reaches = _sweep_shapes(T)[name]
    if name in ("162cta", "163cta") and T < 163:
        pytest.skip(f"track_blocks = {T}: the tracker never runs 163 CTAs on this card")
    d = dt_launch(w, h, T)
    assert reaches(d), (name, d)
    cam = _cam_for(w, h)
    seq = _seq(2, w, h, cam)
    cams = fi.level_cams(*cam, nlevels=1)
    full, lv, disp = _dt_inputs(oracle, seq, cams, w, h, 1)
    # pixel idx is taken by CTA (idx mod stride) / 256 in its step idx / stride (one or kPxBatch steps per loop
    # iteration): every (CTA, step) has a pixel that contributes at the start pose, so a partial sum left out of the
    # final reduction, or a step or batch tail left out of the pixel loop, changes chi2
    res = oracle.dt_residual_image(lv[0], I7)
    contributes = (res[..., 0] == res[..., 1]).ravel()
    idx = np.arange(d["npx"])
    group = (idx // d["stride"]) * d["blocks"] + (idx % d["stride"]) // DT_THREADS
    assert set(group[contributes]) == set(group)
    for flags in (0, 1):
        dt = _dt_handle(svs, full, cams, disp, w, h, flags)
        np.testing.assert_array_equal(dt.get_point_cloud(0), lv[0]["cloud"])
        _check_dt_passes(oracle, dt, lv, flags, poses=(I7, T_OFF, T_FAR), min_frac=0.02)
        np.testing.assert_array_equal(dt.residual_image(0, oracle.se3_exp(T_FAR)),
                                      oracle.dt_residual_image(lv[0], oracle.se3_exp(T_FAR), exact=bool(flags)))
        _check_dt_track(oracle, dt, lv, flags)
        _check_dt_track(oracle, dt, lv, flags, T0=oracle.se3_exp(-0.5 * T_OFF))
        dt.close()


def test_dt_five_levels_640x480(svs, oracle):
    T = _track_blocks()
    d = [dt_launch(640 >> l, 480 >> l, T) for l in range(5)]
    assert d[0]["batched"] and d[0]["npx"] > 4 * d[0]["stride"] and d[4]["blocks"] == 5 and d[3]["blocks"] == 19
    seq = si.sequence(2)
    cams = fi.level_cams(nlevels=5)
    full, lv, disp = _dt_inputs(oracle, seq, cams, 640, 480, 5)
    dt = _dt_handle(svs, full, cams, disp, 640, 480)
    for l in range(5):
        np.testing.assert_array_equal(dt.get_point_cloud(l), lv[l]["cloud"])
    _check_dt_passes(oracle, dt, lv, 0, levels=(3, 4), poses=(I7, T_OFF), min_frac=0.1)
    T7, st, _ = _check_dt_track(oracle, dt, lv, 0)
    assert abs(T7[6] + 0.02) < 0.01
    dt.close()


def test_dt_eight_levels_1024x768(svs, oracle):
    """SVS_DT_MAX_LEVELS levels: the deepest (8x6) has a handful of pixels and may contribute none; a level without a
    contributing pixel leaves the pose as it found it, in the oracle and on the device."""
    w0, h0, nl = 1024, 768, 8
    cam = _cam_for(w0, h0)
    cams = fi.level_cams(*cam, nlevels=nl)
    seq = _seq(2, w0, h0, cam)
    full, lv, disp = _dt_inputs(oracle, seq, cams, w0, h0, nl)
    assert lv[7]["prev"].shape == (6, 8) and dt_launch(8, 6, _track_blocks())["blocks"] == 1
    dt = _dt_handle(svs, full, cams, disp, w0, h0)
    for l in range(nl):
        np.testing.assert_array_equal(dt.get_point_cloud(l), lv[l]["cloud"])
    T_track, st, sto = _check_dt_track(oracle, dt, lv, 0)
    assert abs(T_track[6] + 0.02) < 0.01
    T0 = oracle.se3_exp(np.array([0.01, -0.002, 0.004, 0.0005, 0.001, -0.0003]))
    for l in range(nl):
        _, _, _, n = oracle.dt_pass(lv[l], T0)
        chi, (H, b, chi2) = dt.chi2(l, T0), dt.jacobian_reduction(l, T0)
        if n == 0:
            assert chi == chi2 == 0.0 and not H.any() and not b.any()
    # the deepest level on its own, once with its own cloud and once with no depth at all
    empty = dict(lv[7], cloud=np.where(np.arange(4) == 3, -1.0, 0.0).astype(np.float32) * np.ones((6, 8, 1), np.float32))
    for level in (lv[7], empty):
        one = svs.DenseTracker(8, 6, 1)
        one.set_intrinsics(0, level["f"], level["px"], level["py"])
        one.set_images(0, level["prev"], level["cur"], level["dx"], level["dy"])
        one.set_point_cloud(0, level["cloud"])
        T1, st1 = one.track(T0)
        To1, sto1 = oracle.dt_track([level], T0)
        assert st1["passes"] == sto1["passes"]
        np.testing.assert_allclose(T1, To1, rtol=0, atol=1e-9)
        if oracle.dt_pass(level, T0)[3] == 0:
            assert np.array_equal(T1, T0) and np.array_equal(To1, T0) and st1["passes"] == [3] and st1["chi2"] == [0.0]
        one.close()
    assert oracle.dt_pass(empty, T0)[3] == 0
    dt.close()


# ---------------------------------------------------------------- 4. k_dtc_level below 512 points

def test_dtc_below_512_points(svs, oracle):
    w0, h0, nl = 1024, 768, 5
    pts = [((w0 >> l) // DTC_NTH) * ((h0 >> l) // DTC_NTH) for l in range(nl)]
    assert pts[4] == 192 < DTC_THREADS and pts[3] == 768 > DTC_THREADS
    cam = _cam_for(w0, h0)
    T, st, lv = _dtc_check(svs, oracle, _seq(2, w0, h0, cam), fi.level_cams(*cam, nlevels=nl), w0, h0, nl)
    assert oracle.dtc_pass(lv[4], I7)[3] > 0 and abs(T[6] + 0.02) < 0.01


# ---------------------------------------------------------------- 5. FAST grids beyond one round

GRIDS = {(6, 6): (30, 2), (7, 7): (28, 2), (8, 8): (32, 2), (8, 4): (32, 1), (4, 8): (32, 1), (32, 2): (32, 2)}


@pytest.mark.parametrize("shape", ["nc", "odd"])
@pytest.mark.parametrize("grid", list(GRIDS), ids=[f"{a}x{b}" for a, b in GRIDS])
def test_fast_grids_beyond_one_round(svs, oracle, nc_seq, odd_seq, shape, grid):
    gw, gh = grid
    per_round, rounds, scan_rounds = fast_rounds(gw, gh)
    assert (per_round, rounds) == GRIDS[grid] and gw * gh <= FAST_MAX_CELLS
    assert scan_rounds == -(-gw * gh // 32)
    if grid == (32, 2):
        assert per_round == gw            # one grid row per round
    seq = nc_seq if shape == "nc" else odd_seq
    imgs = [f["img"] for f in seq + seq[::-1]]
    h, w = imgs[0].shape
    args = _grid_args(w, h, gw, gh)
    cw, ch = w // gw, h // gh
    if shape == "odd" or grid in ((7, 7), (6, 6)):
        assert cw % 32 or ch % 8          # cells that are not whole 32x8 score tiles
    _check_fast_trajectory(svs, oracle, imgs, args)


def test_fast_grid_limits_raise(svs, nc_seq):
    img = nc_seq[0]["img"]
    fg = svs.FastGrid(*_grid_args(NC_W, NC_H, 33, 1))          # 33 cells: k_fast_select walks at most 32 per row
    fg.set_image(img)
    with pytest.raises(svs.SvsError) as e:
        fg.detect_adaptively(5)
    assert e.value.rc == SVS_ERR_UNSUPPORTED
    fg.detect(fg.cell_list())                                 # static thresholds take any grid of <= 64 cells
    fg.close()
    with pytest.raises(svs.SvsError) as e:                    # 65 cells
        svs.FastGrid(*_grid_args(NC_W, NC_H, 13, 5))
    assert e.value.rc == SVS_ERR_INVALID
    fg = svs.FastGrid(*_grid_args(NC_W, NC_H, 8, 8))
    fg.set_image(img)
    cells = [(0, 64, 0, 64, 20)] * (FAST_MAX_CELLS + 1)
    with pytest.raises(svs.SvsError) as e:
        fg.detect(cells)
    assert e.value.rc == SVS_ERR_INVALID
    fg.close()
