"""CPU checks behind tests/test_frontend_shapes_gpu.py: the renderer's default images are unchanged by its camera
argument, and the oracles it compares against behave at the reference's own stereo camera (data/newcollege.cfg,
512x384): dense tracking recovers the rendered motion, and the FAST oracle equals OpenCV on a full-image cell."""
import hashlib

import numpy as np

from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth
from scavislam_b200 import synth_images as si

I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])
NC_W, NC_H = 512, 384
NC_CAM = (389.956085, 254.903519, 201.899490, 0.120005)   # data/newcollege.cfg: cam.f, cam.px, cam.py, cam.baseline


def test_default_sequence_is_unchanged():
    """sequence(2) with the default camera, as the existing fixtures and the benchmark render it (hash taken before the
    renderer took a camera argument)."""
    h = hashlib.sha256()
    for f in si.sequence(2):
        h.update(f["img"].tobytes())
        h.update(f["disp"].tobytes())
    assert h.hexdigest() == "5ae23b51f6acead9148e0a33e0e40c45ad13a1816e83a3371051ede8edf397c7"
    img, disp = si.render_frame(np.zeros(3), 0.0)
    img2, disp2 = si.render_frame(np.zeros(3), 0.0, cam=(synth.CAM_F, synth.CAM_PX, synth.CAM_PY, synth.CAM_B))
    assert np.array_equal(img, img2) and np.array_equal(disp, disp2)


def test_renderer_takes_the_camera():
    img, disp = si.render_frame(np.zeros(3), 0.0, w=NC_W, h=NC_H, cam=NC_CAM)
    assert img.shape == disp.shape == (NC_H, NC_W) and img.dtype == np.uint8 and disp.dtype == np.float32
    # disparity is f b / depth: the baseline enters linearly
    _, disp2 = si.render_frame(np.zeros(3), 0.0, w=NC_W, h=NC_H, cam=NC_CAM[:3] + (2 * NC_CAM[3],))
    ok = disp > 0
    assert ok.mean() > 0.99
    np.testing.assert_allclose(disp2[ok], 2 * disp[ok], rtol=1e-6)


def test_oracle_tracking_recovers_the_rendered_motion_at_newcollege(oracle):
    seq = si.sequence(2, w=NC_W, h=NC_H, cam=NC_CAM)
    cams = fi.level_cams(*NC_CAM, nlevels=3)
    prev, cur = fi.float_pyramid(seq[0]["img"], 3), fi.float_pyramid(seq[1]["img"], 3)
    levels = []
    for l in range(3):
        dx, dy = fi.gradients(cur[l])
        h, w = prev[l].shape
        assert (w, h) == (NC_W >> l, NC_H >> l)
        levels.append(dict(prev=prev[l], cur=cur[l], dx=dx, dy=dy, f=cams[l][0], px=cams[l][1], py=cams[l][2],
                           cloud=oracle.dt_point_cloud(I7, cams[l], seq[0]["disp"], l, w, h)))
    chi0 = oracle.dt_pass(levels[0], I7)[0]
    T, st = oracle.dt_track(levels, I7)
    assert st["chi2"][0] < 0.5 * chi0
    # 2 cm forward, 0.2 deg of yaw between the frames (synth_images.sequence)
    assert abs(T[6] + 0.02) < 0.005 and abs(abs(T[1]) - np.sin(np.deg2rad(0.1))) < 5e-4
    assert all(2 <= p <= 17 for p in st["passes"])


def test_fast_oracle_equals_opencv_on_a_full_image_cell(oracle):
    import cv2
    img = si.render_frame(np.zeros(3), 0.0, w=NC_W, h=NC_H, cam=NC_CAM)[0]
    for thr in (12, 25):
        xy, off = oracle.fast_detect(img, [(0, NC_W, 0, NC_H, thr)])
        det = cv2.FastFeatureDetector_create(thr, False, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
        ref = np.array([[int(k.pt[0]), int(k.pt[1])] for k in det.detect(img)], np.int32).reshape(-1, 2)
        assert len(ref) > 500 and off.tolist() == [0, len(ref)]
        np.testing.assert_array_equal(xy, ref)
