"""CPU checks of the stereo disparity module: the svs_stereo handle keeps the handle contract without a GPU (null
handle, SVS_ERR_NOGPU with *out left null, SvsError from the wrapper), render_stereo_pair is deterministic, the new
noise_seed argument leaves render_frame's output as it was, and OpenCV's StereoBM with the reference's settings finds
the renderer's ground-truth disparity on a rendered pair (a check of the right camera)."""
import ctypes as C
import hashlib

import cv2
import numpy as np
import pytest

from scavislam_b200 import synth_images as si

SVS_ERR_INVALID = -1
SVS_ERR_NOGPU = -5


def _fn(L, name, restype, *argtypes):
    return C.CFUNCTYPE(restype, *argtypes)(C.cast(getattr(L, name), C.c_void_p).value)


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")


def _create(L, *args):
    out = C.c_void_p(0x1234)
    rc = _fn(L, "svs_stereo_create", C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p)(*args, C.addressof(out))
    return rc, out


def test_null_handle(svs):
    L = svs.lib()
    assert _fn(L, "svs_stereo_last_error", C.c_char_p, C.c_void_p)(None) == b"null handle"
    _fn(L, "svs_stereo_destroy", None, C.c_void_p)(None)
    compute = _fn(L, "svs_stereo_compute", C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int)
    assert compute(None, None, 0, 0, None, 0, 0) == SVS_ERR_INVALID


@pytest.mark.parametrize("ndisp", [0, 8, 24, 170, 176])
def test_create_refuses_bad_num_disparities(svs, ndisp):
    rc, out = _create(svs.lib(), -1, 640, 480, ndisp)
    assert rc == SVS_ERR_INVALID and not out.value


@pytest.mark.parametrize("w,h", [(0, 480), (640, 0), (65536, 480), (640, 65536), (65535, 40000)])
def test_create_refuses_bad_sizes(svs, w, h):
    rc, out = _create(svs.lib(), -1, w, h, 32)
    assert rc == SVS_ERR_INVALID and not out.value


def test_create_without_gpu(svs):
    _no_gpu()
    rc, out = _create(svs.lib(), -1, 640, 480, 32)
    assert rc == SVS_ERR_NOGPU and not out.value
    with pytest.raises(svs.SvsError):
        svs.StereoMatcher(640, 480, 32)


def test_render_stereo_pair_is_deterministic():
    cam = (150.0, 79.5, 59.5, 0.075)
    a = si.render_stereo_pair(np.array([0.1, 0.0, 0.3]), 0.05, 9, 160, 120, cam)
    b = si.render_stereo_pair(np.array([0.1, 0.0, 0.3]), 0.05, 9, 160, 120, cam)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    left, right, disp = a
    assert left.dtype == right.dtype == np.uint8 and disp.dtype == np.float32
    assert left.tobytes() == si.render_frame(np.array([0.1, 0.0, 0.3]), 0.05, 9, 160, 120, cam)[0].tobytes()
    assert not np.array_equal(left, right)


# render_frame's outputs before noise_seed existed (sha256 prefixes of the image and disparity bytes)
RENDER_FRAME_HASHES = [
    ((np.array([0.0, 0.0, 0.0]), 0.0, 77, 160, 120, (150.0, 80.0, 60.0, 0.075)), ("2a59d08926c00643", "d8b023f9fe18b29a")),
    ((np.array([0.3, -0.1, 0.5]), 0.1, 5, 96, 64, (90.0, 47.5, 31.5, 0.1)), ("95cc6ade164502df", "eddb12253460e2ec")),
]


@pytest.mark.parametrize("case", range(len(RENDER_FRAME_HASHES)))
def test_render_frame_is_unchanged_by_noise_seed(case):
    args, want = RENDER_FRAME_HASHES[case]
    out = si.render_frame(*args)
    assert tuple(hashlib.sha256(a.tobytes()).hexdigest()[:16] for a in out) == want
    explicit = si.render_frame(*args, noise_seed=args[2] + 100)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(out, explicit))


def test_opencv_stereobm_finds_the_rendered_disparity():
    left, right, gt = si.render_stereo_pair(np.array([0.0, 0.0, 0.0]), 0.0, 77)
    bm = cv2.StereoBM_create(numDisparities=32, blockSize=7)
    bm.setPreFilterCap(31); bm.setTextureThreshold(10); bm.setUniquenessRatio(15)
    bm.setSpeckleWindowSize(100); bm.setSpeckleRange(32); bm.setDisp12MaxDiff(1)
    d = bm.compute(left, right).astype(np.float32) / 16
    valid = d > 0
    assert valid.mean() > 0.5
    assert np.mean(np.abs(d[valid] - gt[valid]) <= 1) >= 0.95
