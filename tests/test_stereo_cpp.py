"""svs::StereoBM (include/svs_b200.hpp) from C++: compiles with plain g++ against the C ABI, fails loudly without a
GPU, and on the GPU gives what the C ABI gives, which is OpenCV's StereoBM with the reference's settings."""
import os
import subprocess

import cv2
import numpy as np
import pytest

from scavislam_b200 import synth_images as si

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "stereo_main")


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "stereo_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


def _dump(left, right, nd, path):
    with open(path, "wb") as f:
        np.array([left.shape[1], left.shape[0], nd], np.int32).tofile(f)
        np.ascontiguousarray(left).tofile(f)
        np.ascontiguousarray(right).tofile(f)


def test_stereo_cpp_compiles_and_fails_loudly_without_gpu(svs, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    rng = np.random.default_rng(0)
    _dump(rng.integers(0, 256, (48, 64), np.uint8), rng.integers(0, 256, (48, 64), np.uint8), 16, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout


@pytest.mark.gpu
def test_stereo_cpp_matches_c_abi_and_opencv(svs, tmp_path):
    exe = _build()
    left, right, _ = si.render_stereo_pair(np.array([0.0, 0.0, 0.0]), 0.0, 5)
    _dump(left, right, 32, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    d = np.fromfile(tmp_path / "out.bin", np.float32).reshape(left.shape)
    sm = svs.StereoMatcher(640, 480, 32, device=0)
    sm.compute(left, right)
    assert d.tobytes() == sm.disparity().tobytes()
    sm.close()
    bm = cv2.StereoBM_create(numDisparities=32, blockSize=7)
    bm.setPreFilterCap(31); bm.setTextureThreshold(10); bm.setUniquenessRatio(15)
    bm.setSpeckleWindowSize(100); bm.setSpeckleRange(32); bm.setDisp12MaxDiff(1)
    assert np.array_equal((d * 16).astype(np.int16), bm.compute(left, right))
    assert (d > 0).mean() > 0.5
