"""svs::PlaceRecognizer (include/svs_b200.hpp) from C++: compiles with plain g++ against the C ABI, fails loudly
without a GPU, and on the GPU gives what the C ABI and the Python binding give."""
import os
import subprocess

import numpy as np
import pytest

from scavislam_b200 import synth_place as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "place_main")


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "place_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


def _dump(words, kfs, path):
    with open(path, "wb") as f:
        np.array([len(words)], np.int32).tofile(f)
        np.asarray(sp.CAM, np.float64).tofile(f)
        np.ascontiguousarray(words, np.float32).tofile(f)
        np.array([len(kfs)], np.int32).tofile(f)
        for k in kfs:
            excl = np.array([k["id"] - 1] if k["id"] else [], np.int32)
            np.array([k["id"], len(k["desc"]), 1, len(excl)], np.int32).tofile(f)
            excl.tofile(f)
            np.ascontiguousarray(k["desc"], np.float32).tofile(f)
            np.ascontiguousarray(k["uvu"], np.float64).tofile(f)


def test_place_cpp_compiles_and_fails_loudly_without_gpu(svs, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    words, kfs = sp.make_sequence(num_keyframes=3, num_scenes=3, num_words=100, landmarks=20, seed=1)
    _dump(words, kfs, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout


@pytest.mark.gpu
def test_place_cpp_matches_c_abi_and_python(svs, tmp_path):
    exe = _build()
    words, kfs = sp.make_sequence(num_keyframes=50, num_scenes=40, seed=21)
    _dump(words, kfs, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    rec = np.dtype([("i", "<i4", 3), ("T", "<f8", 7)])
    out = np.frombuffer(raw, rec)
    pr = svs.PlaceRecognizer(words, sp.CAM, device=0)
    loops = 0
    for k, o in zip(kfs, out):
        res = pr.add_location(k["id"], k["desc"], k["uvu"], exclude=[k["id"] - 1] if k["id"] else [])
        assert o["i"].tolist() == [res["best_keyframe_id"], res["num_inliers"], int(res["loop_found"])]
        assert o["T"].tobytes() == res["T_query_from_loop"].tobytes()
        loops += res["loop_found"]
    assert f"loops={loops}" in r.stdout and loops > 0
