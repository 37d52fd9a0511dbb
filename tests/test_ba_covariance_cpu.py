"""svs::StereoGraph::computeMarginals without a GPU: the program of tests/cpp/ba_covariance_main.cpp compiles against
include/svs_b200.hpp and reports the missing device (SVS_ERR_NOGPU from svs_ba_create)."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "ba_covariance_main.cpp")


def test_cpp_compute_marginals_compiles_and_reports_no_gpu(svs, tmp_path):
    exe = str(tmp_path / "ba_covariance_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
                           "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    import torch
    if torch.cuda.is_available():
        return
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:   # one fixed identity pose, nothing else
        np.array([1, 0, 0, 0, 0, 1, 0], np.int32).tofile(f)
        np.array([500.0, 320.0, 240.0, 0.1, 0.0]).tofile(f)
        np.array([0, 0, 0, 1, 0, 0, 0], np.float64).tofile(f)
        np.array([1], np.int32).tofile(f)
    r = subprocess.run([exe, str(inp), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout, r.stdout + r.stderr
