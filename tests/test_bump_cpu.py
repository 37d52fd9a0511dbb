"""svs::Bump, the typed bump allocator in scavislam_b200/csrc/handle.cuh that lays out every module's device buffers:
built with plain g++ (handle.cuh needs only the CUDA headers, none of its CUDA calls is linked) and run on the host."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INCLUDE = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


def test_bump_sizing_and_carve_agree(tmp_path):
    exe = tmp_path / "bump_main"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", f"-I{CUDA_INCLUDE}",
                           "-I", os.path.join(ROOT, "scavislam_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "bump_main.cpp"), "-o", str(exe)])
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK 7 arrays"), r.stdout
