"""svs_chol6 marginals without a GPU: the adapter with its solveBlocks / solvePattern overrides compiles against
include/svs_b200.hpp and reports the missing device, and INTEGRATION.md prints exactly the tested overrides."""
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "chol6_marginals_main.cpp")
OVR = re.compile(r"// ---- INTEGRATION.md overrides begin\n(.*?)// ---- INTEGRATION.md overrides end\n", re.S)


def _code(text):
    return [ln.rstrip() for ln in text.strip("\n").splitlines()]


def test_cpp_marginals_adapter_compiles_and_reports_no_gpu(svs, tmp_path):
    exe = str(tmp_path / "chol6_marginals_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
                           "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    import torch
    if torch.cuda.is_available():
        return
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:   # P = 1: one identity block, one request
        f.write(bytes.fromhex("01000000" "01000000" "00000000" "01000000" "00000000"))
        np.eye(6).ravel(order="F").tofile(f)
        np.array([1, 0, 0], np.int32).tofile(f)
    r = subprocess.run([exe, str(inp), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout, r.stdout + r.stderr


def test_integration_doc_prints_the_tested_overrides():
    src = open(SRC).read()
    overrides = OVR.search(src).group(1)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    blocks = re.findall(r"```cpp\n(.*?)```", doc, re.S)
    assert any(_code(overrides) == _code(b) for b in blocks), \
        "INTEGRATION.md must print the overrides of tests/cpp/chol6_marginals_main.cpp"


def test_marginals_adapter_is_the_printed_adapter_plus_overrides():
    """Without its overrides, the class of chol6_marginals_main.cpp is the adapter of chol6_main.cpp."""
    adapter = re.search(r"// ---- INTEGRATION.md adapter begin\n(.*?)// ---- INTEGRATION.md adapter end",
                        open(os.path.join(ROOT, "tests", "cpp", "chol6_main.cpp")).read(), re.S).group(1)
    src = OVR.sub("", open(SRC).read())
    cls = re.search(r"(template <typename MatrixType>\nclass LinearSolverSvs .*?\n};\n)", src, re.S).group(1)
    assert [ln for ln in _code(cls) if ln] == [ln for ln in _code(adapter) if ln]
