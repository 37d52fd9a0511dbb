"""svs_chol6 without a GPU: the handle refuses to exist (no CPU fallback), and the C++ adapter of INTEGRATION.md
compiles against include/svs_b200.hpp and is the one the document prints."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "chol6_main.cpp")


def test_create_without_gpu_fails(svs):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    assert svs.lib().svs_chol6_create(0, C.byref(h)) == -5   # SVS_ERR_NOGPU
    assert not h.value
    with pytest.raises(svs.SvsError):
        svs.BlockCholesky6()


def test_cpp_adapter_compiles(svs, tmp_path):
    exe = str(tmp_path / "chol6_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
                           "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    import torch
    if torch.cuda.is_available():
        return
    (tmp_path / "in.bin").write_bytes(b"")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 2 and "BAD_INPUT" in r.stdout


def _code(text):
    return [ln.rstrip() for ln in text.strip("\n").splitlines()]


def test_integration_doc_prints_the_tested_adapter():
    src = open(SRC).read()
    adapter = re.search(r"// ---- INTEGRATION.md adapter begin\n(.*?)// ---- INTEGRATION.md adapter end", src, re.S).group(1)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    blocks = re.findall(r"```cpp\n(.*?)```", doc, re.S)
    assert any(_code(adapter) == _code(b)[-len(_code(adapter)):] for b in blocks), \
        "INTEGRATION.md must print the adapter of tests/cpp/chol6_main.cpp"
