"""svs::DeviceMap::prepareForOptimization and windowState (include/svs_b200.hpp) from C++: compiles with plain g++
against the C ABI, fails loudly without a GPU, turns a refusal into std::runtime_error, and on the GPU gives what the
Python layer gives, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import map_reference as mr
import prepare_reference as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "prepare_main")
ROOT_V, INNER, DBL = 9, 3, 7


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "prepare_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


def _case():
    m = mr.make_map(14, 30, seed=6)
    ptr, ids, _, _ = mr.covisibility_graph(m, max_neighbours=4, with_constraints=False)
    T, L = pr.consistent_graph(ptr, ids, np.random.default_rng(6))
    g = dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=np.zeros(len(ids), np.int32), nbr_T=T, nbr_Lambda=L)
    return m, g


def _dump(path, m, g):
    hd = [len(m["poses"]), len(m["point_anchor"]), len(m["vis_pose"]), len(g["nbr_id"]), ROOT_V, -1, INNER, DBL]
    parts = [hd] + [np.ravel(m[k]) for k in ("poses", "point_anchor", "xyz_anchor", "vis_ptr", "vis_pose", "feat_center", "feat_level")]
    parts += [np.ravel(g[k]) for k in ("nbr_ptr", "nbr_id", "nbr_strength", "nbr_T", "nbr_Lambda")]
    np.concatenate([np.asarray(p, np.float64) for p in parts]).tofile(path)


def test_prepare_cpp_compiles_and_fails_loudly_without_gpu(svs, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    _dump(tmp_path / "in.bin", *_case())
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout


@pytest.mark.gpu
def test_prepare_cpp_matches_python(svs, tmp_path):
    exe = _build()
    m, g = _case()
    _dump(tmp_path / "in.bin", m, g)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = np.fromfile(tmp_path / "out.bin", np.float64)
    dm = svs.DeviceMap(device=0)
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_pose_graph(g["nbr_ptr"], g["nbr_id"], g["nbr_strength"], g["nbr_T"], g["nbr_Lambda"])
    w = dm.prepare_for_optimization(ROOT_V, -1, INNER, DBL)
    wt, mg = dm.window_state()
    poses, _ = dm.get()
    dm.close()
    assert w["do_optimization"] and len(w["c_i"]) > 0
    want = np.concatenate([[1, len(w["window_vertex"])], w["window_vertex"], w["inner"], [len(w["active_point"])], w["active_point"],
                           [len(w["c_i"])], w["c_i"], w["c_j"], w["c_T"].ravel(), w["c_Lambda"].ravel(), wt, mg,
                           poses.ravel()]).astype(np.float64)
    assert out.tobytes() == want.tobytes()
