"""svs::DeviceMap::localRegisterFrame (include/svs_b200.hpp) from C++: compiles with plain g++ against the C ABI, fails
loudly without a GPU, and on the GPU gives what the C ABI (checked inside the driver) and the Python binding give."""
import functools
import os
import subprocess

import numpy as np
import pytest

from scavislam_b200 import synth_loop as sl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "register_main")


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "register_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


@functools.lru_cache(maxsize=1)
def _scene():
    from oracle import pyoracle
    return sl.make_register_scene(pyoracle)


def _dump(sc, covis, path):
    m, lv = sc["map"], sc["levels"]
    V = len(m["poses"])
    rf = sc["frames"][sc["root"]]
    with open(path, "wb") as f:
        w = lambda a, t: np.ascontiguousarray(a, t).tofile(f)
        w([V, len(m["point_anchor"]), len(m["vis_pose"]), len(lv)], np.int32)
        w(m["poses"], np.float64); w(m["point_anchor"], np.int32); w(m["xyz_anchor"], np.float64)
        w(m["vis_ptr"], np.int32); w(m["vis_pose"], np.int32); w(m["feat_center"], np.float64); w(m["feat_level"], np.int32)
        w(sc["nbr_ptr"], np.int32); w(sc["nbr_id"], np.int32)
        for (lw, lh, lf_, lpx, lpy) in lv:
            w([lw, lh], np.int32); w([lf_, lpx, lpy], np.float64)
        w(sc["cam"], np.float64)
        w([covis, sc["root"], len(sc["window"])], np.int32); w(sc["window"], np.int32)
        w(np.arange(V), np.int32); w([V], np.int32)
        for v in range(V):
            for im in sc["frames"][v]["pyr"]:
                w(im, np.uint8)
        for im in rf["pyr"]:
            w(im, np.uint8)
        w(rf["disp"], np.float32)
        for xy, c in sc["root_features"]:
            w([len(c)], np.int32); w(xy, np.int32); w(c, np.int32)


def test_register_cpp_compiles_and_fails_loudly_without_gpu(svs, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe, os.path.join(ROOT, "README.md"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode != 0
    from oracle import pyoracle
    sc = sl.make_register_scene(pyoracle, n_kf=4, per_level=(20, 10))
    _dump(sc, 5, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout


@pytest.mark.gpu
def test_register_cpp_matches_c_abi_and_python(svs, tmp_path):
    from scavislam_b200 import capi
    exe = _build()
    sc = _scene()
    _dump(sc, 20, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    counts = np.frombuffer(raw, np.int32, 11)
    T = np.frombuffer(raw, np.float64, 21, 44).reshape(3, 7)
    o = 44 + 168
    ns = int(np.frombuffer(raw, np.int32, 1, o)[0]); o += 4
    stats = np.frombuffer(raw, capi.REGISTER_STATS_DTYPE, ns, o); o += 28 * ns
    nt = int(np.frombuffer(raw, np.int32, 1, o)[0]); o += 4
    tp = np.frombuffer(raw, np.int32, nt, o); o += 4 * nt
    tl = np.frombuffer(raw, np.int32, nt, o); o += 4 * nt
    tc = np.frombuffer(raw, np.int32, nt, o); o += 4 * nt
    tu = np.frombuffer(raw, np.float64, 3 * nt, o).reshape(nt, 3)
    m = sc["map"]
    V = len(m["poses"])
    dm = svs.DeviceMap()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_graph(sc["nbr_ptr"], sc["nbr_id"])
    mt = svs.GuidedMatcher(sc["levels"], max_keyframes=V, max_points=8192)
    for v in range(V):
        mt.set_keyframe(v, np.array([0, 0, 0, 1, 0, 0, 0.0]), sc["frames"][v]["pyr"])
    rf = sc["frames"][sc["root"]]
    mt.set_current(rf["pyr"], rf["disp"])
    for l, (xy, c) in enumerate(sc["root_features"]):
        mt.set_features(l, xy, c)
    po = svs.PoseOptimizer(max_obs=8192)
    res, st, tracks = dm.local_register_frame(mt, po, sc["cam"], 20, sc["root"], sc["window"], np.arange(V, dtype=np.int32))
    assert res["registered"] == 1 and f"registered=1 tracks={nt}" in r.stdout
    assert counts.tolist() == [res[k] for k in capi.REGISTER_COUNTS]
    for i, k in enumerate(("T_align1", "T_newroot_from_oldroot", "T_newroot_from_w")):
        assert T[i].tobytes() == res[k].tobytes()
    assert stats.tobytes() == st.tobytes()
    np.testing.assert_array_equal(tp, tracks["point"]); np.testing.assert_array_equal(tl, tracks["level"])
    np.testing.assert_array_equal(tc, tracks["committed"]); np.testing.assert_array_equal(tu, tracks["uvu"])
    for h in (dm, mt, po):
        h.close()
