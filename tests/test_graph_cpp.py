"""svs::DeviceMap's pose-graph growth (include/svs_b200.hpp) from C++: compiles with plain g++ against the C ABI, fails
loudly without a GPU, and on the GPU gives what the C ABI gives on a second handle and what the Python layer gives,
bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import map_reference as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "graph_main")
W, H, THR = 640, 480, 4


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "graph_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


def _case():
    m = mr.make_map(12, 40, seed=4)
    rng = np.random.default_rng(4)
    V, Np = len(m["poses"]), len(m["point_anchor"])
    vp, vs = m["vis_ptr"], m["vis_pose"]
    pt = np.repeat(np.arange(Np), np.diff(vp))
    tp = rng.permutation(np.unique(pt[vs >= V - 3]))[:80].astype(np.int32)
    n = 10
    kf = dict(T=np.array([0, 0, 0, 1.0, -0.05, 0, 0]), new_anchor=np.full(n, V - 1, np.int32),
              new_xyz=np.stack([rng.uniform(-2, 2, n), rng.uniform(-1, 1, n), rng.uniform(4, 9, n)], 1),
              new_anchor_center=rng.uniform(0, 400, (n, 3)), new_anchor_level=np.zeros(n, np.int32),
              new_center=rng.uniform(0, 400, (n, 3)), new_level=np.ones(n, np.int32), track_point=tp,
              track_center=np.stack([rng.uniform(0, W, len(tp)), rng.uniform(0, H, len(tp)), np.zeros(len(tp))], 1),
              track_level=np.zeros(len(tp), np.int32))
    edges = (np.array([0, 1], np.int32), np.array([V, V], np.int32), np.array([9, 9], np.int32))
    T_moved = np.concatenate([[0, 0, 0, 1.0], [-0.6, 0.01, 0.0]])
    return m, kf, edges, V, T_moved


def _dump(path, m, kf, edges, V, T_moved):
    hd = [V, len(m["point_anchor"]), len(m["vis_pose"]), V - 1, len(kf["new_anchor"]), len(kf["track_point"]), THR, W, H,
          len(edges[0]), V]
    parts = [hd] + [np.ravel(m[k]) for k in ("poses", "point_anchor", "xyz_anchor", "vis_ptr", "vis_pose", "feat_center", "feat_level")]
    parts += [np.ravel(kf[k]) for k in ("T", "new_anchor", "new_xyz", "new_anchor_center", "new_anchor_level", "new_center",
                                        "new_level", "track_point", "track_center", "track_level")]
    parts += [np.ravel(e) for e in edges] + [T_moved]
    np.concatenate([np.asarray(p, np.float64) for p in parts]).tofile(path)


def test_graph_cpp_compiles_and_fails_loudly_without_gpu(svs, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    _dump(tmp_path / "in.bin", *_case())
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stdout


@pytest.mark.gpu
def test_graph_cpp_matches_c_abi_and_python(svs, tmp_path):
    exe = _build()
    m, kf, edges, V, T_moved = _case()
    _dump(tmp_path / "in.bin", m, kf, edges, V, T_moved)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = np.fromfile(tmp_path / "out.bin", np.float64)
    dm = svs.DeviceMap(device=0)
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_pose_graph(np.zeros(V + 1, np.int32), [], [], np.zeros((0, 7)), np.zeros((0, 36)))
    _, _, table, ne = dm.add_keyframe_graph(V - 1, kf["T"], THR, W, H, **{k: kf[k] for k in kf if k != "T"})
    assert ne > 0
    dm.add_edges(*edges, moved_vertex=V, T_moved_from_w=T_moved)
    g = dm.get_graph()
    dm.close()
    nt = int(out[0])
    want = np.concatenate([[nt], table.ravel(), g["nbr_ptr"], g["nbr_id"], g["nbr_strength"], g["nbr_T"].ravel(),
                           g["nbr_Lambda"].ravel()]).astype(np.float64)
    assert out.tobytes() == want.tobytes()
