"""svs::GuidedMatcher::{matchAndTrack, processMatchedPoints, addNewPoints, addMorePoints} and svs::shallWeDropNewKeyframe
(include/svs_b200.hpp) from C++: compiles with plain g++ against the C ABI, fails loudly without a GPU, and on the GPU
gives what the C ABI (checked inside the driver) and the Python binding give."""
import os
import subprocess

import numpy as np
import pytest

from scavislam_b200 import frontend_inputs as fi
from scavislam_b200 import synth_images as si

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "frontend_points_main")
NLV = 2


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "frontend_points_main.cpp")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    hdr = os.path.join(ROOT, "include", "svs_b200.hpp")
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return EXE


def _scene(oracle):
    seq = si.sequence(2)
    cams = fi.level_cams(nlevels=NLV)
    levels = [(640 >> l, 480 >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(NLV)]
    kf_pyr = fi.uint8_pyramid(seq[0]["img"], NLV)
    cur_pyr = fi.uint8_pyramid(seq[1]["img"], NLV)
    feats, pts = [], []
    for l in range(NLV):
        g = oracle.fast_grid(640 >> l, 480 >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
        xy, off = oracle.fast_detect_adaptively(cur_pyr[l], g, 5)
        feats.append((xy, np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(9)]).astype(np.int32)))
        kxy, _ = oracle.fast_detect_adaptively(kf_pyr[l], g, 5)
        d = seq[0]["disp"][kxy[:, 1] << l, kxy[:, 0] << l] / (1 << l)
        kxy, d = kxy[d > 0], d[d > 0]
        z = cams[l][0] * cams[l][3] / d
        p = np.zeros(len(kxy), oracle.MATCH_POINT_DTYPE)
        p["anchor_level"] = l
        p["xyz_anchor"] = np.stack([(kxy[:, 0] - cams[l][1]) / cams[l][0] * z, (kxy[:, 1] - cams[l][2]) / cams[l][0] * z, z], 1)
        p["anchor_obs_pyr"] = kxy
        pts.append(p)
    pts = np.concatenate(pts)
    n = len(pts)
    sizes = [n // 4, n // 4, n - 2 * (n // 4)]
    T_cur = oracle.se3_exp(np.array([0.001, 0.0, -0.02, 0.0, -0.0035, 0.0]))
    T_key_w = oracle.se3_exp(np.array([0.3, -0.1, 0.2, 0.01, 0.02, -0.01]))
    return dict(levels=levels, cam=tuple(cams[0][:4]), kf=kf_pyr, cur=cur_pyr, disp=seq[1]["disp"], feats=feats, pts=pts,
                sizes=sizes, T_cur=T_cur, T_key_w=T_key_w, nmax=300)


def _dump(sc, path):
    with open(path, "wb") as f:
        w = lambda a, t: np.ascontiguousarray(a, t).tofile(f)
        w([len(sc["levels"])], np.int32)
        for (lw, lh, lf_, lpx, lpy) in sc["levels"]:
            w([lw, lh], np.int32); w([lf_, lpx, lpy], np.float64)
        w(sc["cam"], np.float64)
        for im in sc["kf"] + sc["cur"]:
            w(im, np.uint8)
        w(sc["disp"], np.float32)
        for xy, c in sc["feats"]:
            w([len(c)], np.int32); w(xy, np.int32); w(c, np.int32)
        w(sc["T_cur"], np.float64); w(sc["T_key_w"], np.float64)
        w([len(sc["sizes"])] + list(sc["sizes"]), np.int32)
        sc["pts"].tofile(f)
        w([sc["nmax"]], np.int32)


def test_frontend_points_cpp_compiles_and_fails_loudly_without_gpu(oracle, tmp_path):
    import torch
    exe = _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe, os.path.join(ROOT, "README.md"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode != 0
    _dump(_scene(oracle), tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_GPU" in r.stderr


@pytest.mark.gpu
def test_frontend_points_cpp_matches_c_abi_and_python(svs, oracle, tmp_path):
    exe = _build()
    sc = _scene(oracle)
    _dump(sc, tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    num_obs, num_new, drop, ng = np.frombuffer(raw, np.int32, 4)
    o = 16
    tr = np.frombuffer(raw, svs.TRACKED_POINT_DTYPE, ng, o); o += svs.TRACKED_POINT_DTYPE.itemsize * ng
    st = svs.SvsPointStats.from_buffer_copy(raw[o:o + svs.C.sizeof(svs.SvsPointStats)]).as_dict()
    o += svs.C.sizeof(svs.SvsPointStats)
    nf = int(np.frombuffer(raw, np.int32, 1, o)[0]); o += 4
    fresh = np.frombuffer(raw, svs.NEW_POINT_DTYPE, nf, o); o += svs.NEW_POINT_DTYPE.itemsize * nf
    nm = int(np.frombuffer(raw, np.int32, 1, o)[0]); o += 4
    more = np.frombuffer(raw, svs.NEW_POINT_DTYPE, nm, o)
    m = svs.GuidedMatcher(sc["levels"])
    m.set_keyframe(0, sc["T_key_w"], sc["kf"])
    m.set_current(sc["cur"], sc["disp"])
    for l, (xy, c) in enumerate(sc["feats"]):
        m.set_features(l, xy, c)
    f_py = m.add_more_points(1, sc["cam"], 1)
    ends = np.cumsum(sc["sizes"])
    groups = [sc["pts"][a:b] for a, b in zip([0] + list(ends[:-1]), ends)]
    res, a, b = m.match_track(sc["T_cur"], sc["T_key_w"], groups, sc["nmax"], 4, 22, 10)
    out, st_py, flags, drop_py = m.process_matched_points(sc["T_cur"], sc["cam"], int(ends[-2]))
    m_py = m.add_more_points(0, sc["cam"], 2)
    m.close()
    assert (num_obs, num_new, bool(drop), ng) == (b, a, drop_py, len(out))
    assert tr.tobytes() == out.tobytes()
    for k in ("num_matched_points", "num_tracked", "num_new"):
        assert st[k] == st_py[k]
    assert np.array_equal(st["grid3x3"], st_py["grid3x3"]) and np.array_equal(st["grid2x2"], st_py["grid2x2"])
    assert fresh.tobytes() == f_py[0].tobytes() and more.tobytes() == m_py[0].tobytes()
    assert nf > 0   # the second seeding may legitimately take nothing (every 3x3 cell above min_num_points)
