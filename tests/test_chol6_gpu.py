"""svs_chol6: the device block Cholesky of the BA path as g2o's LinearSolver<Matrix6d>::solve(A, x, b) for a
caller's own upper block-CCS system.  Checked against numpy on the dense matrix, against the BA handle's own
reduced-system solve, and through the C++ adapter of INTEGRATION.md."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from scavislam_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SVS_ERR_INVALID = -1

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- helpers

def random_spd(P, pairs, seed, diag=1.0):
    """Dense 6P x 6P SPD matrix: sum of J^T J over random couplings of the pose pairs (i, j), plus diag * I."""
    rng = np.random.default_rng(seed)
    A = np.zeros((6 * P, 6 * P))
    for i, j in pairs:
        idx = np.r_[6 * i:6 * i + 6, 6 * j:6 * j + 6]
        J = rng.standard_normal((6, 12))
        A[np.ix_(idx, idx)] += J.T @ J
    A += diag * np.eye(6 * P)
    return A


def to_upper_ccs(A, pattern=None):
    """Upper block CCS of the dense A: the blocks with a nonzero entry (or the (i, j) pairs of `pattern`) with
    i <= j, plus every diagonal block; each block column-major."""
    P = A.shape[0] // 6
    blk = lambda i, j: A[6 * i:6 * i + 6, 6 * j:6 * j + 6]
    if pattern is None:
        nz = np.abs(A.reshape(P, 6, P, 6)).max(axis=(1, 3)) > 0
    else:
        nz = np.zeros((P, P), bool)
        for i, j in pattern:
            nz[min(i, j), max(i, j)] = True
    col_ptr, row_idx, blocks = [0], [], []
    for j in range(P):
        for i in range(j + 1):
            if i == j or nz[i, j]:
                row_idx.append(i)
                blocks.append(blk(i, j).ravel(order="F"))
        col_ptr.append(len(row_idx))
    return (np.array(col_ptr, np.int32), np.array(row_idx, np.int32),
            np.ascontiguousarray(np.array(blocks, np.float64).reshape(-1, 36)))


def banded_pairs(P, w, seed, n=None):
    rng = np.random.default_rng(seed)
    n = n or 3 * P
    pairs = [(i, i + 1) for i in range(P - 1)]
    for _ in range(n):
        i = int(rng.integers(0, P - 1))
        j = min(P - 1, i + int(rng.integers(1, w + 1)))
        pairs.append((i, j))
    return pairs


def check_numpy(A, b, x, tol=1e-9):
    x_ref = np.linalg.solve(A, b)
    assert np.abs(x - x_ref).max() <= tol * np.abs(x_ref).max()
    assert np.linalg.norm(A @ x - b) <= 1e-10 * np.linalg.norm(b)


@pytest.fixture
def chol(svs):
    h = svs.BlockCholesky6(device=0)
    yield h
    h.close()


# ---------------------------------------------------------------------------------------------- 1. banded window

def test_banded_window_two_ended(chol):
    P = 200
    A = random_spd(P, banded_pairs(P, 8, seed=1), seed=2)
    b = np.random.default_rng(3).standard_normal(6 * P)
    x, rc, st = chol.solve(*to_upper_ccs(A), b)
    assert rc == 0
    check_numpy(A, b, x)
    assert st["nbranch"] == 2 and st["general"] == 0
    assert st["P"] == P and st["nnzb_L"] >= st["nnzb_A"] and st["ms"] > 0


# ---------------------------------------------------------------------------------------------- 2. same answer as the BA solve

@pytest.mark.parametrize("which", ["C1", "window90"])
def test_same_answer_as_ba_solve(svs, chol, which):
    pb = synth.make_config("C1") if which == "C1" else synth.make_window(90, 4000, seed=34)
    ba = svs.BundleAdjuster(device=0)
    try:
        ba.set_problem(pb)
        S, bs, _ = ba.reduced_system(True, 1.0, 50.0)
        x_ba, rc_ba = ba.solve_reduced(True, 1.0, 50.0)
    finally:
        ba.close()
    assert rc_ba == 0
    x, rc, st = chol.solve(*to_upper_ccs(S), bs)
    assert rc == 0
    assert np.abs(x - x_ba).max() <= 1e-12 * np.abs(x_ba).max()


# ---------------------------------------------------------------------------------------------- 3. every solver path

def test_loop_closure_fill_in(chol):
    P = 120
    pairs = banded_pairs(P, 4, seed=5) + [(3, 110), (10, 95), (20, 80), (0, 119)]
    A = random_spd(P, pairs, seed=6)
    b = np.random.default_rng(7).standard_normal(6 * P)
    x, rc, st = chol.solve(*to_upper_ccs(A), b)
    assert rc == 0
    check_numpy(A, b, x)
    assert st["nnzb_L"] > st["nnzb_A"]


def test_all_to_all_takes_general_solver(chol):
    P = 140
    pairs = [(i, j) for i in range(P) for j in range(i + 1, P)]
    rng = np.random.default_rng(8)
    M = rng.standard_normal((6 * P, 6 * P))
    A = M @ M.T / (6 * P) + np.eye(6 * P)
    b = rng.standard_normal(6 * P)
    x, rc, st = chol.solve(*to_upper_ccs(A, pairs), b)
    assert rc == 0
    check_numpy(A, b, x)
    assert st["general"] == 1


@pytest.mark.parametrize("P", [1, 5])
def test_small(chol, P):
    pairs = [(i, j) for i in range(P) for j in range(i, P)]
    A = random_spd(P, pairs, seed=P)
    b = np.random.default_rng(P + 1).standard_normal(6 * P)
    x, rc, st = chol.solve(*to_upper_ccs(A), b)
    assert rc == 0
    check_numpy(A, b, x)
    assert st["nbranch"] == 1


def test_block_diagonal(chol):
    P = 30
    A = random_spd(P, [(i, i) for i in range(P)], seed=9)   # (i, i) couplings: diagonal blocks only
    assert np.abs(A.reshape(P, 6, P, 6)).max(axis=(1, 3))[~np.eye(P, dtype=bool)].max() == 0
    b = np.random.default_rng(10).standard_normal(6 * P)
    x, rc, st = chol.solve(*to_upper_ccs(A), b)
    assert rc == 0
    check_numpy(A, b, x)
    assert st["nnzb_A"] == P and st["nnzb_L"] == P


# ---------------------------------------------------------------------------------------------- 4. not positive definite

def test_not_positive_definite_then_recovers(chol):
    P = 40
    pairs = banded_pairs(P, 3, seed=11)
    A = random_spd(P, pairs, seed=12)
    b = np.random.default_rng(13).standard_normal(6 * P)
    bad = A.copy()
    bad[6 * 17 + 2, 6 * 17 + 2] = -1e3
    x, rc, _ = chol.solve(*to_upper_ccs(bad, pairs), b)
    assert rc == 1
    assert not x.any()
    x, rc, _ = chol.solve(*to_upper_ccs(A, pairs), b)
    assert rc == 0
    check_numpy(A, b, x)


# ---------------------------------------------------------------------------------------------- 5. lower triangle ignored

def test_lower_triangle_of_diagonal_blocks_ignored(chol):
    P = 60
    A = random_spd(P, banded_pairs(P, 5, seed=14), seed=15)
    b = np.random.default_rng(16).standard_normal(6 * P)
    cp, ri, blocks = to_upper_ccs(A)
    x0, rc0, _ = chol.solve(cp, ri, blocks, b)
    poisoned = blocks.copy()
    lower = np.tril(np.ones((6, 6), bool), -1).ravel(order="F")   # (r > c) in column-major order
    for j in range(P):
        poisoned[cp[j + 1] - 1, lower] = np.nan
    x1, rc1, _ = chol.solve(cp, ri, poisoned, b)
    assert rc0 == 0 and rc1 == 0
    assert np.array_equal(x0, x1)


# ---------------------------------------------------------------------------------------------- 6. cache

def test_symbolic_cache(chol):
    P = 80
    pa, pb_ = banded_pairs(P, 4, seed=17), banded_pairs(P, 6, seed=18)
    b = np.random.default_rng(19).standard_normal(6 * P)
    A1 = random_spd(P, pa, seed=20)
    _, rc, st = chol.solve(*to_upper_ccs(A1, pa), b)
    assert rc == 0 and st["symbolic_reused"] == 0
    A2 = random_spd(P, pa, seed=21)
    x, rc, st = chol.solve(*to_upper_ccs(A2, pa), b)
    assert rc == 0 and st["symbolic_reused"] == 1
    check_numpy(A2, b, x)
    A3 = random_spd(P, pb_, seed=22)
    x, rc, st = chol.solve(*to_upper_ccs(A3, pb_), b)
    assert rc == 0 and st["symbolic_reused"] == 0
    check_numpy(A3, b, x)
    x, rc, st = chol.solve(*to_upper_ccs(A3, pb_), b)
    assert st["symbolic_reused"] == 1
    chol.init()
    x, rc, st = chol.solve(*to_upper_ccs(A3, pb_), b)
    assert rc == 0 and st["symbolic_reused"] == 0
    check_numpy(A3, b, x)


# ---------------------------------------------------------------------------------------------- 7. device input

def test_device_input_matches_host(chol):
    import torch
    P = 150
    A = random_spd(P, banded_pairs(P, 6, seed=23), seed=24)
    b = np.random.default_rng(25).standard_normal(6 * P)
    cp, ri, blocks = to_upper_ccs(A)
    x_h, rc_h, _ = chol.solve(cp, ri, blocks, b)
    x_d, rc_d, st = chol.solve(cp, ri, torch.from_numpy(blocks).cuda(), torch.from_numpy(b).cuda())
    assert rc_h == 0 and rc_d == 0
    assert isinstance(x_d, torch.Tensor) and x_d.is_cuda
    assert np.array_equal(x_h, x_d.cpu().numpy())


# ---------------------------------------------------------------------------------------------- 8. malformed input

def _raw_solve(svs, chol, P, cp, ri, blocks, b, x):
    ptr = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    return svs.lib().svs_chol6_solve(chol._h, P, ptr(cp, C.c_int), ptr(ri, C.c_int),
                                     None if blocks is None else blocks.ctypes.data,
                                     None if b is None else b.ctypes.data, None if x is None else x.ctypes.data, 0, None)


def test_malformed_input_rejected_and_handle_survives(svs, chol):
    P = 20
    pairs = banded_pairs(P, 3, seed=26)
    A = random_spd(P, pairs, seed=27)
    b = np.random.default_rng(28).standard_normal(6 * P)
    cp, ri, blocks = to_upper_ccs(A, pairs)
    x = np.zeros(6 * P)
    assert _raw_solve(svs, chol, P, cp, ri, blocks, b, x) == 0
    j = next(j for j in range(P) if cp[j + 1] - cp[j] >= 2)   # a column with an off-diagonal block
    cases = {}
    r = ri.copy(); r[cp[j]] = j + 1                          # row > column
    cases["row > column"] = (P, cp, r, blocks, b, x)
    r = ri.copy(); r[cp[j]], r[cp[j] + 1] = r[cp[j] + 1], r[cp[j]]   # unsorted
    cases["unsorted rows"] = (P, cp, r, blocks, b, x)
    r = ri.copy(); r[cp[j] + 1] = r[cp[j]]                  # repeated
    cases["repeated row"] = (P, cp, r, blocks, b, x)
    nodiag_cp, nodiag_ri = cp.copy(), np.delete(ri, cp[j + 1] - 1)   # missing diagonal of column j
    nodiag_cp[j + 1:] -= 1
    cases["missing diagonal"] = (P, nodiag_cp, nodiag_ri, np.delete(blocks, cp[j + 1] - 1, axis=0), b, x)
    c = cp.copy(); c[0] = 1
    cases["col_ptr[0] != 0"] = (P, c, ri, blocks, b, x)
    c = cp.copy(); c[5] = c[4] - 1
    cases["decreasing col_ptr"] = (P, c, ri, blocks, b, x)
    cases["P < 0"] = (-1, cp, ri, blocks, b, x)
    cases["null col_ptr"] = (P, None, ri, blocks, b, x)
    cases["null row_idx"] = (P, cp, None, blocks, b, x)
    cases["null blocks"] = (P, cp, ri, None, b, x)
    cases["null b"] = (P, cp, ri, blocks, None, x)
    cases["null x"] = (P, cp, ri, blocks, b, None)
    for name, args in cases.items():
        assert _raw_solve(svs, chol, *args) == SVS_ERR_INVALID, name
        assert svs.lib().svs_chol6_last_error(chol._h).decode(), name
    # the handle still solves (and still has the analysis of the good pattern)
    x[:] = 0
    st = svs.SvsChol6Stats()
    rc = svs.lib().svs_chol6_solve(chol._h, P, cp.ctypes.data_as(C.POINTER(C.c_int)), ri.ctypes.data_as(C.POINTER(C.c_int)),
                                   blocks.ctypes.data, b.ctypes.data, x.ctypes.data, 0, C.byref(st))
    assert rc == 0 and st.symbolic_reused == 1
    check_numpy(A, b, x)
    with pytest.raises(svs.SvsError):
        chol.solve(cp, ri.copy()[::-1].copy(), blocks, b)


# ---------------------------------------------------------------------------------------------- 9. C++ adapter

def _build_cpp(tmp_path):
    exe = str(tmp_path / "chol6_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "chol6_main.cpp"), "-o", exe,
                           "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    return exe


def write_system(path, cp, ri, blocks, b):
    with open(path, "wb") as f:
        np.array([len(cp) - 1, len(ri)], np.int32).tofile(f)
        cp.astype(np.int32).tofile(f)
        ri.astype(np.int32).tofile(f)
        np.ascontiguousarray(blocks, np.float64).tofile(f)
        np.ascontiguousarray(b, np.float64).tofile(f)


def test_cpp_adapter_matches_python(chol, tmp_path):
    exe = _build_cpp(tmp_path)
    P = 100
    A = random_spd(P, banded_pairs(P, 6, seed=29) + [(2, 90)], seed=30)
    b = np.random.default_rng(31).standard_normal(6 * P)
    cp, ri, blocks = to_upper_ccs(A)
    write_system(tmp_path / "in.bin", cp, ri, blocks, b)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK solved=1" in r.stdout
    x_cpp = np.fromfile(tmp_path / "out.bin", np.float64)
    x_py, rc, _ = chol.solve(cp, ri, blocks, b)
    assert rc == 0
    assert np.abs(x_cpp - x_py).max() <= 1e-12 * np.abs(x_py).max()
