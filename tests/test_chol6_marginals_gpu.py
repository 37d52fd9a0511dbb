"""svs_chol6 marginals: LinearSolver::solveBlocks / solvePattern (blocks of A^-1) from the device factor, checked
against numpy's inverse of the dense matrix, on every solver path, and through the C++ adapter of INTEGRATION.md."""
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
    """Upper block CCS of the dense A (blocks with a nonzero entry, or the pairs of `pattern`, plus every diagonal
    block), each block column-major."""
    P = A.shape[0] // 6
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
                blocks.append(A[6 * i:6 * i + 6, 6 * j:6 * j + 6].ravel(order="F"))
        col_ptr.append(len(row_idx))
    return (np.array(col_ptr, np.int32), np.array(row_idx, np.int32),
            np.ascontiguousarray(np.array(blocks, np.float64).reshape(-1, 36)))


def banded_pairs(P, w, seed, n=None):
    rng = np.random.default_rng(seed)
    n = n or 3 * P
    pairs = [(i, i + 1) for i in range(P - 1)]
    for _ in range(n):
        i = int(rng.integers(0, P - 1))
        pairs.append((i, min(P - 1, i + int(rng.integers(1, w + 1)))))
    return pairs


def blk(Z, r, c):
    return Z[6 * r:6 * r + 6, 6 * c:6 * c + 6]


def check_blocks(Z, pairs, out, tol=1e-9):
    ref = np.array([blk(Z, r, c) for r, c in pairs])
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() <= tol * np.abs(Z).max()


def check_diag(A, inv_diag):
    check_blocks(np.linalg.inv(A), [(p, p) for p in range(A.shape[0] // 6)], inv_diag)


def upper_pairs(cp, ri):
    return [(int(ri[k]), j) for j in range(len(cp) - 1) for k in range(cp[j], cp[j + 1])]


@pytest.fixture
def chol(svs):
    h = svs.BlockCholesky6(device=0)
    yield h
    h.close()


# ---------------------------------------------------------------------------------------------- banded window

def test_banded_window_blocks(chol):
    P = 200
    A = random_spd(P, banded_pairs(P, 8, seed=1), seed=2)
    inv_diag, rc, st = chol.solve_blocks(*to_upper_ccs(A))
    assert rc == 0
    check_diag(A, inv_diag)
    assert st["nbranch"] == 2 and st["general"] == 0
    assert st["P"] == P and st["n_in_pattern"] == P and st["n_cols_solved"] == 0 and st["ms"] > 0
    assert np.array_equal(inv_diag, inv_diag.swapaxes(1, 2))   # the diagonal blocks are exactly symmetric


def test_banded_window_pattern_and_far_pairs(chol):
    P = 200
    A = random_spd(P, banded_pairs(P, 8, seed=3), seed=4)
    Z = np.linalg.inv(A)
    cp, ri, blocks = to_upper_ccs(A)
    up = upper_pairs(cp, ri)
    out, rc, st = chol.solve_pattern(cp, ri, blocks, up)
    assert rc == 0 and st["n_cols_solved"] == 0 and st["n_in_pattern"] == len(up)
    check_blocks(Z, up, out)
    far = [(0, 199), (199, 0), (5, 150), (150, 5), (40, 120), (5, 150), (120, 40), (3, 3)]
    pairs = up[::7] + far
    out, rc, st = chol.solve_pattern(cp, ri, blocks, pairs)
    assert rc == 0 and st["n_cols_solved"] > 0
    check_blocks(Z, pairs, out)


# ---------------------------------------------------------------------------------------------- every solver path

def test_loop_closure_fill_in(chol):
    P = 120
    pairs = banded_pairs(P, 4, seed=5) + [(3, 110), (10, 95), (20, 80), (0, 119)]
    A = random_spd(P, pairs, seed=6)
    Z = np.linalg.inv(A)
    cp, ri, blocks = to_upper_ccs(A)
    inv_diag, rc, st = chol.solve_blocks(cp, ri, blocks)
    assert rc == 0 and st["nnzb_L"] > st["nnzb_A"]
    check_diag(A, inv_diag)
    req = upper_pairs(cp, ri) + [(110, 3), (60, 2), (2, 60), (119, 50)]
    out, rc, st = chol.solve_pattern(cp, ri, blocks, req)
    assert rc == 0
    check_blocks(Z, req, out)


def test_all_to_all_takes_general_solver(chol):
    P = 140
    pairs = [(i, j) for i in range(P) for j in range(i + 1, P)]
    rng = np.random.default_rng(8)
    M = rng.standard_normal((6 * P, 6 * P))
    A = M @ M.T / (6 * P) + np.eye(6 * P)
    cp, ri, blocks = to_upper_ccs(A, pairs)
    inv_diag, rc, st = chol.solve_blocks(cp, ri, blocks)
    assert rc == 0 and st["general"] == 1
    check_diag(A, inv_diag)
    req = [(0, 139), (139, 0), (70, 71), (12, 12)]
    out, rc, st = chol.solve_pattern(cp, ri, blocks, req)
    assert rc == 0 and st["general"] == 1 and st["n_cols_solved"] == 0
    check_blocks(np.linalg.inv(A), req, out)


@pytest.mark.parametrize("P", [1, 5])
def test_small(chol, P):
    A = random_spd(P, [(i, j) for i in range(P) for j in range(i, P)], seed=P)
    inv_diag, rc, st = chol.solve_blocks(*to_upper_ccs(A))
    assert rc == 0 and st["nbranch"] == 1
    check_diag(A, inv_diag)


def test_block_diagonal(chol):
    P = 30
    A = random_spd(P, [(i, i) for i in range(P)], seed=9)
    cp, ri, blocks = to_upper_ccs(A)
    inv_diag, rc, st = chol.solve_blocks(cp, ri, blocks)
    assert rc == 0 and st["nnzb_L"] == P
    check_diag(A, inv_diag)
    out, rc, st = chol.solve_pattern(cp, ri, blocks, [(0, 29), (29, 0), (4, 7)])   # zero blocks, outside the pattern
    assert rc == 0 and st["n_cols_solved"] > 0
    assert np.abs(out).max() == 0


def test_all_pairs_reproduce_the_inverse(chol):
    P = 30
    A = random_spd(P, banded_pairs(P, 3, seed=32) + [(1, 25)], seed=33)
    Z = np.linalg.inv(A)
    pairs = [(r, c) for r in range(P) for c in range(P)]
    out, rc, st = chol.solve_pattern(*to_upper_ccs(A), pairs)
    assert rc == 0 and st["n_in_pattern"] + st["n_cols_solved"] > 0
    full = out.reshape(P, P, 6, 6).transpose(0, 2, 1, 3).reshape(6 * P, 6 * P)
    assert np.abs(full - Z).max() <= 1e-9 * np.abs(Z).max()
    assert np.abs(full - full.T).max() <= 1e-12 * np.abs(Z).max()


# ---------------------------------------------------------------------------------------------- reduced systems of BA

@pytest.mark.parametrize("which", ["C1", "window90"])
def test_reduced_system_marginals(svs, chol, which):
    pb = synth.make_config("C1") if which == "C1" else synth.make_window(90, 4000, seed=34)
    ba = svs.BundleAdjuster(device=0)
    try:
        ba.set_problem(pb)
        S, _, _ = ba.reduced_system(True, 1.0, 50.0)
    finally:
        ba.close()
    inv_diag, rc, _ = chol.solve_blocks(*to_upper_ccs(S))
    assert rc == 0
    check_diag(S, inv_diag)


# ---------------------------------------------------------------------------------------------- failure and errors

def test_not_positive_definite_then_recovers(chol):
    P = 40
    pairs = banded_pairs(P, 3, seed=11)
    A = random_spd(P, pairs, seed=12)
    bad = A.copy()
    bad[6 * 17 + 2, 6 * 17 + 2] = -1e3
    inv_diag, rc, _ = chol.solve_blocks(*to_upper_ccs(bad, pairs))
    assert rc == 1 and not inv_diag.any()
    out, rc, _ = chol.solve_pattern(*to_upper_ccs(bad, pairs), [(0, 39), (3, 4)])
    assert rc == 1 and not out.any()
    inv_diag, rc, _ = chol.solve_blocks(*to_upper_ccs(A, pairs))
    assert rc == 0
    check_diag(A, inv_diag)
    b = np.random.default_rng(13).standard_normal(6 * P)
    x, rc, _ = chol.solve(*to_upper_ccs(A, pairs), b)
    assert rc == 0
    assert np.abs(x - np.linalg.solve(A, b)).max() <= 1e-9 * np.abs(x).max()


def _raw_pattern(svs, chol, P, cp, ri, blocks, n, r, c, out):
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int))
    return svs.lib().svs_chol6_solve_pattern(chol._h, P, ptr(cp), ptr(ri), None if blocks is None else blocks.ctypes.data,
                                             n, ptr(r), ptr(c), None if out is None else out.ctypes.data, 0, None)


def test_malformed_requests_rejected_and_handle_survives(svs, chol):
    P = 20
    pairs = banded_pairs(P, 3, seed=26)
    A = random_spd(P, pairs, seed=27)
    cp, ri, blocks = to_upper_ccs(A, pairs)
    r, c = np.array([0, 3], np.int32), np.array([5, 19], np.int32)
    out = np.zeros((2, 36))
    assert _raw_pattern(svs, chol, P, cp, ri, blocks, 2, r, c, out) == 0
    cases = {
        "row -1": (P, cp, ri, blocks, 2, np.array([-1, 3], np.int32), c, out),
        "col P": (P, cp, ri, blocks, 2, r, np.array([5, P], np.int32), out),
        "n < 0": (P, cp, ri, blocks, -1, r, c, out),
        "null r": (P, cp, ri, blocks, 2, None, c, out),
        "null c": (P, cp, ri, blocks, 2, r, None, out),
        "null out": (P, cp, ri, blocks, 2, r, c, None),
        "null blocks": (P, cp, ri, None, 2, r, c, out),
    }
    for name, args in cases.items():
        assert _raw_pattern(svs, chol, *args) == SVS_ERR_INVALID, name
        assert svs.lib().svs_chol6_last_error(chol._h).decode(), name
    assert svs.lib().svs_chol6_solve_blocks(chol._h, P, cp.ctypes.data_as(C.POINTER(C.c_int)),
                                            ri.ctypes.data_as(C.POINTER(C.c_int)), blocks.ctypes.data, None, 0,
                                            None) == SVS_ERR_INVALID
    with pytest.raises(svs.SvsError):
        chol.solve_pattern(cp, ri, blocks, [(0, P)])
    out, rc, st = chol.solve_pattern(cp, ri, blocks, [(0, 5), (3, 19)])
    assert rc == 0 and st["symbolic_reused"] == 1
    check_blocks(np.linalg.inv(A), [(0, 5), (3, 19)], out)


# ---------------------------------------------------------------------------------------------- shared analysis

def test_solve_then_blocks_then_solve(chol):
    P = 80
    pairs = banded_pairs(P, 4, seed=17)
    A = random_spd(P, pairs, seed=20)
    b = np.random.default_rng(19).standard_normal(6 * P)
    cp, ri, blocks = to_upper_ccs(A, pairs)
    x0, rc, st = chol.solve(cp, ri, blocks, b)
    assert rc == 0 and st["symbolic_reused"] == 0
    inv_diag, rc, st = chol.solve_blocks(cp, ri, blocks)
    assert rc == 0 and st["symbolic_reused"] == 1
    check_diag(A, inv_diag)
    x1, rc, st = chol.solve(cp, ri, blocks, b)
    assert rc == 0 and st["symbolic_reused"] == 1
    assert np.array_equal(x0, x1)


def test_device_input_matches_host(chol):
    import torch
    P = 150
    A = random_spd(P, banded_pairs(P, 6, seed=23), seed=24)
    cp, ri, blocks = to_upper_ccs(A)
    req = [(0, 149), (10, 11), (7, 7), (120, 3)]
    d_h, rc_h, _ = chol.solve_blocks(cp, ri, blocks)
    o_h, ro_h, _ = chol.solve_pattern(cp, ri, blocks, req)
    d_d, rc_d, _ = chol.solve_blocks(cp, ri, torch.from_numpy(blocks).cuda())
    o_d, ro_d, _ = chol.solve_pattern(cp, ri, torch.from_numpy(blocks).cuda(), req)
    assert rc_h == rc_d == ro_h == ro_d == 0
    assert isinstance(d_d, torch.Tensor) and d_d.is_cuda and d_d.shape == (P, 6, 6)
    assert np.array_equal(d_h, d_d.cpu().numpy())
    assert np.array_equal(o_h, o_d.cpu().numpy())


# ---------------------------------------------------------------------------------------------- C++ adapter

def test_cpp_adapter_matches_python(chol, tmp_path):
    exe = str(tmp_path / "chol6_marginals_main")
    lib_dir = os.path.join(ROOT, "scavislam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "chol6_marginals_main.cpp"), "-o", exe,
                           "-L", lib_dir, "-lsvsb200", f"-Wl,-rpath,{lib_dir}"])
    P = 100
    A = random_spd(P, banded_pairs(P, 6, seed=29) + [(2, 90)], seed=30)
    cp, ri, blocks = to_upper_ccs(A)
    req = upper_pairs(cp, ri)[::3] + [(0, 99), (99, 0), (50, 10)]
    r = np.array([p[0] for p in req], np.int32)
    c = np.array([p[1] for p in req], np.int32)
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([P, len(ri)], np.int32).tofile(f)
        cp.tofile(f)
        ri.tofile(f)
        blocks.tofile(f)
        np.array([len(req)], np.int32).tofile(f)
        r.tofile(f)
        c.tofile(f)
    res = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "OK blocks=1 pattern=1" in res.stdout
    got = np.fromfile(tmp_path / "out.bin", np.float64).reshape(-1, 6, 6).swapaxes(1, 2)   # column-major blocks
    d_py, _, _ = chol.solve_blocks(cp, ri, blocks)
    o_py, _, _ = chol.solve_pattern(cp, ri, blocks, req)
    assert np.array_equal(got[:P], d_py)
    assert np.array_equal(got[P:], o_py)
