"""k_solve's N warps: the folded factor N_ij = L_ij L_jj^-1 that the backward pass streams back is formed beside the row
warps' right-hand side and written to the row-major position of each block.  Columns narrower and wider than the N warps
(64 threads, 6 rows per block: more than ten sub-diagonal blocks take a second round), one handle solving systems of
different structure one after the other, against numpy on the dense matrix."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def banded_spd(P, w, seed):
    """SPD matrix whose columns carry w sub-diagonal blocks: J^T J over every pose pair (i, i + k), k <= w, plus I."""
    rng = np.random.default_rng(seed)
    A = np.zeros((6 * P, 6 * P))
    for i in range(P):
        for j in range(i + 1, min(P, i + w + 1)):
            idx = np.r_[6 * i:6 * i + 6, 6 * j:6 * j + 6]
            J = rng.standard_normal((6, 12))
            A[np.ix_(idx, idx)] += J.T @ J
    A += np.eye(6 * P)
    return A


def upper_ccs(A):
    P = A.shape[0] // 6
    nz = np.abs(A.reshape(P, 6, P, 6)).max(axis=(1, 3)) > 0
    col_ptr, row_idx, blocks = [0], [], []
    for j in range(P):
        for i in range(j + 1):
            if i == j or nz[i, j]:
                row_idx.append(i)
                blocks.append(A[6 * i:6 * i + 6, 6 * j:6 * j + 6].ravel(order="F"))
        col_ptr.append(len(row_idx))
    return np.array(col_ptr, np.int32), np.array(row_idx, np.int32), np.array(blocks, np.float64).reshape(-1, 36)


def solve_and_check(chol, A, seed):
    b = np.random.default_rng(seed).standard_normal(A.shape[0])
    x, rc, st = chol.solve(*upper_ccs(A), b)
    assert rc == 0
    x_ref = np.linalg.solve(A, b)
    assert np.abs(x - x_ref).max() <= 1e-9 * np.abs(x_ref).max()
    assert np.linalg.norm(A @ x - b) <= 1e-10 * np.linalg.norm(b)
    assert st["general"] == 0   # the chain kernel, not the global-memory one
    return st


@pytest.fixture
def chol(svs):
    h = svs.BlockCholesky6(device=0)
    yield h
    h.close()


@pytest.mark.parametrize("P, w", [(9, 3), (60, 7), (120, 10), (120, 11), (160, 14)])
def test_column_widths_around_the_row_warps(chol, P, w):
    st = solve_and_check(chol, banded_spd(P, w, seed=P + w), seed=w)
    assert st["P"] == P


def test_one_handle_alternating_structures(chol):
    # every solve re-analyses (a different pattern), so the row positions the N warps fetch change between calls
    wide, narrow = banded_spd(100, 12, seed=1), banded_spd(100, 3, seed=2)
    for A, seed in ((wide, 3), (narrow, 4), (wide, 5), (narrow, 6)):
        solve_and_check(chol, A, seed)
