"""k_solve at the shapes where its launch changes: ring capacity and refill period next to the general-solver boundary,
backward passes of more than one round, hub rows, wide separators, breaks in the chain, a window too large for shared
memory, badly scaled and ill-conditioned systems, a failed pivot in each team, the marginals at the same shapes, and the
C5 window (1 000 keyframes, 100 000 landmarks) of the bench against the oracle.

Every system is an SPD block-sparse matrix kept in scipy.sparse.  The reference solution is scipy's sparse LU in FP64
refined twice with the residual b - A x in long double (block products over the CCS blocks); the dense inverse is
only formed up to 6P = 6 000.  Each case asserts the launch path it means to reach from a restatement of the host's
symbolic analysis (ba_host.cu: analyse, choose_branches, analyse_pattern) and of the shared-memory budget of k_solve
(ba_solve.cu: solve_fixed_bytes, solve_ring_capacity, solve_uses_chain_kernel, launch_solve, scatter_rows), checked
against the nnzb_L, nbranch and general the library reports."""
import os
from contextlib import contextmanager, nullcontext

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from scavislam_b200 import synth

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53
POSE_RTOL = 1e-6


# ---------------------------------------------------------------------------------------------- systems

def spd_system(P, pairs, seed, diag=1.0, relative=False):
    """6P x 6P SPD matrix (scipy CSR): a random J^T J (J 6 x 12) over every pose pair (i, j) of `pairs`, plus
    diag * I.  relative=True: J = [K, -K], a coupling that only sees the difference of the two poses (a window
    without its gauge fixed), so that diag sets the smallest eigenvalues."""
    rng = np.random.default_rng(seed)
    pr = np.asarray(pairs, np.int64).reshape(-1, 2)
    if relative:
        K = rng.standard_normal((len(pr), 6, 6))
        J = np.concatenate([K, -K], axis=2)
    else:
        J = rng.standard_normal((len(pr), 6, 12))
    M = np.einsum("nki,nkj->nij", J, J)                         # [n, 12, 12]
    idx = np.concatenate([6 * pr[:, :1] + np.arange(6), 6 * pr[:, 1:] + np.arange(6)], axis=1)   # [n, 12]
    rows = np.broadcast_to(idx[:, :, None], M.shape).ravel()
    cols = np.broadcast_to(idx[:, None, :], M.shape).ravel()
    A = sp.coo_matrix((M.ravel(), (rows, cols)), shape=(6 * P, 6 * P)).tocsr()
    return sym(A + diag * sp.identity(6 * P, format="csr"))


def sym(A):
    """(A + A^T) / 2: exactly symmetric (the duplicate sums above need not be)."""
    A = sp.csr_matrix(A)
    return ((A + A.T) * 0.5).tocsr()


def band(P, w, lo=0):
    """Every pair of poses of [lo, P) at most w apart: a full band, which the minimum-degree order keeps as it is."""
    return [(i, j) for i in range(lo, P) for j in range(i + 1, min(P, i + w + 1))]


def upper_ccs(A):
    """Upper block CCS of the symmetric sparse A: every block with a stored entry plus the diagonal, each block
    column-major.  Block row j of A's BSR holds A_ji = A_ij^T, whose row-major order is A_ij's column-major order."""
    P = A.shape[0] // 6
    B = sp.csr_matrix(A).tobsr(blocksize=(6, 6))
    B.sort_indices()
    cols = np.repeat(np.arange(P), np.diff(B.indptr))
    keep = B.indices <= cols                                    # block (i, j) with i <= j of column j
    row_idx = B.indices[keep].astype(np.int32)
    col_ptr = np.concatenate([[0], np.cumsum(np.bincount(cols[keep], minlength=P))]).astype(np.int32)
    blocks = np.ascontiguousarray(B.data[keep].reshape(-1, 36))
    return col_ptr, row_idx, blocks


def ccs_matvec(cp, ri, blocks, x, dtype=np.longdouble):
    """A x from the upper block CCS (the upper triangle of each diagonal block mirrored, as the library reads it), in
    `dtype`, vectorised over the blocks."""
    P = len(cp) - 1
    col = np.repeat(np.arange(P), np.diff(cp))
    Bm = blocks.reshape(-1, 6, 6).transpose(0, 2, 1).astype(dtype)   # row-major A_ij
    diag = ri == col
    up = np.triu(np.ones((6, 6), bool))
    Bd = np.where(up, Bm[diag], Bm[diag].transpose(0, 2, 1))          # symmetric from the upper triangle
    Bm[diag] = Bd
    X = np.asarray(x).astype(dtype).reshape(P, 6)
    y = np.zeros((P, 6), dtype)
    np.add.at(y, ri, np.einsum("nij,nj->ni", Bm, X[col]))
    off = ~diag
    np.add.at(y, col[off], np.einsum("nji,nj->ni", Bm[off], X[ri[off]]))
    return y.ravel()


def reference_solve(A, b, cp, ri, blocks):
    """splu in FP64, then two steps of iterative refinement with the residual in long double."""
    lu = spla.splu(A.tocsc())
    x = lu.solve(b)
    for _ in range(2):
        r = np.asarray(b, np.longdouble) - ccs_matvec(cp, ri, blocks, x)
        x = x + lu.solve(r.astype(np.float64))
    return x


def backward_error(A, b, x, cp, ri, blocks):
    """Normwise backward error ||b - A x||inf / (||A||inf ||x||inf + ||b||inf), in long double."""
    r = np.asarray(b, np.longdouble) - ccs_matvec(cp, ri, blocks, x)
    normA = np.longdouble(abs(A).sum(axis=1).max())
    return float(np.abs(r).max() / (normA * np.abs(x).max() + np.abs(b).max()))


# Bound on the normwise backward error.  A block Cholesky in FP64 is backward stable: the computed factor satisfies
# L L^T = A + dA with |dA| <= gamma_(n+1) |L| |L^T| (Higham, Accuracy and Stability, thm 10.3), and the two triangular
# solves add terms of the same form, so the normwise backward error is a modest multiple of n u with n = 6P and
# u = 2^-53.  The bound is 6P u itself, set from that argument and not from the data.  Measured on an H100 80GB HBM3 (400 W
# power limit) over every solve of this file: at most 5.2e-16 (about 5 u, the one-chain sweep at P = 300 and width
# 63), 2.6e-3 of the bound; the C5 reduced system 6.9e-17.
def be_bound(P):
    return 6 * P * EPS


def check_solve(A, b, x, rc, cp, ri, blocks, fwd_tol=1e-9, x_ref=None):
    assert rc == 0
    P = len(cp) - 1
    if x_ref is None:
        x_ref = reference_solve(A, b, cp, ri, blocks)
    be = backward_error(A, b, x, cp, ri, blocks)
    assert be <= be_bound(P), (be, be_bound(P))
    if fwd_tol is not None:
        assert np.abs(x - x_ref).max() <= fwd_tol * np.abs(x_ref).max()
    return be


# ---------------------------------------------------------------------------------------------- restated analysis

def pattern_of(cp, ri):
    """P x P boolean adjacency of the pose graph (no diagonal) from the upper block CCS."""
    P = len(cp) - 1
    col = np.repeat(np.arange(P), np.diff(cp))
    adj = np.zeros((P, P), bool)
    adj[ri, col] = True
    adj[col, ri] = True
    np.fill_diagonal(adj, False)
    return adj


def eliminate(adj, order=None):
    """ba_host.cu analyse: greedy minimum degree (ties to the lowest index) or the given order; returns the column
    widths (blocks below the diagonal), the row counts of the row-major index (rptr) and nblk."""
    P = adj.shape[0]
    G = adj.copy()
    deg = G.sum(axis=1).astype(np.int64)
    done = np.zeros(P, bool)
    pos = np.empty(P, np.int64)
    cols = []
    for step in range(P):
        v = int(np.argmin(np.where(done, np.int64(1) << 40, deg))) if order is None else int(order[step])
        done[v] = True
        pos[v] = step
        nb = np.flatnonzero(G[v] & ~done)
        cols.append(nb)
        deg[nb] -= 1
        G[nb, v] = False
        if len(nb) > 1:
            sub = G[np.ix_(nb, nb)]
            new = ~sub
            np.fill_diagonal(new, False)
            G[np.ix_(nb, nb)] = sub | new
            deg[nb] += new.sum(axis=1)
    width = np.array([len(c) for c in cols], np.int64)
    rows = np.concatenate([pos[c] for c in cols]) if width.sum() else np.zeros(0, np.int64)
    rcount = np.bincount(rows, minlength=P)
    return dict(width=width, rcount=rcount, nblk=int(P + width.sum()), pos=pos)


def choose_branches(adj):
    """ba_host.cu choose_branches: (order, branch_ptr) of the two-ended split, or None for one chain."""
    P = adj.shape[0]
    if P < 8:
        return None
    iu, ju = np.nonzero(np.triu(adj, 1))
    hist = np.bincount(ju - iu, minlength=P)
    w, longer = P - 1, 0
    while w > 0 and longer + hist[w] <= 24:
        longer += hist[w]
        w -= 1
    if w == 0 or (P - w) // 2 < 3 * w:
        return None
    left = (P - w) // 2
    side = lambda p: 0 if p < left else (1 if p >= left + w else 2)
    in_sep = np.zeros(P, bool)
    for i in range(P):
        for j in np.flatnonzero(adj[i]):
            if j - i > w and side(i) + side(j) == 1 and not in_sep[i] and not in_sep[j]:
                in_sep[j] = True
    b0 = [i for i in range(left) if not in_sep[i]]
    b1 = [i for i in range(P - 1, left + w - 1, -1) if not in_sep[i]]
    order = b0 + b1 + [i for i in range(P) if in_sep[i]] + list(range(left, left + w))
    return order, [0, len(b0), len(b0) + len(b1)]


def solve_fixed_bytes(P, nblk, nsep):
    y = (6 * P * 8 + 15) // 16 * 16
    meta = ((2 * (P + 1) + nblk) * 4 + P + 15) // 16 * 16
    return y + meta + nsep * 288


def solve_ring_capacity(P, nblk, nsep, optin):
    budget = optin - 2048 - 256                                  # kStaticSmem, and a margin
    fixed = solve_fixed_bytes(P, nblk, nsep)
    if fixed >= budget:
        return 0
    avail = (budget - fixed) // 288
    cap = 1
    while cap * 2 <= avail:
        cap *= 2
    return cap if cap <= avail else 0


def greedy_chunks(rcount, lo, hi, half):
    """scatter_rows: the chunks (whole rows, at most `half` blocks unless one row is longer) of rows [lo, hi)."""
    rptr = np.concatenate([[0], np.cumsum(rcount)])
    n, a = 0, hi
    while a > lo:
        b = a - 1
        while b > lo and rptr[a] - rptr[b - 1] <= half:
            b -= 1
        n += 1
        a = b
    return n


def restate(cp, ri, optin, chain_only=False):
    """What svs_chol6 decides for this pattern: nbranch, nnzb_L, general, and for the chain kernel the ring capacity,
    refill period and the backward chunk count of the longest scatter_rows range.  `rejected`: the numbers of a
    two-ended split that the analysis tried and turned down (else None)."""
    adj = pattern_of(cp, ri)
    P = adj.shape[0]
    split = None if chain_only else choose_branches(adj)
    r, rejected = None, None
    if split is not None:
        order, bptr = split
        r = eliminate(adj, order)
        sep0 = bptr[2]
        w = r["width"]
        mcb, mcs = int(w[:sep0].max(initial=0)), int(w[sep0:].max(initial=0))
        nsep = r["nblk"] - (sep0 + int(w[:sep0].sum()))           # blocks of the separator columns: nblk - col_ptr[sep0]
        cap = solve_ring_capacity(P, r["nblk"], nsep, optin)
        if not (cap >= 4 * (mcb + 1) and cap // 2 >= mcs + 2):
            split, rejected = None, dict(cap=cap, max_col_branch=mcb, max_col_sep=mcs, nsep=nsep)
    if split is None:
        r = eliminate(adj)
        sep0, bptr, nsep = P, [0, P], 0
        mcb, mcs = 0, int(r["width"].max(initial=0))
    G = len(bptr) - 1
    max_row = int(r["rcount"].max(initial=0))
    col_sep = max(mcs, max_row - 2)                              # adopt_structure: solve_col_sep
    cap = solve_ring_capacity(P, r["nblk"], nsep if G > 1 else 0, optin)
    widest = mcb if G > 1 else col_sep
    general = cap == 0 or cap < 4 * (widest + 1) or cap // 2 < col_sep + 2
    out = dict(P=P, nbranch=G, nnzb_L=r["nblk"], general=int(general), nsep=nsep, max_col_branch=mcb,
               max_col_sep=mcs, max_row=max_row, cap=cap, pos=r["pos"], sep0=sep0, branch_ptr=bptr, rejected=rejected)
    if not general:
        while G == 1 and cap // 2 >= r["nblk"] and cap // 2 >= 4 * (widest + 1):
            cap //= 2
        out["cap"] = cap
        out["period"] = min(64, max(1, cap // (widest + 1) - 3))
        ranges = [(0, P)] if G == 1 else [(bptr[0], bptr[1]), (bptr[1], bptr[2]), (bptr[2], P)]
        out["chunks"] = max(greedy_chunks(r["rcount"], lo, hi, cap // 2) for lo, hi in ranges)
    return out


def check_path(st, rs):
    """The library's choice equals the restatement's."""
    assert (st["nnzb_L"], st["nbranch"], st["general"]) == (rs["nnzb_L"], rs["nbranch"], rs["general"]), (st, rs)


# ---------------------------------------------------------------------------------------------- fixtures

@pytest.fixture(scope="module")
def optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@pytest.fixture
def chol(svs):
    h = svs.BlockCholesky6(device=0)
    yield h
    h.close()


@contextmanager
def one_chain():
    """SVS_SOLVE_CHAIN=1: the analysis never splits the window into two ends."""
    os.environ["SVS_SOLVE_CHAIN"] = "1"
    try:
        yield
    finally:
        del os.environ["SVS_SOLVE_CHAIN"]


def run_case(chol, optin, A, b, chain_only=False, fwd_tol=1e-9):
    cp, ri, blocks = upper_ccs(A)
    rs = restate(cp, ri, optin, chain_only)
    x, rc, st = chol.solve(cp, ri, blocks, b)
    check_path(st, rs)
    x_ref = reference_solve(A, b, cp, ri, blocks)
    check_solve(A, b, x, rc, cp, ri, blocks, fwd_tol, x_ref)
    return x, rs, x_ref


# ---------------------------------------------------------------------------------------------- 1. ring capacity / refill period

@pytest.mark.parametrize("chain_only", [False, True], ids=["two_ends", "one_chain"])
def test_band_width_sweep_across_the_general_boundary(svs, optin, chain_only):
    """P = 300, full bands of every width from 28 to 66.  The default analysis splits widths up to 30 into two ends
    (ring of 128 blocks, refill period 1) and turns the split down from 31 on (its ring would be 64 blocks, less than
    four branch columns).  As one chain, k_solve's ring (cap = 256 from width 60 on) holds four columns up to width 63,
    where the refill period is 1; k_solve_general takes width 64 on."""
    P = 300
    by_width = {}
    h = svs.BlockCholesky6(device=0)     # fresh: a handle that saw a pattern may keep its earlier split
    try:
        with (one_chain() if chain_only else nullcontext()):
            for w in range(28, 67):
                A = spd_system(P, band(P, w), seed=w)
                b = np.random.default_rng(w).standard_normal(6 * P)
                _, by_width[w], _ = run_case(h, optin, A, b, chain_only)
    finally:
        h.close()
    chain = [w for w, rs in by_width.items() if not rs["general"]]
    assert max(chain) == 63 and all(by_width[w]["general"] for w in range(64, 67))
    last = by_width[63]
    assert last["nbranch"] == 1 and last["cap"] == 256 and last["period"] == 1
    split = [w for w, rs in by_width.items() if rs["nbranch"] == 2]
    if chain_only:
        assert not split
    else:
        assert split == [28, 29, 30]
        assert by_width[30]["cap"] == 128 and by_width[30]["period"] == 1 and not by_width[30]["general"]
        rj = by_width[31]["rejected"]
        assert rj["cap"] < 4 * (rj["max_col_branch"] + 1)


# ---------------------------------------------------------------------------------------------- 2. backward pass in rounds

@pytest.mark.parametrize("P,w,cap", [(1000, 7, 256), (500, 26, 512)])
def test_backward_pass_of_more_than_one_round(svs, optin, P, w, cap):
    """One chain whose backward pass needs more than kMaxChunks = 48 chunks of cap / 2 blocks, and the same system
    as two ends (each branch with its own chunk count); both answers agree to 1e-12."""
    A = spd_system(P, band(P, w), seed=P + w)
    b = np.random.default_rng(P).standard_normal(6 * P)
    cp, ri, blocks = upper_ccs(A)
    x_ref = reference_solve(A, b, cp, ri, blocks)
    h = svs.BlockCholesky6(device=0)
    try:
        with one_chain():
            rs1 = restate(cp, ri, optin, chain_only=True)
            x1, rc1, st1 = h.solve(cp, ri, blocks, b)
    finally:
        h.close()
    check_path(st1, rs1)
    assert rs1["nbranch"] == 1 and not rs1["general"] and rs1["cap"] == cap
    # from the reported numbers alone: the off-diagonal blocks need more than 48 chunks of cap / 2
    assert (st1["nnzb_L"] - P) / (cap // 2) > 48 and rs1["chunks"] > 48
    check_solve(A, b, x1, rc1, cp, ri, blocks, x_ref=x_ref)
    h = svs.BlockCholesky6(device=0)
    try:
        rs2 = restate(cp, ri, optin)
        x2, rc2, st2 = h.solve(cp, ri, blocks, b)
    finally:
        h.close()
    check_path(st2, rs2)
    assert rs2["nbranch"] == 2 and not rs2["general"]
    check_solve(A, b, x2, rc2, cp, ri, blocks, x_ref=x_ref)
    assert np.abs(x1 - x2).max() <= 1e-12 * np.abs(x1).max()


# ---------------------------------------------------------------------------------------------- 3. hub rows

def hub_all(P, h, w=3):
    """A band plus one pose coupled to every other pose (an arrowhead)."""
    return band(P, w) + [(min(h, j), max(h, j)) for j in range(P) if j != h and abs(j - h) > w]


def hub_two(P, where, w=3):
    """A band plus loop closures from one pose to both ends: the middle pose (which the split puts in the separator)
    or pose 0 (which puts pose P - 1 there); either way one separator row fills across both branches."""
    if where == "middle":
        return band(P, w) + [(0, P // 2), (P // 2, P - 1)]
    return band(P, w) + [(0, P - 1)]


@pytest.mark.parametrize("where", ["middle", "end"])
def test_hub_coupled_to_every_pose(chol, optin, where):
    """max_row (the hub's row) decides solve_col_sep and, for one chain, the widest column: k_solve while
    4 (max_row - 1) <= cap, k_solve_general past it.  Too many long edges for the two-ended split."""
    seen = set()
    for P in range(128, 141, 2):
        h = P // 2 if where == "middle" else 0
        A = spd_system(P, hub_all(P, h), seed=P)
        b = np.random.default_rng(P).standard_normal(6 * P)
        _, rs, _ = run_case(chol, optin, A, b)
        assert rs["nbranch"] == 1 and rs["max_row"] - 2 > rs["max_col_sep"]
        seen.add(rs["general"])
    assert seen == {0, 1}


@pytest.mark.parametrize("where", ["middle", "end"])
def test_hub_row_across_both_branches(svs, optin, where):
    """Two ends whose separator holds a row spanning both branches: the analysis keeps the split (its test does not
    look at rows), and the launch goes to k_solve_general once max_row > cap / 2.  Also as one chain."""
    seen = set()
    for chain_only in (False, True):
        h = svs.BlockCholesky6(device=0)
        try:
            with (one_chain() if chain_only else nullcontext()):
                for P in range(248, 267, 2):
                    A = spd_system(P, hub_two(P, where), seed=P)
                    b = np.random.default_rng(P).standard_normal(6 * P)
                    _, rs, _ = run_case(h, optin, A, b, chain_only)
                    if not chain_only:
                        assert rs["nbranch"] == 2 and rs["max_row"] > rs["P"] - 20
                        seen.add(rs["general"])
        finally:
            h.close()
    assert seen == {0, 1}


# ---------------------------------------------------------------------------------------------- 4. separator width

def test_separator_widened_by_loop_closures(svs, optin):
    """A band of 12 over 400 poses plus k short loop closures across the middle: each pulls one pose into the
    separator and widens its columns, and the branch columns next to it by one as well.  The split holds up to
    k = 19 (ring of 128 blocks); at k = 20 its ring would be 64 blocks, too small for four branch columns and for the
    separator's widest column alike, and the analysis keeps one chain.  With and without the split."""
    P, w = 400, 12
    left = (P - w) // 2
    seen = set()
    for chain_only in (False, True):
        h = svs.BlockCholesky6(device=0)
        try:
            with (one_chain() if chain_only else nullcontext()):
                for k in range(12, 22):
                    A = spd_system(P, band(P, w) + [(left - 1 - i, left + w + i) for i in range(k)], seed=k)
                    b = np.random.default_rng(k).standard_normal(6 * P)
                    _, rs, _ = run_case(h, optin, A, b, chain_only)
                    assert not rs["general"]
                    if not chain_only:
                        seen.add(rs["nbranch"])
                        assert rs["nbranch"] == (2 if k < 20 else 1)
                        if rs["nbranch"] == 2:
                            assert rs["max_col_sep"] >= w - 1 + k
                        else:
                            rj = rs["rejected"]
                            assert rj["cap"] < 4 * (rj["max_col_branch"] + 1) and rj["cap"] // 2 < rj["max_col_sep"] + 2
        finally:
            h.close()
    assert seen == {1, 2}


def dense_separator(P, W):
    """A band of 3, a clique of the W middle poses (exactly where choose_branches puts the separator), and edges of
    length W spread over both ends, at least 25 and one column apart, so that the band-width estimate (which ignores
    the 24 longest edges) is W.  The separator's columns are W - 1 wide while the branch columns stay at 4."""
    left = (P - W) // 2
    starts = list(range(4, left - W - 4, W + 1)) + list(range(left + W + 4, P - W - 4, W + 1))
    assert len(starts) > 24
    return band(P, 3) + [(i, j) for i in range(left, left + W) for j in range(i + 1, left + W)] + [(i, i + W) for i in starts]


def test_separator_just_under_half_the_ring(svs, optin):
    """P = 900 with a dense separator of W = 24..31 poses: the separator term cap / 2 >= max_col_sep + 2 is the one
    that ends the split.  At W = 30 the ring is 64 blocks and max_col_sep = 29 sits just under cap / 2 - 2 = 30 while
    the branch columns are 4 wide; at W = 31 the analysis turns the split down on the separator term alone.  With and
    without the split."""
    P = 900
    by_w = {}
    for chain_only in (False, True):
        h = svs.BlockCholesky6(device=0)
        try:
            with (one_chain() if chain_only else nullcontext()):
                for W in range(24, 32):
                    A = spd_system(P, dense_separator(P, W), seed=W)
                    b = np.random.default_rng(W).standard_normal(6 * P)
                    _, rs, _ = run_case(h, optin, A, b, chain_only)
                    assert not rs["general"]
                    if not chain_only:
                        by_w[W] = rs
        finally:
            h.close()
    assert [W for W, rs in by_w.items() if rs["nbranch"] == 2] == list(range(24, 31))
    last = by_w[30]
    assert last["cap"] == 64 and last["max_col_branch"] <= 5
    assert last["cap"] // 2 - 2 - 2 <= last["max_col_sep"] <= last["cap"] // 2 - 2
    rj = by_w[31]["rejected"]
    assert rj["cap"] >= 4 * (rj["max_col_branch"] + 1) and rj["cap"] // 2 < rj["max_col_sep"] + 2


# ---------------------------------------------------------------------------------------------- 5. breaks in the chain

@pytest.mark.parametrize("pieces", [[(0, 147), (147, 300)], [(0, 60), (60, 130), (130, 220), (220, 300)]],
                         ids=["branch_without_link", "four_pieces"])
def test_disconnected_pieces(svs, optin, pieces):
    """Windows of disconnected banded pieces: a column without its successor row in the middle of a branch, and
    (first case) a branch with no link to the separator at all.  Two ends and one chain."""
    P, w = 300, 5
    pairs = [p for lo, hi in pieces for p in band(hi, w, lo)]
    A = spd_system(P, pairs, seed=len(pieces))
    b = np.random.default_rng(len(pieces)).standard_normal(6 * P)
    x2, rs, _ = run_case_fresh(svs, optin, A, b, False)
    assert rs["nbranch"] == 2 and not rs["general"]
    if len(pieces) == 2:   # branch 0 is the whole first piece: nothing of it reaches the separator
        adj = pattern_of(*upper_ccs(A)[:2])
        assert not adj[:147, 147:].any() and rs["branch_ptr"][1] == 147
    x1, rs1, _ = run_case_fresh(svs, optin, A, b, True)
    assert rs1["nbranch"] == 1 and not rs1["general"]
    assert np.abs(x1 - x2).max() <= 1e-12 * np.abs(x1).max()


def run_case_fresh(svs, optin, A, b, chain_only):
    h = svs.BlockCholesky6(device=0)
    try:
        with (one_chain() if chain_only else nullcontext()):
            return run_case(h, optin, A, b, chain_only)
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------- 6. general solver, large

def test_large_window_on_the_general_solver(chol, optin):
    """P = 3 000 with a band of 4: the fixed part of k_solve's shared memory (y, indices) leaves no ring (cap = 0)."""
    P = 3000
    A = spd_system(P, band(P, 4), seed=6)
    b = np.random.default_rng(6).standard_normal(6 * P)
    cp, ri, _ = upper_ccs(A)
    assert solve_ring_capacity(P, restate(cp, ri, optin)["nnzb_L"], 0, optin) == 0
    _, rs, _ = run_case(chol, optin, A, b)
    assert rs["general"] == 1 and rs["cap"] == 0


# ---------------------------------------------------------------------------------------------- 7. scale and conditioning

@pytest.mark.parametrize("chain_only", [False, True], ids=["two_ends", "one_chain"])
def test_badly_scaled_components(svs, optin, chain_only):
    """D A D with each of the 6P components scaled by a power of ten in [1e-4, 1e4] (rotations against translations
    in other units): pivots from 1e-8 to 1e8 through rsqrt.approx.ftz and its one correction step.  Cholesky is
    insensitive to such a scaling, so D y must match the solution of the unscaled system."""
    P = 200
    A0 = spd_system(P, band(P, 8), seed=71)
    b0 = np.random.default_rng(71).standard_normal(6 * P)
    cp0, ri0, bl0 = upper_ccs(A0)
    x0 = reference_solve(A0, b0, cp0, ri0, bl0)
    d = 10.0 ** np.random.default_rng(72).integers(-4, 5, 6 * P)
    Dm = sp.diags(d)
    A = sym(Dm @ A0 @ Dm)
    b = d * b0
    cp, ri, blocks = upper_ccs(A)
    rs = restate(cp, ri, optin, chain_only)
    h = svs.BlockCholesky6(device=0)
    try:
        with (one_chain() if chain_only else nullcontext()):
            y, rc, st = h.solve(cp, ri, blocks, b)
    finally:
        h.close()
    check_path(st, rs)
    assert rs["nbranch"] == (1 if chain_only else 2)
    # the normwise backward error is dominated by the 1e8 entries here (measured 4e-24 on an H100); the bar is D y
    # (measured 6.6e-16 relative)
    check_solve(A, b, y, rc, cp, ri, blocks, fwd_tol=None)
    assert np.abs(d * y - x0).max() <= 1e-9 * np.abs(x0).max()


def test_ill_conditioned_window(chol, optin):
    """A window whose couplings only see pose differences (gauge not fixed), damped by lambda = 1e-10 of its largest
    eigenvalue: condition number about 1e10, as BA windows with a small lambda reach."""
    P = 200
    A0 = spd_system(P, band(P, 8), seed=73, diag=0.0, relative=True)
    ev = np.linalg.eigvalsh(A0.toarray())
    A = sym(A0 + (ev[-1] * 1e-10) * sp.identity(6 * P))
    ev = np.linalg.eigvalsh(A.toarray())
    cond = ev[-1] / ev[0]
    assert 3e9 < cond < 3e10
    b = np.random.default_rng(74).standard_normal(6 * P)
    x, rs, x_ref = run_case(chol, optin, A, b, fwd_tol=None)
    assert rs["nbranch"] == 2 and not rs["general"]
    # first-order perturbation bound: relative forward error <= 2 cond * (normwise backward error).  Measured on an
    # H100: forward error 1.9e-7 (backward error 1.7e-16), against a bound of about 2.7e-3
    assert np.abs(x - x_ref).max() <= 2 * cond * be_bound(P) * np.abs(x_ref).max()


# ---------------------------------------------------------------------------------------------- 8. not positive definite

def _npd_case(kind):
    """(A, P): a banded window of 200 poses, or an arrowhead of 140 that only k_solve_general takes."""
    if kind == "general":
        P = 140
        return spd_system(P, hub_all(P, P // 2), seed=81), P
    P = 200
    return spd_system(P, band(P, 8), seed=82), P


@pytest.mark.parametrize("kind", ["two_ends", "one_chain", "general"])
def test_not_positive_definite_in_each_team(svs, optin, kind):
    """A negative diagonal entry in pose 0, pose P - 1 or the middle pose: for two ends these fail in CTA 0's branch,
    CTA 1's branch and the separator.  Each solve returns 1 with x = 0, and the handle then solves a good system."""
    A, P = _npd_case(kind)
    b = np.random.default_rng(83).standard_normal(6 * P)
    cp, ri, blocks = upper_ccs(A)
    rs = restate(cp, ri, optin, kind == "one_chain")
    assert (rs["nbranch"], rs["general"]) == {"two_ends": (2, 0), "one_chain": (1, 0), "general": (1, 1)}[kind]
    if kind == "two_ends":   # elimination positions: branch 0, branch 1, separator
        bp = rs["branch_ptr"]
        assert rs["pos"][0] < bp[1] and bp[1] <= rs["pos"][P - 1] < bp[2] and rs["pos"][P // 2] >= bp[2]
    x_ref = reference_solve(A, b, cp, ri, blocks)
    h = svs.BlockCholesky6(device=0)
    try:
        with (one_chain() if kind == "one_chain" else nullcontext()):
            for pose in (0, P - 1, P // 2):
                bad = A.tolil()
                bad[6 * pose + 2, 6 * pose + 2] = -1e3
                bcp, bri, bbl = upper_ccs(bad.tocsr())
                assert np.array_equal(bcp, cp) and np.array_equal(bri, ri)
                x, rc, st = h.solve(bcp, bri, bbl, b)
                assert rc == 1 and not x.any(), pose
                check_path(st, rs)
                x, rc, st = h.solve(cp, ri, blocks, b)
                check_solve(A, b, x, rc, cp, ri, blocks, x_ref=x_ref)
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------- 9. marginals

def _diag_blocks(Z, P):
    return np.array([Z[6 * p:6 * p + 6, 6 * p:6 * p + 6] for p in range(P)])


def test_marginals_backward_pass_in_rounds(svs, optin):
    """solve_blocks (k_solve's kDiag instance, then the selected inversion) at P = 1 000, cap = 256, as two ends and
    as one chain, against the dense inverse; solve_pattern with pairs far outside the factor's pattern."""
    P = 1000
    A = spd_system(P, band(P, 7), seed=91)
    cp, ri, blocks = upper_ccs(A)
    Z = np.linalg.inv(A.toarray())
    ref = _diag_blocks(Z, P)
    far = [(0, 999), (999, 0), (3, 500), (500, 3), (250, 750), (498, 502), (12, 12)]
    for chain_only in (False, True):
        rs = restate(cp, ri, optin, chain_only)
        assert rs["nbranch"] == (1 if chain_only else 2) and not rs["general"] and rs["cap"] == 256
        h = svs.BlockCholesky6(device=0)
        try:
            with (one_chain() if chain_only else nullcontext()):
                inv_diag, rc, st = h.solve_blocks(cp, ri, blocks)
                assert rc == 0 and (st["nbranch"], st["general"], st["nnzb_L"]) == (rs["nbranch"], 0, rs["nnzb_L"])
                assert np.abs(inv_diag - ref).max() <= 1e-9 * np.abs(ref).max()
                if chain_only:
                    out, rc, st = h.solve_pattern(cp, ri, blocks, far)
                    assert rc == 0 and st["n_cols_solved"] > 0
                    fr = np.array([Z[6 * r:6 * r + 6, 6 * c:6 * c + 6] for r, c in far])
                    assert np.abs(out - fr).max() <= 1e-9 * np.abs(Z).max()
        finally:
            h.close()


@pytest.mark.parametrize("case", ["hub_all", "hub_two"])
def test_marginals_with_a_hub_row(chol, optin, case):
    P, pairs = (134, hub_all(134, 67)) if case == "hub_all" else (252, hub_two(252, "middle"))
    A = spd_system(P, pairs, seed=92)
    cp, ri, blocks = upper_ccs(A)
    rs = restate(cp, ri, optin)
    assert not rs["general"] and rs["nbranch"] == (1 if case == "hub_all" else 2)
    inv_diag, rc, st = chol.solve_blocks(cp, ri, blocks)
    assert rc == 0 and (st["nbranch"], st["general"], st["nnzb_L"]) == (rs["nbranch"], 0, rs["nnzb_L"])
    ref = _diag_blocks(np.linalg.inv(A.toarray()), P)
    assert np.abs(inv_diag - ref).max() <= 1e-9 * np.abs(ref).max()


# ---------------------------------------------------------------------------------------------- C5 through the BA handle

def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture(scope="module")
def c5():
    return synth.make_config("C5")


def test_c5_optimize_matches_oracle(svs, oracle, optin, c5):
    """BASELINE config C5 (1 000 keyframes, 100 000 landmarks), 10 iterations: the overlapped build + solve of the
    bench at cap = 256."""
    ba = svs.BundleAdjuster(device=0)
    try:
        ba.set_problem(c5)
        it, st = ba.optimize(10)
        poses, points = ba.poses(), ba.points()
    finally:
        ba.close()
    po, pso, sto = oracle.optimize(c5, 10)
    # the handle's own factor has the size the restated analysis of the oracle's reduced system gives
    So, _, _ = oracle.reduced_system(c5, True, 1.0, 50.0)
    cp, ri, _ = upper_ccs(sym(sp.csr_matrix(So)))
    rs = restate(cp, ri, optin)
    assert st["nnzb_L"] == rs["nnzb_L"] and rs["nbranch"] == 2 and not rs["general"] and rs["cap"] == 256
    assert it == sto["iterations"] == 10
    assert st["trials_iter"] == sto["trials_iter"] and st["trials_total"] == sto["trials_total"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    assert _rel(poses, po) < POSE_RTOL
    assert _rel(points, pso) < POSE_RTOL
    assert all(a >= b for a, b in zip([st["chi2_init"]] + st["chi2_iter"][:-1], st["chi2_iter"]))


def test_c5_reduced_system_and_solve(svs, oracle, optin, c5):
    """The reduced system at lambda = 50 against the oracle, and its solve against the sparse reference, as two ends
    and as one chain (whose backward pass runs in two rounds)."""
    ba = svs.BundleAdjuster(device=0)
    try:
        ba.set_problem(c5)
        S, bs, chi = ba.reduced_system(True, 1.0, 50.0)
        x2, rc2 = ba.solve_reduced(True, 1.0, 50.0)
        cst2 = ba.covariance(True, 1.0, 50.0)[4]     # (its stats name the handle's factor and solver)
    finally:
        ba.close()
    So, bso, chio = oracle.reduced_system(c5, True, 1.0, 50.0)
    assert abs(chi - chio) <= 1e-11 * abs(chio)
    assert _rel(S, So) < 1e-11
    assert _rel(bs, bso) < 1e-10
    A = sym(sp.csr_matrix(S))
    cp, ri, blocks = upper_ccs(A)
    x_ref = reference_solve(A, bs, cp, ri, blocks)
    rs2 = restate(cp, ri, optin)
    assert rs2["nbranch"] == 2 and not rs2["general"] and rs2["cap"] == 256
    check_path(cst2, rs2)
    check_solve(A, bs, x2, rc2, cp, ri, blocks, x_ref=x_ref)
    rs1 = restate(cp, ri, optin, chain_only=True)
    assert rs1["nbranch"] == 1 and not rs1["general"] and rs1["cap"] == 256
    assert (rs1["nnzb_L"] - 1000) / 128 > 48 and rs1["chunks"] > 48
    with one_chain():
        ba = svs.BundleAdjuster(device=0)
        try:
            ba.set_problem(c5)
            x1, rc1 = ba.solve_reduced(True, 1.0, 50.0)
            cst1 = ba.covariance(True, 1.0, 50.0)[4]
        finally:
            ba.close()
    check_path(cst1, rs1)
    check_solve(A, bs, x1, rc1, cp, ri, blocks, x_ref=x_ref)
    assert np.abs(x1 - x2).max() <= 1e-12 * np.abs(x2).max()
