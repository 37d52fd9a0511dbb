"""Golden fixture of tests/test_solve_tail_gpu.py (GPU box): the bits of svs_chol6_solve's x on C2's and C5's reduced
camera systems.

The systems are the oracle's reduced systems at lambda = 50 (robust, delta 1), which the sequential C oracle computes
the same way on every run; their SHA-256 is stored beside x, so the test can tell a changed input from a changed solve.
Usage: python scripts/make_golden_solve_tail.py [out.npz]"""
import hashlib
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle import pyoracle
from scavislam_b200 import capi, synth

CONFIGS = ("C2", "C5")


def upper_ccs(S):
    """The upper block CCS g2o's fillCCS(..., upperTriangle = true) gives for a dense symmetric S."""
    P = S.shape[0] // 6
    nz = np.abs(S.reshape(P, 6, P, 6)).max(axis=(1, 3)) > 0
    col_ptr, row_idx, blocks = [0], [], []
    for j in range(P):
        rows = [i for i in np.nonzero(nz[:j + 1, j])[0]]
        if not rows or rows[-1] != j:
            rows.append(j)
        for i in rows:
            row_idx.append(i)
            blocks.append(S[6 * i:6 * i + 6, 6 * j:6 * j + 6].ravel(order="F"))
        col_ptr.append(len(row_idx))
    return np.array(col_ptr, np.int32), np.array(row_idx, np.int32), np.ascontiguousarray(np.array(blocks).reshape(-1, 36))


def system(name):
    """(cp, ri, blocks, b, sha256 of the dense system and right-hand side)."""
    S, b, _ = pyoracle.reduced_system(synth.make_config(name), True, 1.0, 50.0)
    h = hashlib.sha256(np.ascontiguousarray(S).tobytes())
    h.update(np.ascontiguousarray(b).tobytes())
    return (*upper_ccs(S), b, h.hexdigest())


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                             "tests", "golden", "solve_tail_golden.npz")
    chol = capi.BlockCholesky6(device=0)
    arrays = {}
    for name in CONFIGS:
        cp, ri, blocks, b, sha = system(name)
        x, rc, st = chol.solve(cp, ri, blocks, b)
        assert rc == 0 and st["nbranch"] == 2 and not st["general"], (rc, st)
        arrays[f"{name}_x_bits"] = np.ascontiguousarray(x).view(np.uint64)
        arrays[f"{name}_sha256"] = np.array(sha)
        print(name, "P", len(cp) - 1, "blocks", len(ri), "nnzb_L", st["nnzb_L"], "sha256", sha)
    chol.close()
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()
