"""k_solve's backward pass and pose-update tail leave the solution's bits alone: svs_chol6_solve on C2's and C5's reduced
camera systems (two-ended, on the chain kernel) returns exactly the x of the fixture, which an earlier build of the
library produced (scripts/make_golden_solve_tail.py).  The factor and the backward sums run in an order fixed by the
structure and k_solve uses no atomics, so any difference in x is a change of the arithmetic, not rounding."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import make_golden_solve_tail as gen  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "solve_tail_golden.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", gen.CONFIGS)
def test_solution_bits_unchanged(svs, oracle, golden, name):
    cp, ri, blocks, b, sha = gen.system(name)
    assert sha == str(golden[f"{name}_sha256"]), "the oracle's reduced system is not the one the fixture was made from"
    chol = svs.BlockCholesky6(device=0)
    try:
        x, rc, st = chol.solve(cp, ri, blocks, b)
    finally:
        chol.close()
    assert rc == 0 and st["nbranch"] == 2 and not st["general"], (rc, st)
    bits = np.ascontiguousarray(x).view(np.uint64)
    want = golden[f"{name}_x_bits"]
    diff = np.nonzero(bits != want)[0]
    assert diff.size == 0, (f"{diff.size} of {bits.size} elements differ, first at {diff[:8]}, "
                            f"max |dx| {np.abs(x - want.view(np.float64)).max():.3e}")
