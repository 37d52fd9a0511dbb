"""svs_ba_optimize's chained trials (programmatic dependent launch, DESIGN.md 5): the statistics the kernels stamp
themselves, and trials enqueued past the end of a call that terminates early."""
import numpy as np
import pytest

from scavislam_b200 import synth

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture(scope="module")
def ba(svs):
    b = svs.BundleAdjuster()
    yield b
    b.close()


def test_c2_kernel_times_come_from_the_kernels(ba):
    ba.set_problem(synth.make_config("C2"))
    ba.optimize(10)
    ba.reset_state()
    it, st = ba.optimize(10)
    assert it == 10 and st["launches"] == 3 * st["trials_total"]
    assert st["ms_build"] > 0 and st["ms_solve"] > 0 and st["ms_update"] > 0 and st["ms_control"] == 0
    # the kernels run one after the other: their durations fit into the call's device time
    assert st["ms_build"] + st["ms_solve"] + st["ms_update"] < st["ms_total"], st


def test_terminate_before_num_iters(ba, oracle):
    """max_trials = 1 ends the call after the first of ten iterations: the nine chained trials behind it return at once,
    and the next call on the handle starts clean."""
    pb = synth.make_window(40, 2000, seed=7)
    ba.set_problem(pb)
    it, st = ba.optimize(10, True, 1.0, 50.0, 1)
    po_, ps_, sto = oracle.optimize(pb, 10, True, 1.0, 50.0, 1)
    assert it == sto["iterations"] == 1 and st["trials_iter"] == sto["trials_iter"]
    np.testing.assert_allclose(st["chi2_iter"], sto["chi2_iter"], rtol=1e-7)
    assert _rel(ba.poses(), po_) < 1e-6 and _rel(ba.points(), ps_) < 1e-6
    ba.reset_state()
    it2, st2 = ba.optimize(10, True, 1.0, 50.0, 1)
    assert it2 == 1
    np.testing.assert_allclose(st2["chi2_iter"], st["chi2_iter"], rtol=1e-12)
