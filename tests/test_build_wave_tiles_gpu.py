"""k_build_wave's tensor-core tiles at the shapes where they are padded, against the long-double reference of
tests/build_reference.py (the bars and both set-ups of test_build_shapes_gpu._check).

The task's 6K x 6K block is covered by 8 x 8 tiles, so at K = 1, 3, 5, 7 the last tile has columns past 6K; the
k-dimension of a wave is 3 nw rows per slot and for the Schur term, padded to a multiple of 4.  Each window holds
tasks of 1, nw_max and nw_max + 1 landmarks (the last wave of the latter has one landmark: 3 rows and one padding row,
after a full wave has left its rows in the warp's shared memory) and of 2 nw_max + 3, with and without a self edge,
with the self edge's anchor term kept and skipped."""
import pytest

import build_reference as br
from test_build_shapes_gpu import _check, _shape_track

pytestmark = pytest.mark.gpu

CASES = [(K, s, skip) for K in (1, 3, 5, 7) for s in ((True,) if K == 1 else (True, False)) for skip in (False, True)]


@pytest.mark.parametrize("K,self_edge,skip_self", CASES,
                         ids=[f"K{K}-{'self' if s else 'anchorless'}{'-skip_self' if sk else ''}" for K, s, sk in CASES])
def test_wave_tile_padding(svs, oracle, monkeypatch, K, self_edge, skip_self):
    monkeypatch.setenv("SVS_BUILD_CHUNK", "32")
    k = K if self_edge else K - 1
    nw = br.nw_max(k, K)
    counts = [1, nw, nw + 1, 2 * nw + 3]
    assert any(3 * (c % nw) % 4 for c in counts)   # a wave whose k-dimension is not a multiple of 4
    pb = br.make_tracks_window(40, [_shape_track(8 * i, K, self_edge, c) for i, c in enumerate(counts)], seed=20 + K, C=3)
    flags = svs.SVS_BA_SKIP_SELF_ANCHOR_HESSIAN if skip_self else 0
    rt, _ = _check(svs, oracle, pb, flags=flags)
    assert not rt.gen and not rt.long
    assert sorted(rt.task_shape(t) for t in range(len(rt.tasks))) == sorted((k, K, self_edge, c) for c in counts)
