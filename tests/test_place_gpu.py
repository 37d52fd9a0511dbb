"""svs_place (csrc/place.cu) against the place-recognition oracle: words, scores, the candidate, matches and
distances bit-equal, the same hypotheses and inliers, T to 1e-9 -- over a sequence with revisits and at the shapes
where k_place_nn changes its launch."""
import numpy as np
import pytest

from oracle import place_pyoracle as pp
from scavislam_b200 import capi, synth_place as sp

pytestmark = pytest.mark.gpu
TILE = 64


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def nn_grid(n, m, sms):
    """Restatement of csrc/place.cu nn_grid: query blocks of 64 rows; the train tiles split over about two waves."""
    qb, tiles = -(-n // TILE), -(-m // TILE)
    return qb, max(1, min(tiles, -(-2 * sms // qb)))


def _residual(T, xyz, obs):
    """max |obs - map_uvu(T xyz)| over the three components (belowThreshold compares each with pixel_thr)."""
    P = sp.se3_apply(T, xyz[None])
    return np.abs(obs - sp.map_uvu(P)[0]).max()


def _unmap(uvu):
    f, px, py, b = sp.CAM
    z = f / ((uvu[0] - uvu[2]) / b)
    return np.array([(uvu[0] - px) / f * z, (uvu[1] - py) / f * z, z])


def _check(g, o, kid, desc, uvu, **kw):
    rg = g.add_location(kid, desc, uvu, **kw)
    ro = o.add_location(kid, desc, uvu, **kw)
    if not hasattr(o, "stored_uvu"):
        o.stored_uvu = {}
    o.stored_uvu[kid] = np.asarray(uvu, np.float64).reshape(-1, 3)
    n = len(desc)
    wg = g.last_words()
    assert wg.tobytes() == ro["words"].tobytes()
    ids, sc = g.last_scores()
    assert ids.tolist() == ro["score_ids"].tolist() and sc.tobytes() == ro["scores"].tobytes()
    assert rg["best_keyframe_id"] == ro["best_keyframe_id"]
    assert np.float32(rg["best_score"]).tobytes() == np.float32(ro["best_score"]).tobytes()
    tg, dg = g.last_matches()
    assert rg["num_matches"] == ro["num_matches"] == len(tg)
    assert tg.tolist() == ro["train_idx"].tolist() and dg.tobytes() == ro["dist"].tobytes()
    tri, inl, best = g.last_hypotheses()
    assert tri.tolist() == ro["hyp_triple"].tolist() and inl.tolist() == ro["hyp_inliers"].tolist()
    assert best == ro["best_hypothesis"]
    np.testing.assert_allclose(rg["T_query_from_loop"], ro["T_query_from_loop"], rtol=0, atol=1e-9)
    a, b = set(rg["inlier_query"].tolist()), set(ro["inlier_query"].tolist())
    if a != b:   # only a residual at the threshold may decide differently
        train_uvu = o.stored_uvu[ro["best_keyframe_id"]]
        for r in sorted(a ^ b):
            res = _residual(ro["T_query_from_loop"], _unmap(train_uvu[ro["train_idx"][r]]), uvu[r])
            print(f"keyframe {kid}: inlier decision differs at row {r}: residual {res!r}")
            assert abs(res - kw.get("pixel_thr", 2.5)) < 1e-6
    else:
        assert rg["inlier_train"].tolist() == ro["inlier_train"].tolist()
    assert rg["num_inliers"] == ro["num_inliers"] and rg["loop_found"] == ro["loop_found"]
    assert g.num_places == o.num_places
    assert rg["ms"] > 0
    return rg, ro


def _pair(g, o, m, W, seed, dummies=5):
    """Stores `dummies` unrelated places and a place of m rows (0..dummies); returns its points, words and rows."""
    rng = np.random.default_rng(seed)
    words = o.words
    for d in range(dummies):
        k = 12
        w = words[W - 1 - (d * k + np.arange(k)) % max(W // 2, 1)]
        uvu = np.tile([320.0, 240.0, 300.0], (k, 1))
        _check(g, o, 1000 + d, w + rng.normal(size=w.shape).astype(np.float32) * 0.01, uvu)
    z = rng.uniform(2, 8, m)
    u, v = rng.uniform(40, 600, m), rng.uniform(40, 440, m)
    f, px, py, b = sp.CAM
    X = np.stack([(u - px) / f * z, (v - py) / f * z, z], 1)
    wid = np.arange(m) % max(W // 2, 1)
    desc = (words[wid] + rng.normal(size=(m, 64)) * 0.01).astype(np.float32)
    _check(g, o, 0, desc, sp.map_uvu(X))
    return X, wid, desc


def _query(X, desc, n, T, seed):
    rng = np.random.default_rng(seed + 1)
    rows = np.arange(n) % len(X)
    uvu = sp.map_uvu(sp.se3_apply(T, X[rows])) + rng.normal(size=(n, 3)) * 0.2
    q = (desc[rows] + rng.normal(size=(n, 64)) * 0.01).astype(np.float32)
    return q, uvu


T_TRUE = np.array([0.01, -0.02, 0.015, 0.9996, 0.1, -0.05, 0.2])
T_TRUE[:4] /= np.linalg.norm(T_TRUE[:4])


@pytest.fixture(scope="module")
def seq():
    return sp.make_sequence(num_keyframes=60, num_scenes=40, seed=11)


def _run_sequence(words, kfs):
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    out = []
    for k in kfs:
        excl = [k["id"] - 1] if k["id"] else []
        rg, ro = _check(g, o, k["id"], k["desc"], k["uvu"], exclude=excl, seed=k["id"])
        out.append(rg)
    return out


def test_sequence_matches_oracle_and_repeats(seq):
    words, kfs = seq
    a = _run_sequence(words, kfs)
    assert sum(r["loop_found"] for r in a) >= 8
    b = _run_sequence(words, kfs)          # a fresh handle gives the same bits
    for x, y in zip(a, b):
        assert x["T_query_from_loop"].tobytes() == y["T_query_from_loop"].tobytes()
        assert x["inlier_query"].tolist() == y["inlier_query"].tolist()


@pytest.mark.parametrize("n", [0, 1, 2, 3])
def test_tiny_queries(n):
    W = 200
    words = sp.make_vocabulary(W, seed=n)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, 3, W, seed=n, dummies=1)
    q, uvu = _query(X, desc, n, T_TRUE, n)
    _check(g, o, 7, q, uvu)


SHAPE_W = 2048
SHAPES = [(n, m) for n in (63, 64, 65) for m in (63, 64, 65)] + [(128, 64), (129, 64), (512, 2000), (513, 2000),
                                                                (2112, 130)]


def test_shapes_reach_every_launch_path():
    """From the launch arithmetic: the cases take one and several query blocks, a full and a partial last train tile,
    and splits of the train tiles bounded by the tile count and by the two-wave target, for the word search (n x W)
    and for the match (n x m)."""
    sms = _sms()
    seen = set()
    for n, m in SHAPES:
        for what, cols in (("words", SHAPE_W), ("match", max(m, 12))):
            qb, S = nn_grid(n, cols, sms)
            tiles = -(-cols // TILE)
            seen.add((what, "qb>1" if qb > 1 else "qb=1"))
            seen.add((what, "split=tiles" if S == tiles else "split=waves"))
        seen.add(("match", "partial tile" if m % TILE else "full tile"))
    for what in ("words", "match"):
        for path in ("qb>1", "qb=1", "split=tiles", "split=waves"):
            assert (what, path) in seen, (what, path)
    assert ("match", "partial tile") in seen and ("match", "full tile") in seen


@pytest.mark.parametrize("n,m", SHAPES)
def test_launch_shapes(n, m):
    W = SHAPE_W
    words = sp.make_vocabulary(W, seed=n + m)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, m, W, seed=n * 7 + m)
    q, uvu = _query(X, desc, n, T_TRUE, n)
    rg, _ = _check(g, o, 9, q, uvu)
    assert rg["best_keyframe_id"] == 0 and rg["num_matches"] == n


def test_vocabulary_10000_query_1500():
    W, n = 10000, 1500
    words = sp.make_vocabulary(W, seed=4)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, 1000, W, seed=4)
    q, uvu = _query(X, desc, n, T_TRUE, 4)
    rg, _ = _check(g, o, 9, q, uvu)
    assert rg["loop_found"]


def test_database_of_2000_places():
    W = 600
    words = sp.make_vocabulary(W, seed=8)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    rng = np.random.default_rng(8)
    for k in range(2000):
        n = 12
        wid = rng.integers(0, W, n)
        desc = (words[wid] + rng.normal(size=(n, 64)) * 0.02).astype(np.float32)
        uvu = np.stack([rng.uniform(0, 640, n), rng.uniform(0, 480, n)], 1)
        uvu = np.concatenate([uvu, uvu[:, :1] - rng.uniform(2, 40, (n, 1))], 1)
        if k % 97 == 0 or k > 1990:
            _check(g, o, k, desc, uvu, num_ransac=20)
        else:
            g.add_location(k, desc, uvu, num_ransac=20)
            o.add_location(k, desc, uvu, num_ransac=20)
    assert g.num_places == 2000


def test_duplicated_train_descriptors_take_the_lowest_index():
    W = 300
    words = sp.make_vocabulary(W, seed=9)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, 40, W, seed=9)
    g2, o2 = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    dup = np.concatenate([desc, desc])                     # rows j and j + 40 are identical
    Xd = np.concatenate([X, X])
    for d in range(5):
        _check(g2, o2, 1000 + d, words[W - 1 - d * 10 - np.arange(10)], np.tile([320.0, 240.0, 300.0], (10, 1)))
    _check(g2, o2, 0, dup, sp.map_uvu(Xd))
    q, uvu = _query(X, desc, 60, T_TRUE, 9)
    rg, _ = _check(g2, o2, 9, q, uvu)
    t, _ = g2.last_matches()
    assert rg["num_matches"] == 60 and t.max() < 40


def test_all_matches_share_one_train_index():
    W = 300
    words = sp.make_vocabulary(W, seed=10)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, 30, W, seed=10)
    q = np.repeat(desc[:1], 200, 0)                        # every query row matches train row 0 (and words[wid[0]])
    q = q + np.random.default_rng(1).normal(size=q.shape).astype(np.float32) * 1e-3
    uvu = np.tile(sp.map_uvu(X[:1]), (200, 1))
    # score: one word shared with place 0, 200 times -> well above 2 with 7 places
    rg, ro = _check(g, o, 9, q, uvu)
    tri, inl, best = g.last_hypotheses()
    assert rg["best_keyframe_id"] == 0 and len(inl) == 100 and (inl == -1).all() and best == -1


def test_zero_disparity_row_poisons_only_its_hypotheses():
    W = 400
    words = sp.make_vocabulary(W, seed=12)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    X, wid, desc = _pair(g, o, 80, W, seed=12)
    q, uvu = _query(X, desc, 80, T_TRUE, 12)
    uvu[5, 2] = uvu[5, 0]                                   # u == u_right
    rg, _ = _check(g, o, 9, q, uvu)
    tri, inl, _ = g.last_hypotheses()
    poisoned = (tri == 5).any(1)
    assert poisoned.any() and (inl[poisoned] == 0).all() and rg["loop_found"]


def test_policies_without_candidate_or_hypotheses():
    words, kfs = sp.make_sequence(num_keyframes=45, num_scenes=40, seed=13)
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    for k in kfs[:40]:
        _check(g, o, k["id"], k["desc"], k["uvu"], do_loop_detection=False)
        assert g.last_scores()[0].size == 0
    k = kfs[40]
    rg, _ = _check(g, o, k["id"], k["desc"], k["uvu"], exclude=list(range(40)))    # exclude set covers every place
    assert rg["best_keyframe_id"] == -1 and g.last_scores()[0].size == 0
    k = kfs[41]
    rg, _ = _check(g, o, k["id"], k["desc"], k["uvu"], num_ransac=0)
    assert rg["best_keyframe_id"] >= 0 and g.last_hypotheses()[0].shape == (0, 3)
    np.testing.assert_array_equal(rg["T_query_from_loop"], [0, 0, 0, 1, 0, 0, 0])


def test_refused_inputs_leave_the_database_alone(seq):
    words, kfs = seq
    g, o = capi.PlaceRecognizer(words, sp.CAM, device=0), pp.PlaceOracle(words, sp.CAM)
    clean = capi.PlaceRecognizer(words, sp.CAM, device=0)
    for k in kfs[:41]:
        g.add_location(k["id"], k["desc"], k["uvu"])
        clean.add_location(k["id"], k["desc"], k["uvu"])
    k = kfs[41]
    L = capi.lib()
    bad = [dict(keyframe_id=3), dict(num_ransac=-1), dict(pixel_thr=0.0), dict(pixel_thr=float("nan")),
           dict(pixel_thr=float("inf"))]
    for b in bad:
        kw = dict(keyframe_id=k["id"], desc=k["desc"], uvu=k["uvu"])
        kw.update(b)
        with pytest.raises(capi.SvsError) as e:
            g.add_location(**kw)
        assert e.value.rc == -1
    res = capi.SvsPlaceResult()
    assert L.svs_place_add_location(g._h, 99, -1, None, None, 1, 0, None, None, res, None, None) == -1
    assert L.svs_place_add_location(g._h, 99, 5, None, None, 1, 0, None, None, res, None, None) == -1
    assert g.num_places == 41
    a, b = g.add_location(k["id"], k["desc"], k["uvu"]), clean.add_location(k["id"], k["desc"], k["uvu"])
    for key in ("best_keyframe_id", "num_matches", "num_inliers"):
        assert a[key] == b[key]
    assert a["T_query_from_loop"].tobytes() == b["T_query_from_loop"].tobytes()
    assert a["inlier_query"].tolist() == b["inlier_query"].tolist()
