"""The place-recognition oracle (oracle/place_oracle.c) against independent restatements: OpenCV's BFMatcher, a
float64 word search, a literal transcription of calcLoopStatistics / addLocation (placerecognizer.cpp:131-172,
206-324), numpy Kabsch and a numpy SplitMix64."""
import numpy as np
import pytest

from oracle import place_pyoracle as pp
from scavislam_b200 import capi, synth_place as sp

M64 = (1 << 64) - 1


def test_matches_equal_opencv_bfmatcher():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    q = rng.normal(size=(300, 64)).astype(np.float32)
    t = rng.normal(size=(700, 64)).astype(np.float32)
    d64 = ((q[:, None, :].astype(np.float64) - t[None].astype(np.float64)) ** 2).sum(-1)
    srt = np.sort(d64, 1)
    keep = (srt[:, 1] - srt[:, 0]) > 1e-3 * srt[:, 0]          # no near-ties
    idx, d = pp.nn(q, t)
    ms = cv2.BFMatcher(cv2.NORM_L2).match(q, t)
    cv_idx = np.array([m.trainIdx for m in ms])
    cv_d = np.array([m.distance for m in ms], np.float64)
    assert keep.sum() > 250
    assert np.array_equal(idx[keep], cv_idx[keep])
    np.testing.assert_allclose(np.sqrt(d.astype(np.float64))[keep], cv_d[keep], rtol=1e-6)


def test_words_equal_float64_argmin():
    words = sp.make_vocabulary(3000, seed=5)
    rng = np.random.default_rng(1)
    base = words[rng.integers(0, 3000, 800)].astype(np.float64)
    desc = (base + rng.normal(size=base.shape) * rng.choice([0.02, 0.035, 0.05], (800, 1))).astype(np.float32)
    o = pp.PlaceOracle(words, sp.CAM)
    r = o.add_location(0, desc, np.tile([300.0, 200.0, 280.0], (800, 1)), do_loop_detection=False)
    d64 = ((desc[:, None, :].astype(np.float64) - words[None].astype(np.float64)) ** 2).sum(-1)
    order = np.argsort(d64, 1)
    best = d64[np.arange(800), order[:, 0]]
    second = d64[np.arange(800), order[:, 1]]
    clean = ((second - best) > 1e-5) & (np.abs(best - 0.1) > 1e-5)
    ref = np.where(best < 0.1, order[:, 0], -1)
    assert clean.sum() > 700 and (ref >= 0).sum() > 100 and (ref < 0).sum() > 100
    assert np.array_equal(r["words"][clean], ref[clean])
    assert r["number_of_words"] == int((r["words"] >= 0).sum())


def _literal_add_location(state, kf_id, word_rows, exclude, do_loop):
    """calcLoopStatistics / addLocation as the reference writes them: dicts, float32 scalars, the inverted index
    filled descriptor by descriptor."""
    inverted, location_nwords = state
    f32 = np.float32
    stats = {}
    nw = 0
    for w in word_rows:
        if w < 0:
            continue
        nw += 1
        kmap = inverted.setdefault(int(w), {})
        if do_loop:
            nloc, ncont = f32(len(location_nwords)), f32(len(kmap))
            if ncont > 0:
                idf = f32(nloc / ncont)
                for other, cnt in kmap.items():
                    if other == kf_id or other in exclude:
                        continue
                    tf = f32(f32(cnt) / f32(location_nwords[other]))
                    stats[other] = f32(stats.get(other, f32(0)) + f32(tf * idf))
        kmap[kf_id] = kmap.get(kf_id, 0) + 1
    location_nwords[kf_id] = nw
    return stats


def test_tfidf_scores_bit_equal_literal_transcription():
    words, kfs = sp.make_sequence(num_keyframes=30, num_scenes=20, num_words=1500, landmarks=100, seed=7,
                                  shared_word_frac=0.2)
    o = pp.PlaceOracle(words, sp.CAM)
    state = ({}, {})
    seen_repeat = seen_excl = 0
    for k in kfs:
        excl = {k["id"] - 1, k["id"] - 2, 3} if k["id"] > 4 else set()
        r = o.add_location(k["id"], k["desc"], k["uvu"], exclude=sorted(excl), num_ransac=10)
        wr = r["words"]
        seen_repeat += len(wr[wr >= 0]) > len(set(wr[wr >= 0]))
        stats = _literal_add_location(state, k["id"], wr, excl, True)
        got = dict(zip(r["score_ids"].tolist(), r["scores"]))
        assert set(got) == set(stats)
        for kid, v in stats.items():
            assert got[kid].tobytes() == np.float32(v).tobytes(), (k["id"], kid, got[kid], v)
        assert not set(got) & excl
        seen_excl += bool(excl)
        cand = [kid for kid, v in stats.items() if v > 2]
        best = max(cand, key=lambda kid: (stats[kid], -kid)) if cand else -1
        assert r["best_keyframe_id"] == best
    assert seen_repeat > 5 and seen_excl > 5


def _np_kabsch(p0, p1):
    c0, c1 = p0.mean(0), p1.mean(0)
    H = (p1 - c1).T @ (p0 - c0)
    U, S, Vt = np.linalg.svd(H)
    V = Vt.T
    d = np.sign(np.linalg.det(V @ U.T))
    R = V @ np.diag([1, 1, d]) @ U.T
    return R, c0 - R @ c1


def test_kabsch_equals_numpy_svd_including_reflections():
    rng = np.random.default_rng(3)
    nref = 0
    for i in range(300):
        p1 = rng.normal(size=(3, 3)) * 3
        q = sp._quat_from_rotvec(rng.normal(size=3))
        R0 = sp._rot(q)
        if i % 3 == 0:
            R0 = R0 @ np.diag([1, 1, -1])                    # a mirrored triple: the naive V U^T is a reflection
        p0 = p1 @ R0.T + rng.normal(size=3) + rng.normal(size=(3, 3)) * 0.05
        c0, c1 = p0.mean(0), p1.mean(0)
        U, S, Vt = np.linalg.svd((p1 - c1).T @ (p0 - c0))
        nref += np.linalg.det(Vt.T @ U.T) < 0
        R, t = pp.kabsch(p0, p1)
        Rn, tn = _np_kabsch(p0, p1)
        assert abs(np.linalg.det(R) - 1) < 1e-12
        np.testing.assert_allclose(R, Rn, atol=1e-12)
        np.testing.assert_allclose(t, tn, atol=1e-12 * max(1.0, np.abs(tn).max()))
    assert nref > 20


def _np_splitmix(state, count):
    out = []
    for _ in range(count):
        state = (state + 0x9E3779B97F4A7C15) & M64
        z = state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        out.append(z ^ (z >> 31))
    return out


def test_splitmix_sampler_equals_numpy_restatement():
    for seed in (0, 1, 0xDEADBEEFCAFEF00D):
        for h in (0, 1, 99):
            st = seed ^ ((0xD1B54A32D192ED03 * (h + 1)) & M64)
            assert pp.splitmix(st, 50) == _np_splitmix(st, 50)
            # the triple: the reference's redraw rules on the stream
            nmatch = 37
            tidx = np.arange(nmatch) // 2                     # pairs of matches share a train index
            zs = iter(_np_splitmix(st, 64))
            tri, draws = [], 0
            while len(tri) < 3:
                x = ((next(zs) >> 32) * nmatch) >> 32
                draws += 1
                if x in tri:
                    continue
                tri.append(x)
                if len(tri) == 3 and len({int(tidx[j]) for j in tri}) < 3:
                    tri = []
            d, got = pp.draw_triple(seed, h, tidx)
            assert d == draws and got.tolist() == tri


def test_draws_bounded_when_train_indices_repeat():
    d, _ = pp.draw_triple(5, 0, np.zeros(20, np.int32))
    assert d == -1


def test_synthetic_revisit_recovers_T():
    words, kfs = sp.make_sequence(seed=3)
    o = pp.PlaceOracle(words, sp.CAM)
    found = 0
    for k in kfs:
        r = o.add_location(k["id"], k["desc"], k["uvu"])
        if k["id"] >= 40 and r["loop_found"]:
            loop = kfs[r["best_keyframe_id"]]
            assert loop["scene"] == k["scene"]
            Tt, T = sp.true_T_query_from_loop(k, loop), r["T_query_from_loop"]
            assert np.abs(T[4:] - Tt[4:]).max() < 0.2
            assert min(np.abs(T[:4] - Tt[:4]).max(), np.abs(T[:4] + Tt[:4]).max()) < 0.03
            found += 1
    assert found >= 8


def test_load_surf_vocabulary_round_trip(tmp_path):
    cv2 = pytest.importorskip("cv2")
    words = sp.make_vocabulary(50, seed=2)
    img = np.ascontiguousarray(words).view(np.uint8)          # [50][256]: every float as four uint8
    path = str(tmp_path / "words.png")
    assert cv2.imwrite(path, img)
    back = capi.load_surf_vocabulary(path)
    assert back.dtype == np.float32 and back.shape == (50, 64)
    assert back.tobytes() == words.tobytes()
