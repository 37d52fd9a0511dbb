"""Seeded synthetic keyframe sequence for place recognition (PlaceRecognizer::addLocation, reference
placerecognizer.cpp:206-324): a vocabulary of unit vectors, scenes of landmarks that each carry a word, and keyframes
that see a scene from a known pose -- first every scene once, then revisits.  A keyframe's rows are noisy copies of
its landmarks' words (some noisy enough to fall outside the 0.1 word radius), landmarks that share a word within a
scene (ambiguous matches), and distractor rows (random descriptors at random pixels).  uvu follows the svs_cam
convention of the other synth modules: (u, v, u_right) of StereoCamera::map_uvu."""
import numpy as np

from .synth_pose import CAM, _quat_from_rotvec, _rot

DIM = 64


def make_vocabulary(num_words, seed=0):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=(num_words, DIM))
    return (w / np.linalg.norm(w, axis=1, keepdims=True)).astype(np.float32)


def map_uvu(xyz, cam=CAM):
    f, px, py, b = cam
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    return np.stack([f * (x / z) + px, f * (y / z) + py, (x - b) / z * f + px], 1)


def se3_apply(T, X):
    return X @ _rot(T[:4]).T + T[4:]


def se3_mul(A, B):
    """A * B for qt = (qx, qy, qz, qw, tx, ty, tz)."""
    Ra, Rb = _rot(A[:4]), _rot(B[:4])
    return _qt(Ra @ Rb, Ra @ B[4:] + A[4:])


def se3_inv(A):
    R = _rot(A[:4])
    return _qt(R.T, -R.T @ A[4:])


def _qt(R, t):
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    if w > 1e-6:
        q = np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
    else:   # rotations near pi do not occur in these sequences
        raise ValueError("rotation too close to pi")
    return np.concatenate([q / np.linalg.norm(q), t])


def make_sequence(num_keyframes=60, num_scenes=40, num_words=4000, landmarks=160, seed=0, cam=CAM,
                  pixel_noise=0.3, shared_word_frac=0.08, far_frac=0.15, distractor_frac=0.1, visible_frac=0.85):
    """Returns (words, keyframes).  keyframes[i] = dict(id, scene, T (camera from scene, qt), desc [n][64] float32,
    uvu [n][3]).  Keyframe i < num_scenes sees scene i; later keyframes revisit earlier scenes."""
    rng = np.random.default_rng(seed)
    words = make_vocabulary(num_words, seed + 1)
    f, px, py, b = cam
    scenes = []
    for s in range(num_scenes):
        z = rng.uniform(2.0, 10.0, landmarks)
        u, v = rng.uniform(40, 600, landmarks), rng.uniform(40, 440, landmarks)
        X = np.stack([(u - px) / f * z, (v - py) / f * z, z], 1)
        wid = rng.choice(num_words, landmarks, replace=False)
        nshare = int(shared_word_frac * landmarks)
        wid[:nshare] = wid[landmarks - nshare:]           # landmarks that share a word within the scene
        scenes.append((X, wid))
    schedule = list(range(min(num_scenes, num_keyframes)))
    schedule += list(rng.integers(0, num_scenes, num_keyframes - len(schedule)))
    kfs = []
    for i, s in enumerate(schedule):
        X, wid = scenes[s]
        T = np.concatenate([_quat_from_rotvec(rng.normal(0, 0.04, 3)), rng.normal(0, 0.15, 3)])
        vis = np.flatnonzero(rng.random(len(X)) < visible_frac)
        P = se3_apply(T, X[vis])
        uvu = map_uvu(P, cam) + rng.normal(0, pixel_noise, (len(vis), 3))
        sigma = np.where(rng.random(len(vis)) < far_frac, 0.07, 0.02)[:, None]
        desc = words[wid[vis]] + rng.normal(size=(len(vis), DIM)) * sigma
        nd = int(distractor_frac * len(vis))
        dd = rng.normal(size=(nd, DIM))
        dd /= np.linalg.norm(dd, axis=1, keepdims=True)
        zd = rng.uniform(2.0, 10.0, nd)
        du = np.stack([rng.uniform(0, 640, nd), rng.uniform(0, 480, nd)], 1)
        uvu_d = np.concatenate([du, (du[:, :1] - f * b / zd[:, None])], 1)
        desc = np.concatenate([desc, dd]).astype(np.float32)
        uvu = np.concatenate([uvu, uvu_d])
        perm = rng.permutation(len(desc))
        kfs.append(dict(id=i, scene=int(s), T=T, desc=np.ascontiguousarray(desc[perm]), uvu=np.ascontiguousarray(uvu[perm])))
    return words, kfs


def true_T_query_from_loop(query, loop):
    """T_query_from_loop of two keyframes of the same scene."""
    assert query["scene"] == loop["scene"]
    return se3_mul(query["T"], se3_inv(loop["T"]))
