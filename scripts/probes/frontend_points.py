"""The tracked frame's bookkeeping over a synthetic stereo sequence (scavislam_b200/synth_images.py, 640x480, 2 matcher
levels): seeding on the first frame (svs_addMorePoints, fresh), then per frame svs_match_track against the active
keyframe's seeded points, the motion-only LM, svs_processMatchedPoints with the drop test, and seeding from the
processed points when the frame becomes a keyframe.  Prints the host clock of each new stage per frame (each call ends
in a device synchronise), wall time per frame, keyframes dropped and points seeded, the C oracle's host time for the
same stages, and the card with its power limit.  --out PATH also writes the record as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import frontend_pyoracle as fp, pyoracle as po  # noqa: E402
from scavislam_b200 import capi, frontend_inputs as fi, synth_images as si  # noqa: E402

NLV = 2
I7 = np.array([0, 0, 0, 1, 0, 0, 0.0])


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--out")
    args = ap.parse_args()
    seq = si.sequence(args.frames, workers=8)
    cams = fi.level_cams(nlevels=NLV)
    cam = tuple(cams[0][:4])
    levels = [(640 >> l, 480 >> l, cams[l][0], cams[l][1], cams[l][2]) for l in range(NLV)]
    m = capi.GuidedMatcher(levels)
    pose = capi.PoseOptimizer()
    t = {"seed": [], "match_track": [], "process": [], "frame": []}
    t_or = {"seed": [], "process": []}
    drops = seeded = 0

    def frame_inputs(k):
        pyr = fi.uint8_pyramid(seq[k]["img"], NLV)
        feats = []
        for l in range(NLV):
            g = po.fast_grid(640 >> l, 480 >> l, 222 if l == 0 else 55, 74 if l == 0 else 18, 25, 3, 3)
            xy, off = po.fast_detect_adaptively(pyr[l], g, 5)
            feats.append((xy, np.concatenate([np.arange(off[c + 1] - off[c]) for c in range(9)]).astype(np.int32)))
        return pyr, feats

    pyr, feats = frame_inputs(0)
    T_key_w = I7.copy()
    m.set_keyframe(0, T_key_w, pyr)
    m.set_current(pyr, seq[0]["disp"])
    for l in range(NLV):
        m.set_features(l, *feats[l])
    a = time.perf_counter(); _, rows, _ = m.add_more_points(1, cam, 0); t["seed"].append(time.perf_counter() - a)
    seeded += len(rows)
    corners = [f[0] for f in feats]
    a = time.perf_counter()
    fp.c_seed([(640, 480), (320, 240)], corners, seq[0]["disp"], np.zeros(0, fp.TRACKED_DTYPE), [0, 0],
              np.ones(9, np.int32), 2, 300, 0, I7, cam, 0)
    t_or["seed"].append(time.perf_counter() - a)
    points = rows[::-1].copy()          # newpoint_map's push_front order
    T = I7.copy()
    for k in range(1, args.frames):
        pyr, feats = frame_inputs(k)
        f0 = time.perf_counter()
        m.set_current(pyr, seq[k]["disp"])
        for l in range(NLV):
            m.set_features(l, *feats[l])
        half = len(points) // 2
        a = time.perf_counter()
        res, nn, nobs = m.match_track(T, T_key_w, [points[:half], points[half:], points[:0]], 300, 4, 22, 10)
        t["match_track"].append(time.perf_counter() - a)
        if nobs < 20:
            break
        T, _ = pose.calc_fast_motion_only_matched(m, cam, T, True, 2.0, 15)
        a = time.perf_counter()
        out, st, flags, drop = m.process_matched_points(T, cam, len(points))
        t["process"].append(time.perf_counter() - a)
        a = time.perf_counter()
        fp.c_process(res, np.concatenate([points["anchor_level"], points["anchor_level"][:0]]), len(points), T, cam, 640, 480)
        t_or["process"].append(time.perf_counter() - a)
        if drop:
            drops += 1
            a = time.perf_counter(); _, rows, _ = m.add_more_points(0, cam, 0); t["seed"].append(time.perf_counter() - a)
            seeded += len(rows)
            m.set_keyframe(0, capi_compose(T, T_key_w), pyr)
            T_key_w = capi_compose(T, T_key_w)
            T = I7.copy()
            points = rows[::-1].copy()
        t["frame"].append(time.perf_counter() - f0)
    rec = dict(card=card(), frames=args.frames, keyframes_dropped=drops, points_seeded=seeded,
               ms_median={k: 1e3 * float(np.median(v)) if v else None for k, v in t.items()},
               oracle_ms_median={k: 1e3 * float(np.median(v)) if v else None for k, v in t_or.items()},
               note="host clock of each call, which ends in a device synchronise; frame = set_current + features + "
                    "match_track + LM + process (+ seeding on a drop)")
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


def capi_compose(A, B):
    from oracle import loop_pyoracle as lo
    return lo.se3("oloop_se3_mul", A, B)


if __name__ == "__main__":
    main()
