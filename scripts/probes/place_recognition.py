"""Device time of one svs_place_add_location (PlaceRecognizer::addLocation) at n = 1 000 descriptors, W = 10 000
words and 500 / 2 000 stored places, next to the CPU oracle's time for one such call (on a database of 20 places:
its cost is the n x W word search, and filling a 500-place oracle database would take minutes); prints the card and
its power limit.  --out PATH also writes the whole record as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import place_pyoracle as pp  # noqa: E402
from scavislam_b200 import capi, synth_place as sp  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # the numbers are still labelled with the library's own device string
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    args = ap.parse_args()
    W, n, reps = 10000, 1000, 20
    words = sp.make_vocabulary(W, seed=1)
    rng = np.random.default_rng(2)
    out = dict(card=card(), device=capi.device_info(), W=W, n=n, rows=[])

    def place(i):
        wid = rng.integers(0, W, n)
        desc = (words[wid] + rng.normal(size=(n, 64)) * 0.02).astype(np.float32)
        uv = np.stack([rng.uniform(0, 640, n), rng.uniform(0, 480, n)], 1)
        return desc, np.concatenate([uv, uv[:, :1] - rng.uniform(2, 40, (n, 1))], 1)

    for L in (500, 2000):
        g = capi.PlaceRecognizer(words, sp.CAM, device=0)
        o = pp.PlaceOracle(words, sp.CAM) if L == 500 else None
        base = [place(i) for i in range(L)]
        for i, (d, u) in enumerate(base):
            g.add_location(i, d, u, do_loop_detection=False)
            if o is not None and i < 20:
                o.add_location(i, d, u, do_loop_detection=False)
        # queries revisit stored places (a candidate, a match and the RANSAC run every time)
        ms, host = [], []
        for r in range(reps + 3):
            d, u = base[r * 7 % L]
            d = (d + rng.normal(size=d.shape) * 0.01).astype(np.float32)
            t0 = time.perf_counter()
            res = g.add_location(L + r, d, u)          # returns after the stream has synchronised
            t1 = time.perf_counter()
            if r >= 3:
                ms.append(res["ms"]); host.append((t1 - t0) * 1e3)
        row = dict(places=L, device_ms_median=float(np.median(ms)), device_ms_min=float(np.min(ms)),
                   host_ms_median=float(np.median(host)), best=res["best_keyframe_id"], inliers=res["num_inliers"])
        if o is not None:
            d, u = base[0]
            t0 = time.perf_counter()
            o.add_location(L + 10**6, d, u)
            row["oracle_cpu_ms_20_places"] = (time.perf_counter() - t0) * 1e3
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
        g.close()
    print(json.dumps(dict(card=out["card"], device=out["device"])))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
