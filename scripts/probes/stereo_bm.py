"""Time of one svs_stereo_compute (calcDisparityCpu's StereoBM on the device) at 640x480 / ndisp 32, 512x384 / 32
(data/newcollege.cfg's camera) and 1241x376 / 64, after a warm-up: the call's host time (it ends in a stream
synchronise, host images in), and in a separate torch.profiler run the device time of each kernel and copy (the
per-stage split).  Then the cost of handing the map to the dense tracker, its CPU variant and the matcher by device
pointer, against uploading the same map from host memory.  Each map is checked bit for bit against cv2.StereoBM, whose
single-threaded CPU time on the same host is listed for scale.  Prints the card and its power limit; --out PATH also
writes the whole record as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from scavislam_b200 import capi, frontend_inputs as fi, synth_images as si  # noqa: E402

SHAPES = [(640, 480, 32, None), (512, 384, 32, (389.956085, 254.903519, 201.899490, 0.120005)),
          (1241, 376, 64, (700.0, 620.5, 188.0, 0.12))]
STAGES = [("prefilter", "k_stereo_prefilter"), ("cost_wta_uniqueness", "k_stereo_cost"), ("left_right_border", "k_stereo_lr"),
          ("speckle_unite", "k_stereo_unite"), ("speckle_count", "k_stereo_count"), ("speckle_final", "k_stereo_final")]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # the numbers are still labelled with the library's own device string
        return f"nvidia-smi unavailable ({e})"


def cv_bm(left, right, nd):
    bm = cv2.StereoBM_create(numDisparities=nd, blockSize=7)
    bm.setPreFilterCap(31); bm.setTextureThreshold(10); bm.setUniquenessRatio(15)
    bm.setSpeckleWindowSize(100); bm.setSpeckleRange(32); bm.setDisp12MaxDiff(1)
    return bm.compute(left, right)


def stage_split(sm, left, right, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            sm.compute(left, right)
    us = {k: 0.0 for k, _ in STAGES}
    us["h2d_copies"] = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        for k, kern in STAGES:
            if kern in e.key:
                us[k] += t / reps
        if "Memcpy HtoD" in e.key:
            us["h2d_copies"] += t / reps
    torch.cuda.synchronize()
    return {k: round(v, 2) for k, v in us.items()}


def timed(fn, reps):
    import torch
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    out = dict(card=card(), device=capi.device_info(), reps=args.reps, rows=[])
    cv2.setNumThreads(1)
    for w, h, nd, cam in SHAPES:
        left, right, _ = si.render_stereo_pair(np.array([0.0, 0.0, 0.0]), 0.0, 77, w, h, cam)
        sm = capi.StereoMatcher(w, h, nd, device=0)
        for _ in range(10):
            sm.compute(left, right)
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            sm.compute(left, right)            # returns after the stream has synchronised
            ms.append((time.perf_counter() - t0) * 1e3)
        d = sm.disparity()
        ref = cv_bm(left, right, nd)
        t0 = time.perf_counter()
        for _ in range(5):
            cv_bm(left, right, nd)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / 5
        split = stage_split(sm, left, right, 50)
        row = dict(w=w, h=h, ndisp=nd, call_ms_median=float(np.median(ms)), call_ms_min=float(np.min(ms)),
                   device_us_per_stage=split, device_us_kernels=round(sum(v for k, v in split.items() if k != "h2d_copies"), 2),
                   bit_exact_with_cv2=bool(np.array_equal((d * 16).astype(np.int16), ref)),
                   valid_fraction=float((d > 0).mean()), cv2_single_thread_cpu_ms=cpu_ms)
        if (w, h) == (640, 480):
            ptr, stride = sm.device_disparity()
            cams = fi.level_cams(nlevels=3)
            dt, dtc = capi.DenseTracker(w, h, 3), capi.DenseTrackerCpuVariant(w, h, 3)
            m = capi.GuidedMatcher([(w >> l, h >> l) + tuple(cams[l][:3]) for l in range(3)])
            reps = 50
            row["handover_ms_median"] = dict(
                dt_device=timed(lambda: dt.set_disparity_device(ptr, stride), reps),
                dt_host=timed(lambda: dt.set_disparity(d), reps),
                dtc_device=timed(lambda: dtc.set_disparity_device(ptr, stride), reps),
                dtc_host=timed(lambda: dtc.set_disparity(d), reps),
                matcher_device=timed(lambda: m.set_current_disparity_device(ptr, stride), reps),
                matcher_host=timed(lambda: m.set_current_disparity(d), reps))
            dt.close(); dtc.close(); m.close()
        sm.close()
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(card=out["card"], device=out["device"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
