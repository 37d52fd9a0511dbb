"""Developer probe (GPU box): cost of one svs_ba_observation_grad call on the BA handle.

For each config (default C2, P = 200 / L = 20 000, and C5, P = 1000 / L = 100 000): pose 0 fixed, 3 LM iterations,
lambda = 0, a seeded random upstream gradient, medians over `calls` calls after 20 warm-up calls of
  grad_*    svs_ba_observation_grad from host arrays, both outputs to host arrays
  cov_*     svs_ba_covariance, pose blocks only, beside it
  opt1_*    one svs_ba_optimize(1) on the same handle (one Levenberg iteration), re-loaded before each call
where *_host_ms is the wall time of a call (each ends in a stream synchronise) and *_stats_ms the stats' device time.
The GPU name and power limit are read in the same run.
Usage: python scripts/probes/ba_grad.py [calls] [config ...]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch

from scavislam_b200 import capi, synth


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def median_of(fn, calls, warm):
    host, dev = [], []
    for k in range(warm + calls):
        t = time.perf_counter()
        ms = fn()
        dt = time.perf_counter() - t
        if k >= warm:
            host.append(dt * 1e3)
            dev.append(ms)
    return float(np.median(host)), float(np.median(dev))


def probe(config, calls, warm):
    pb = synth.make_config(config)
    pb.fixed = np.zeros(pb.P, np.uint8)
    pb.fixed[0] = 1
    ba = capi.BundleAdjuster(device=0)
    ba.set_problem(pb)
    ba.optimize(3)
    rng = np.random.default_rng(0)
    gp, gl = rng.normal(size=(pb.P, 6)), rng.normal(size=(pb.L, 3))
    dobs, dinfo = np.zeros((pb.E, 3)), np.zeros((pb.E, 3))
    gst, cst = capi.SvsBaGradStats(), capi.SvsBaCovStats()
    pose = np.zeros((pb.P, 6, 6))

    def grad():
        rc = capi.lib().svs_ba_observation_grad(ba._h, 1, 1.0, 0.0, gp.ctypes.data, gl.ctypes.data, dobs.ctypes.data,
                                                dinfo.ctypes.data, 0, C.byref(gst))
        assert rc == 0, rc
        return gst.ms

    def cov():
        rc = capi.lib().svs_ba_covariance(ba._h, 1, 1.0, 0.0, capi._dp(pose), 0, None, None, None, None, C.byref(cst))
        assert rc == 0, rc
        return cst.ms

    g_host, g_dev = median_of(grad, calls, warm)
    c_host, c_dev = median_of(cov, calls, warm)
    poses, points = ba.poses(), ba.points()
    opt_host, opt_dev = [], []
    for k in range(warm + calls):   # one iteration from the same state each time: set_problem is outside the timing
        ba.set_problem(pb)
        t = time.perf_counter()
        _, st = ba.optimize(1)
        dt = time.perf_counter() - t
        if k >= warm:
            opt_host.append(dt * 1e3)
            opt_dev.append(st["ms_total"])
    ba.close()
    assert np.isfinite(dobs).all() and np.isfinite(dinfo).all() and np.isfinite(poses).all() and np.isfinite(points).all()
    return dict(config=config, P=int(pb.P), L=int(pb.L), E=int(pb.E), nnzb_L=gst.nnzb_L, nbranch=gst.nbranch,
                general=gst.general, grad_host_ms=g_host, grad_stats_ms=g_dev, cov_poses_host_ms=c_host,
                cov_poses_stats_ms=c_dev, opt1_host_ms=float(np.median(opt_host)),
                opt1_stats_ms=float(np.median(opt_dev)))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    configs = sys.argv[2:] or ["C2", "C5"]
    rows = [probe(c, calls, 20) for c in configs]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), calls=calls, warmup=20,
                          results=rows)))


if __name__ == "__main__":
    main()
