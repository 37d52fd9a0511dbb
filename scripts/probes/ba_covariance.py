"""Developer probe (GPU box): cost of one svs_ba_covariance call on the BA handle.

For each config (default C2, P = 200 / L = 20 000, and C5, P = 1000 / L = 100 000): pose 0 fixed, 3 LM iterations,
then lambda = 0 and two kinds of call, medians over `calls` calls after a warm-up:
  poses_*   the P diagonal pose blocks only (point_cov = NULL)
  full_*    the P pose blocks and all L landmark blocks
where *_host_ms is the wall time of a call (it ends in a stream synchronise, outputs copied to host memory) and
*_stats_ms the stats' device time (build + factor + selected inversion + landmark kernel).  The GPU name and power
limit are read in the same run.
Usage: python scripts/probes/ba_covariance.py [calls] [config ...]
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


def timed(ba, pose, point, calls, warm):
    host, dev = [], []
    st = capi.SvsBaCovStats()
    for k in range(warm + calls):
        t = time.perf_counter()
        rc = capi.lib().svs_ba_covariance(ba._h, 1, 1.0, 0.0, capi._dp(pose), 0, None, None, None,
                                          capi._dp(point) if point is not None else None, C.byref(st))
        dt = time.perf_counter() - t
        assert rc == 0, rc
        if k >= warm:
            host.append(dt * 1e3)
            dev.append(st.ms)
    return st.as_dict(), float(np.median(host)), float(np.median(dev))


def probe(config, calls, warm):
    pb = synth.make_config(config)
    pb.fixed = np.zeros(pb.P, np.uint8)
    pb.fixed[0] = 1
    ba = capi.BundleAdjuster(device=0)
    ba.set_problem(pb)
    ba.optimize(3)
    pose, point = np.zeros((pb.P, 6, 6)), np.zeros((pb.L, 3, 3))
    st, p_host, p_dev = timed(ba, pose, None, calls, warm)
    _, f_host, f_dev = timed(ba, pose, point, calls, warm)
    ev = np.linalg.eigvalsh(point)
    ba.close()
    return dict(config=config, P=int(pb.P), L=int(pb.L), nnzb_L=st["nnzb_L"], nbranch=st["nbranch"], general=st["general"],
                poses_host_ms=p_host, poses_stats_ms=p_dev, full_host_ms=f_host, full_stats_ms=f_dev,
                landmark_kernel_ms_est=f_dev - p_dev, landmark_blocks_pd=bool((ev > 0).all()))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    configs = sys.argv[2:] or ["C2", "C5"]
    rows = [probe(c, calls, 20) for c in configs]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), calls=calls, warmup=20,
                          results=rows)))


if __name__ == "__main__":
    main()
