"""Developer probe (GPU box): device time of svs_pose_grad beside the forward svs_calcFastMotionOnly it differentiates.

For n = 333 (one CTA), 1800 (shared points) and 5000 (8-CTA cluster) observations of synth_pose.make_track with 10 %
outliers: the forward from host arrays with the reference's front-end setting (robust, kernel_param 2, 15 iterations),
then svs_pose_grad with every output to host arrays, lambda = 0 and a seeded random upstream gradient.  Medians of the
stats' device time (fwd_ms: the LM kernel; grad_ms: the gradient kernels) over `calls` rounds after 20 warm-up rounds,
the two calls in turn within each round.  The GPU name, power limit and maximum SM clock are read in the same run.
Usage: python scripts/probes/pose_grad.py [calls]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch

from scavislam_b200 import capi
from scavislam_b200 import synth_pose as sp


def gpu_settings():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def probe(n, shared, calls, warm):
    tr = sp.make_track(n, seed=n, outlier_frac=0.1, shared_points=shared)
    po = capi.PoseOptimizer(device=0)
    g = np.random.default_rng(0).normal(size=6)
    fwd, grad, host = [], [], []
    for it in range(warm + calls):
        _, st = po.calc_fast_motion_only(tr["pid"], tr["obs"], tr["xyz"], tr["cam"], tr["T_init"], True, 2.0, 15)
        t = time.perf_counter()
        res, rc, gst = po.grad(g)
        dt = time.perf_counter() - t
        assert rc == 0 and all(np.isfinite(a).all() for a in res.values())
        if it >= warm:
            fwd.append(st["ms"])
            grad.append(gst["ms"])
            host.append(dt * 1e3)
    po.close()
    return dict(n=n, npoints=int(len(tr["xyz"])), shared_points=shared, fwd_ms=float(np.median(fwd)),
                grad_ms=float(np.median(grad)), grad_p10_p90=[float(np.percentile(grad, 10)), float(np.percentile(grad, 90))],
                grad_host_ms=float(np.median(host)))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rows = [probe(n, shared, calls, 20) for n, shared in ((333, False), (1800, True), (5000, False))]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=gpu_settings(), calls=calls,
                          warmup=20, results=rows)))


if __name__ == "__main__":
    main()
