"""Developer probe (GPU box): cost of svs_ba_window_grad beside svs_ba_observation_grad on the BA handle.

For each config (default C2, P = 200 / L = 20 000 / C = 1 020, and C5, P = 1000 / L = 100 000 / C = 5 100): pose 0
fixed, 3 LM iterations, lambda = 0, a seeded random upstream gradient, medians over `calls` calls after 20 warm-up calls
of
  all_*   svs_ba_window_grad from host arrays, every output (obs, info, cT, cLambda, cam) to host arrays
  obs_*   svs_ba_window_grad with only dL_dobs / dL_dinfo requested
  og_*    svs_ba_observation_grad from host arrays, both outputs to host arrays
The three run in turn within each round, so that drift of the shared machine falls on all of them alike.  *_host_ms is
the wall time of a call (each ends in a stream synchronise), *_stats_ms the stats' device time (build + factor + solve
+ adjoint kernels).  The GPU name, power limit and maximum SM clock are read in the same run.
Usage: python scripts/probes/ba_window_grad.py [calls] [config ...]
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


def gpu_settings():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def probe(config, calls, warm):
    pb = synth.make_config(config)
    pb.fixed = np.zeros(pb.P, np.uint8)
    pb.fixed[0] = 1
    ba = capi.BundleAdjuster(device=0)
    ba.set_problem(pb)
    ba.optimize(3)
    rng = np.random.default_rng(0)
    gp, gl = rng.normal(size=(pb.P, 6)), rng.normal(size=(pb.L, 3))
    arr = dict(obs=np.zeros((pb.E, 3)), info=np.zeros((pb.E, 3)), cT=np.zeros((pb.C, 6)), cLambda=np.zeros((pb.C, 36)),
               cam=np.zeros(4))
    og_obs, og_info = np.zeros((pb.E, 3)), np.zeros((pb.E, 3))
    st = capi.SvsBaGradStats()
    full, part = capi.SvsBaGradOut(), capi.SvsBaGradOut()
    for k, a in arr.items():
        setattr(full, capi.BundleAdjuster._GRAD_OUT[k][0], a.ctypes.data)
    part.dL_dobs, part.dL_dinfo = arr["obs"].ctypes.data, arr["info"].ctypes.data

    def window(out):
        rc = capi.lib().svs_ba_window_grad(ba._h, 1, 1.0, 0.0, gp.ctypes.data, gl.ctypes.data, C.byref(out), 0,
                                           C.byref(st))
        assert rc == 0, rc
        return st.ms

    def og():
        rc = capi.lib().svs_ba_observation_grad(ba._h, 1, 1.0, 0.0, gp.ctypes.data, gl.ctypes.data, og_obs.ctypes.data,
                                                og_info.ctypes.data, 0, C.byref(st))
        assert rc == 0, rc
        return st.ms

    fns = dict(all=lambda: window(full), obs=lambda: window(part), og=og)
    host = {k: [] for k in fns}
    dev = {k: [] for k in fns}
    for it in range(warm + calls):
        for k, fn in fns.items():
            t = time.perf_counter()
            ms = fn()
            dt = time.perf_counter() - t
            if it >= warm:
                host[k].append(dt * 1e3)
                dev[k].append(ms)
    ba.close()
    assert all(np.isfinite(a).all() for a in arr.values())
    row = dict(config=config, P=int(pb.P), L=int(pb.L), E=int(pb.E), C=int(pb.C), nnzb_L=st.nnzb_L, nbranch=st.nbranch,
               general=st.general)
    for k in fns:
        row[f"{k}_host_ms"] = float(np.median(host[k]))
        row[f"{k}_stats_ms"] = float(np.median(dev[k]))
        row[f"{k}_stats_ms_p10_p90"] = [float(np.percentile(dev[k], 10)), float(np.percentile(dev[k], 90))]
    return row


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    configs = sys.argv[2:] or ["C2", "C5"]
    rows = [probe(c, calls, 20) for c in configs]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=gpu_settings(), calls=calls,
                          warmup=20, results=rows)))


if __name__ == "__main__":
    main()
