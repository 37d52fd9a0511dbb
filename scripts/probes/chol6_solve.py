"""Developer probe (GPU box): cost of one svs_chol6_solve call on C2's reduced camera system.

Takes C2's reduced system from BundleAdjuster.reduced_system(True, 1.0, 50.0) (lambda on the diagonal), converts it to
the upper block CCS g2o's fillCCS(..., upperTriangle = true) would give, and reports medians after a warm-up:
  host_ms      wall time of one call, host arrays in and x out (the call ends in a stream synchronise)
  device_ms    the same with torch CUDA tensors (on_device = 1)
  stats_ms     svs_chol6_stats.ms: device time of scatter + factor + solve
  ba_solve_ms  wall time of svs_ba_solve_reduced on the same window (includes the Schur build of the system)
with the GPU name and power limit of the same run.  Usage: python scripts/probes/chol6_solve.py [calls] [config]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch

from scavislam_b200 import capi, synth


def upper_ccs(S):
    P = S.shape[0] // 6
    nz = np.abs(S.reshape(P, 6, P, 6)).max(axis=(1, 3)) > 0
    col_ptr, row_idx, blocks = [0], [], []
    for j in range(P):
        for i in range(j + 1):
            if i == j or nz[i, j]:
                row_idx.append(i)
                blocks.append(S[6 * i:6 * i + 6, 6 * j:6 * j + 6].ravel(order="F"))
        col_ptr.append(len(row_idx))
    return np.array(col_ptr, np.int32), np.array(row_idx, np.int32), np.ascontiguousarray(np.array(blocks).reshape(-1, 36))


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 300
    config = sys.argv[2] if len(sys.argv) > 2 else "C2"
    warm = 50
    pb = synth.make_config(config)
    ba = capi.BundleAdjuster(device=0)
    ba.set_problem(pb)
    S, bs, _ = ba.reduced_system(True, 1.0, 50.0)
    cp, ri, blocks = upper_ccs(S)
    chol = capi.BlockCholesky6(device=0)

    host, stats_ms, reused = [], [], []
    for k in range(warm + calls):
        t = time.perf_counter()
        x_h, rc, st = chol.solve(cp, ri, blocks, bs)
        dt = time.perf_counter() - t
        if k >= warm:
            host.append(dt * 1e3); stats_ms.append(st["ms"]); reused.append(st["symbolic_reused"])
    assert rc == 0

    d_blocks, d_b = torch.from_numpy(blocks).cuda(), torch.from_numpy(bs).cuda()
    torch.cuda.synchronize()
    dev = []
    for k in range(warm + calls):
        t = time.perf_counter()
        x_d, rc_d, _ = chol.solve(cp, ri, d_blocks, d_b)
        dt = time.perf_counter() - t
        if k >= warm:
            dev.append(dt * 1e3)
    assert rc_d == 0

    ba_ms = []
    for k in range(warm + calls):
        t = time.perf_counter()
        x_ba, rc_ba = ba.solve_reduced(True, 1.0, 50.0)
        dt = time.perf_counter() - t
        if k >= warm:
            ba_ms.append(dt * 1e3)

    out = dict(
        gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), config=config, P=int(pb.P),
        nnzb_A=int(st["nnzb_A"]), nnzb_L=int(st["nnzb_L"]), nbranch=int(st["nbranch"]), general=int(st["general"]),
        calls=calls, warmup=warm, symbolic_reused_all=bool(all(reused)),
        host_ms_median=float(np.median(host)), device_ms_median=float(np.median(dev)),
        stats_ms_median=float(np.median(stats_ms)), ba_solve_reduced_ms_median=float(np.median(ba_ms)),
        x_host_vs_device_max_abs=float(np.abs(x_h - x_d.cpu().numpy()).max()),
        x_vs_ba_rel=float(np.abs(x_h - x_ba).max() / np.abs(x_ba).max()))
    print(json.dumps(out))
    chol.close()
    ba.close()


if __name__ == "__main__":
    main()
