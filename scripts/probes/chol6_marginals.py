"""Developer probe (GPU box): cost of one svs_chol6_solve_blocks / svs_chol6_solve_pattern call.

For each config (default C2, P = 200, and C5, P = 1000) takes the reduced system from
BundleAdjuster.reduced_system(True, 1.0, 50.0), converts it to the upper block CCS g2o's fillCCS(..., true) would give,
and reports medians after a warm-up, with host arrays:
  blocks_*      solve_blocks (the P diagonal blocks of S^-1)
  pattern_*     solve_pattern on the co-visible pairs (every upper block of S, diagonal included)
  solve_*       svs_chol6_solve on the same matrix, for scale
where *_host_ms is the wall time of a call (it ends in a stream synchronise) and *_stats_ms the stats' device time
(scatter + factor + inversion, or + solve).  The GPU name and power limit are read in the same run.
Usage: python scripts/probes/chol6_marginals.py [calls] [config ...]
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


def timed(fn, calls, warm):
    host, dev = [], []
    for k in range(warm + calls):
        t = time.perf_counter()
        res, rc, st = fn()
        dt = time.perf_counter() - t
        assert rc == 0
        if k >= warm:
            host.append(dt * 1e3)
            dev.append(st["ms"])
    return res, st, float(np.median(host)), float(np.median(dev))


def probe(config, calls, warm):
    pb = synth.make_config(config)
    ba = capi.BundleAdjuster(device=0)
    ba.set_problem(pb)
    S, bs, _ = ba.reduced_system(True, 1.0, 50.0)
    ba.close()
    cp, ri, blocks = upper_ccs(S)
    pairs = [(int(ri[k]), j) for j in range(len(cp) - 1) for k in range(cp[j], cp[j + 1])]
    chol = capi.BlockCholesky6(device=0)
    inv_diag, st_b, b_host, b_dev = timed(lambda: chol.solve_blocks(cp, ri, blocks), calls, warm)
    out, st_p, p_host, p_dev = timed(lambda: chol.solve_pattern(cp, ri, blocks, pairs), calls, warm)
    _, st_s, s_host, s_dev = timed(lambda: chol.solve(cp, ri, blocks, bs), calls, warm)
    chol.close()
    Z = np.linalg.inv(S)
    ref = np.array([Z[6 * p:6 * p + 6, 6 * p:6 * p + 6] for p in range(pb.P)])
    return dict(config=config, P=int(pb.P), nnzb_A=int(st_b["nnzb_A"]), nnzb_L=int(st_b["nnzb_L"]),
                nbranch=int(st_b["nbranch"]), general=int(st_b["general"]), n_pairs=len(pairs),
                n_cols_solved=int(st_p["n_cols_solved"]), symbolic_reused=int(st_s["symbolic_reused"]),
                blocks_host_ms=b_host, blocks_stats_ms=b_dev, pattern_host_ms=p_host, pattern_stats_ms=p_dev,
                solve_host_ms=s_host, solve_stats_ms=s_dev,
                blocks_vs_numpy_rel=float(np.abs(inv_diag - ref).max() / np.abs(Z).max()))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    configs = sys.argv[2:] or ["C2", "C5"]
    rows = [probe(c, calls, 20) for c in configs]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), calls=calls, warmup=20,
                          results=rows)))


if __name__ == "__main__":
    main()
