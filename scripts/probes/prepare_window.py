"""Host clock per svs_map_prepare_for_optimization (the window, reinitializePoses and the (un)marginalisation with the
re-marginalised constraints, on the device) against the host route it replaces: svs_map_get_graph + svs_map_get, the
C oracle's prepare (oracle/prepare_oracle.c through its ctypes driver, window selection by oracle/pyoracle.py), then
svs_map_set_pose_graph + svs_map_update_poses.  The host route keeps the window and the flags in its own arrays.  Maps
of V = 200 and 1 000 keyframes (mr.make_map, 20 points per keyframe) with a covisibility pose graph whose constraints
are computeConstraint's; windows (15, 100) and (30, 200); the root slides one keyframe per call.  Both routes must end
with the same graph, flags and poses.  Prints the card and its power limit; --out PATH also writes the record as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import map_reference as mr  # noqa: E402
from oracle import graph_pyoracle as gpo  # noqa: E402
from oracle import prepare_pyoracle as ppo  # noqa: E402
from scavislam_b200 import capi  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:
        return f"nvidia-smi unavailable ({e})"


def _load(dm, m, g):
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_pose_graph(g["nbr_ptr"], g["nbr_id"], g["nbr_strength"], g["nbr_T"], g["nbr_Lambda"])


def run(V, inner, dbl, calls):
    m = mr.make_map(V, 20, seed=V)
    ptr, ids, _, _ = mr.covisibility_graph(m, max_neighbours=6, with_constraints=False)
    fptr, fpt = gpo.feature_tables(m)
    src = np.repeat(np.arange(V), np.diff(ptr))
    T, L, st = gpo.constraints(m["poses"], fptr, fpt, m["point_anchor"], m["xyz_anchor"], ids, src)
    g0 = dict(nbr_ptr=ptr, nbr_id=ids, nbr_strength=np.zeros(len(ids), np.int32), nbr_T=T, nbr_Lambda=L)
    dev, host = capi.DeviceMap(device=0), capi.DeviceMap(device=0)
    _load(dev, m, g0)
    _load(host, m, g0)
    roots = [V // 2 + k for k in range(calls)]
    t_dev = []
    for r in roots:
        t0 = time.perf_counter()
        dev.prepare_for_optimization(r, -1, inner, dbl)
        t_dev.append((time.perf_counter() - t0) * 1e3)
    wt, mg = np.zeros(V, np.int32), np.ones(len(ids), np.uint8)
    t_host = []
    for r in roots:
        t0 = time.perf_counter()
        g = host.get_graph()
        poses, _ = host.get()
        ref = ppo.prepare_for_optimization(g, mg, wt, dict(m, poses=poses), r, -1, inner, dbl, feat=(fptr, fpt))
        gr = ref["graph"]
        host.set_pose_graph(gr["nbr_ptr"], gr["nbr_id"], gr["nbr_strength"], gr["nbr_T"], gr["nbr_Lambda"])
        host.update_poses(np.arange(V), ref["poses"])
        t_host.append((time.perf_counter() - t0) * 1e3)
        wt, mg = ref["window_type"].astype(np.int32), ref["marginalized"]
    a, b = dev.get_graph(), host.get_graph()
    wd, md = dev.window_state()
    pd, ph = dev.get()[0], host.get()[0]
    same = (all(np.array_equal(a[k], b[k]) for k in ("nbr_ptr", "nbr_id", "nbr_strength")) and np.array_equal(wd, wt)
            and np.array_equal(md, mg))
    dT = float(np.abs(a["nbr_T"] - b["nbr_T"]).max())
    dL = float((np.abs(a["nbr_Lambda"] - b["nbr_Lambda"]) / np.maximum(np.abs(b["nbr_Lambda"]), 1.0)).max())
    dP = float(np.abs(pd - ph).max())
    dev.close(); host.close()
    warm = 2   # the first calls grow the buffers
    med = lambda x: float(np.median(x[warm:]))
    return dict(V=V, Np=len(m["point_anchor"]), nnzN=len(ids), inner=inner, double=dbl, calls=calls, same_graph_flags_window=bool(same),
                max_abs_dT=dT, max_rel_dLambda=dL, max_abs_dpose=dP, device_ms_median=med(t_dev),
                device_ms_max=float(np.max(t_dev[warm:])), host_route_ms_median=med(t_host))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    ap.add_argument("--calls", type=int, default=12)
    args = ap.parse_args()
    out = dict(card=card(), device=capi.device_info(), rows=[])
    for V in (200, 1000):
        for inner, dbl in ((15, 100), (30, 200)):
            row = run(V, inner, dbl, args.calls)
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(dict(card=out["card"], device=out["device"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
