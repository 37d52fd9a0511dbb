"""Host clock per keyframe of svs_map_add_keyframe_graph (computeStrength, growth and addNewEdges with the constraints on
the device) against the host-side route it replaces, timed in three parts: svs_map_add_keyframe; computeStrength /
addNewEdges / computeConstraint by the C oracle (oracle/graph_oracle.c, through its ctypes driver, which copies the
graph in and out) on a host mirror of the map; a full svs_map_set_pose_graph upload.  Keeping the mirror itself (the
new vertex's pose read back, the grown observation lists, the per-vertex feature tables) is not timed: a host caller
keeps those in its own tables.  Maps of V = 200 and 1 000 keyframes (mr.make_map, 20 points per keyframe) grow by
`--kf` keyframes of tests/test_graph_gpu.py's generator; both paths must end with the same lists and strengths.
Prints the card and its power limit; --out PATH also writes the record as JSON."""
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
import test_graph_gpu as tg  # noqa: E402
from oracle import graph_pyoracle as gpo  # noqa: E402
from scavislam_b200 import capi  # noqa: E402

THR = 4


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:
        return f"nvidia-smi unavailable ({e})"


def run(V, n_kf, seed):
    m0 = mr.make_map(V, 20, seed=seed)
    rng = np.random.default_rng(seed)
    kfs, m = [], m0
    for _ in range(n_kf):   # the keyframes, generated once on a mirror so both paths see the same input
        kf = tg.make_keyframe(rng, m, len(m["poses"]) - 1, n_track=(100, 200), recent=6, mode="all")
        Vc = len(m["poses"])
        pose = np.asarray(mr._se3_mul(np.asarray(kf["T"], np.longdouble), m["poses"][Vc - 1].astype(np.longdouble)), np.float64)
        m = mr.add_keyframe(m, Vc - 1, pose, kf["new_anchor"], kf["new_xyz"], kf["new_anchor_center"], kf["new_anchor_level"],
                            kf["new_center"], kf["new_level"], kf["track_point"], kf["track_center"], kf["track_level"])
        kfs.append(kf)
    args = lambda kf: {k: kf[k] for k in tg.KF_ARGS}
    dev, host = capi.DeviceMap(device=0), capi.DeviceMap(device=0)
    for dm in (dev, host):
        tg._load(dm, m0)
        tg._set_graph(dm, tg._empty_graph(V))
    t_dev, t_host, edges = [], [], 0
    for kf in kfs:
        Vc = dev.V
        t0 = time.perf_counter()
        _, _, _, ne = dev.add_keyframe_graph(Vc - 1, kf["T"], THR, tg.W, tg.H, **args(kf))
        t_dev.append((time.perf_counter() - t0) * 1e3)
        edges += ne
    m, g = m0, tg._empty_graph(V)
    for kf in kfs:
        Vc = host.V
        t0 = time.perf_counter()
        host.add_keyframe(Vc - 1, kf["T"], **args(kf))
        t1 = time.perf_counter()
        poses, _ = host.get()                              # the mirror, untimed
        m2 = mr.add_keyframe(m, Vc - 1, poses[Vc], kf["new_anchor"], kf["new_xyz"], kf["new_anchor_center"], kf["new_anchor_level"],
                             kf["new_center"], kf["new_level"], kf["track_point"], kf["track_center"], kf["track_level"])
        feat = gpo.feature_tables(m2)
        t2 = time.perf_counter()
        table = gpo.strength_table(m, Vc - 1, kf["new_anchor"], kf["track_point"], kf["track_center"], THR, tg.W, tg.H)
        g = gpo.add_edges(g, m2, *gpo.local_edges(table, THR, Vc), feat=feat)
        t3 = time.perf_counter()
        tg._set_graph(host, g)
        t4 = time.perf_counter()
        m = m2
        t_host.append(((t1 - t0) * 1e3, (t3 - t2) * 1e3, (t4 - t3) * 1e3))
    a = dev.get_graph()
    same = all(np.array_equal(a[k], g[k]) for k in ("nbr_ptr", "nbr_id", "nbr_strength"))
    dev.close(); host.close()
    warm = 2   # the first calls grow the buffers
    h = np.array(t_host[warm:])
    med = lambda x: float(np.median(x))
    return dict(V=V, Np=len(m0["point_anchor"]), keyframes=n_kf, edges_added=edges, lists_equal=bool(same),
                device_ms_median=med(t_dev[warm:]), device_ms_max=float(np.max(t_dev[warm:])),
                host_route_ms_median=dict(add_keyframe=med(h[:, 0]), oracle_bookkeeping=med(h[:, 1]),
                                          set_pose_graph=med(h[:, 2]), total=med(h.sum(1))),
                host_route_ms_max_total=float(np.max(h.sum(1))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    ap.add_argument("--kf", type=int, default=22)
    args = ap.parse_args()
    out = dict(card=card(), device=capi.device_info(), covis_thr=THR, rows=[])
    for V in (200, 1000):
        row = run(V, args.kf, V)
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(card=out["card"], device=out["device"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
