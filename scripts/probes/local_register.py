"""Time of one svs_localRegisterFrame (Backend::localRegisterFrame) at the back-end's operating point: a map of 200
keyframes (the revisit inside the double window of scavislam_b200/synth_loop.make_register_scene, padded with keyframes
that anchor 250 points each, chained to one another but not to the scene), the whole map as the window, 2 pyramid levels
at 640x480.  Prints the host clock of a call (it ends in a device synchronise), the per-kernel device times of one call
from torch.profiler, the CPU oracle's time for the same call, and the card with its power limit.  --out PATH also writes
the record as JSON."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from loop_closure import card, padded_map  # noqa: E402
from oracle import pyoracle as po, register_pyoracle as ro  # noqa: E402
from scavislam_b200 import capi, synth_loop as sl  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    sc = sl.make_register_scene(po, per_level=(400, 150))
    rng = np.random.default_rng(3)
    V0 = len(sc["map"]["poses"])
    m = padded_map(sc["map"], 200, 250, rng)
    V, Np = len(m["poses"]), len(m["point_anchor"])
    nbr = [list(sc["nbr_id"][sc["nbr_ptr"][v]:sc["nbr_ptr"][v + 1]]) for v in range(V0)]
    nbr += [[j for j in (v + 1, v - 1) if V0 <= j < V] for v in range(V0, V)]
    nbr_ptr = np.cumsum([0] + [len(n) for n in nbr]).astype(np.int32)
    nbr_id = np.array(sum(nbr, []), np.int32)
    window = np.arange(V, dtype=np.int32)
    slot = -np.ones(V, np.int32)
    slot[:V0] = np.arange(V0)
    rf = sc["frames"][sc["root"]]
    out = dict(card=card(), device=capi.device_info(), V=V, Np=Np, nnz=len(m["vis_pose"]), scene_keyframes=V0)

    mt = capi.GuidedMatcher(sc["levels"], max_keyframes=V0, max_points=8192, device=0)
    for v in range(V0):
        mt.set_keyframe(v, m["poses"][v], sc["frames"][v]["pyr"])
    mt.set_current(rf["pyr"], rf["disp"])
    for l, (xy, c) in enumerate(sc["root_features"]):
        mt.set_features(l, xy, c)
    pz = capi.PoseOptimizer(max_obs=8192, device=0)
    dm = capi.DeviceMap(device=0)
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_graph(nbr_ptr, nbr_id)
    args_ = (mt, pz, sc["cam"], 20, sc["root"], window, slot)
    res, _, _ = dm.local_register_frame(*args_)                   # warm-up (module load); grows the map once
    out["result"] = {k: v for k, v in res.items() if not k.startswith("T") and k != "lm"}
    times = []
    for _ in range(args.reps):                                    # on the grown map: the same work, no further growth
        t0 = time.perf_counter()
        dm.local_register_frame(*args_)
        times.append((time.perf_counter() - t0) * 1e3)
    out["host_ms_median"] = float(np.median(times))
    out["host_ms_min"] = float(np.min(times))
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        dm.local_register_frame(*args_)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if e.device_type.name == "CUDA" and t > 0:
            kern[e.name] = kern.get(e.name, 0.0) + t / 1e3
    out["kernel_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:20])
    t0 = time.perf_counter()
    ro.local_register_frame(m, nbr_ptr, nbr_id, sc["levels"], rf["pyr"], rf["disp"], sc["root_features"],
                            [sc["frames"][v]["pyr"] for v in range(V0)], sc["cam"], 20, sc["root"], window, slot)
    out["oracle_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    dm.close(); mt.close(); pz.close()


if __name__ == "__main__":
    main()
