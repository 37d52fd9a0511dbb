"""Time of one svs_globalLoopClosure (Backend::globalLoopClosure) at the back-end's operating point: a map of 200
keyframes (the rendered revisit of scavislam_b200/synth_loop.py, padded with keyframes that anchor 250 points each and
that the query does not see), a query with several hundred observations, 2 pyramid levels at 640x480.  Prints the host
clock of a call (it ends in a device synchronise), the per-kernel device times of one call from torch.profiler, the
CPU oracle's time for the same call, and the card with its power limit.  --out PATH also writes the record as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import loop_pyoracle as lo, pyoracle as po  # noqa: E402
from scavislam_b200 import capi, synth_loop as sl  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:
        return f"nvidia-smi unavailable ({e})"


def padded_map(m, V_total, per_kf, rng):
    """m with V_total - V keyframes appended, each anchoring per_kf points seen by itself and its successor."""
    V = len(m["poses"])
    poses = [m["poses"]]
    anchor, xyz, vp, vs, cen, lvl = [m["point_anchor"]], [m["xyz_anchor"]], [m["vis_ptr"]], [m["vis_pose"]], [m["feat_center"]], [m["feat_level"]]
    nnz = len(m["vis_pose"])
    for k in range(V, V_total):
        poses.append(np.array([[0, 0, 0, 1, 0.1 * k, 0, 0]]))
        anchor.append(np.full(per_kf, k, np.int32))
        xyz.append(np.stack([rng.uniform(-3, 3, per_kf), rng.uniform(-2, 2, per_kf), rng.uniform(2, 20, per_kf)], 1))
        obs = np.full(per_kf, 2 if k + 1 < V_total else 1)
        vp.append(nnz + np.cumsum(obs).astype(np.int32))
        nnz += int(obs.sum())
        for n in obs:
            vs.append(np.array([k, k + 1][:n], np.int32))
            cen.append(rng.uniform(0, 480, (n, 3)))
            lvl.append(rng.integers(0, 2, n).astype(np.int32))
    return dict(poses=np.concatenate(poses), point_anchor=np.concatenate(anchor), xyz_anchor=np.concatenate(xyz),
                vis_ptr=np.concatenate(vp).astype(np.int32), vis_pose=np.concatenate(vs), feat_center=np.concatenate(cen),
                feat_level=np.concatenate(lvl))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the record as JSON to this file")
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    sc = sl.make_scene(po, per_level=(400, 150))
    rng = np.random.default_rng(3)
    m = padded_map(sc["map"], 200, 250, rng)
    V, Np = len(m["poses"]), len(m["point_anchor"])
    slot = -np.ones(V, np.int32)
    verts = list(sc["window"]) + [sc["loop"]]
    for s, v in enumerate(verts):
        slot[v] = s
    lf = sc["frames"][sc["loop"]]
    q_obs = int(sum(sc["query"] in m["vis_pose"][m["vis_ptr"][p]:m["vis_ptr"][p + 1]] for p in range(len(sc["map"]["point_anchor"]))))
    out = dict(card=card(), device=capi.device_info(), V=V, Np=Np, nnz=len(m["vis_pose"]), query_observations=q_obs)

    def fresh():
        dm = capi.DeviceMap(device=0)
        dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
        return dm

    mt = capi.GuidedMatcher(sc["levels"], max_keyframes=len(verts), max_points=8192, device=0)
    for s, v in enumerate(verts):
        mt.set_keyframe(s, m["poses"][v], sc["frames"][v]["pyr"])
    mt.set_current(lf["pyr"], lf["disp"])
    for l, (xy, c) in enumerate(sc["loop_features"]):
        mt.set_features(l, xy, c)
    pz = capi.PoseOptimizer(max_obs=8192, device=0)
    args_ = (mt, pz, sc["cam"], 20, sc["query"], sc["loop"], sc["T_query_from_loop"], sc["window"], slot)
    dm = fresh()
    res, _ = dm.global_loop_closure(*args_)                       # warm-up (module load); grows the map once
    out["result"] = {k: v for k, v in res.items() if not k.startswith("T") and k != "lm"}
    times = []
    for _ in range(args.reps):                                    # on the grown map: the same work, no further growth
        t0 = time.perf_counter()
        dm.global_loop_closure(*args_)
        times.append((time.perf_counter() - t0) * 1e3)
    out["host_ms_median"] = float(np.median(times))
    out["host_ms_min"] = float(np.min(times))
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        dm.global_loop_closure(*args_)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) > 0:
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            kern[e.name] = kern.get(e.name, 0.0) + t / 1e3
    out["kernel_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:20])
    t0 = time.perf_counter()
    lo.global_loop_closure(m, sc["levels"], lf["pyr"], lf["disp"], sc["loop_features"], [sc["frames"][v]["pyr"] for v in verts],
                           sc["cam"], 20, sc["query"], sc["loop"], sc["T_query_from_loop"], sc["window"], slot)
    out["oracle_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    dm.close(); mt.close(); pz.close()


if __name__ == "__main__":
    main()
