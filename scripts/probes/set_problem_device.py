"""Developer probe (GPU box): what the device structure analysis of svs_ba_set_problem_device costs.

  1. set_problem on C2 and C5 from CUDA tensors against host arrays: a new structure every call (two windows with
     different edge lists, alternating, as e2e_host_phases.py does) and the same structure again.  Wall time per call
     until the handle's stream is idle (a 7P-double read-back of the poses closes every call on both paths).
  2. A back-end tick from the device map -- select_window -> set_problem_from_map -> optimize(2) -> absorb -- with this
     tree's library and, with --parent DIR, with an older build of the package (DIR/scavislam_b200, library included),
     run in alternating subprocesses.

Medians after warm-up.  The card's name, power limit and maximum SM clock are printed with the numbers.
usage: python scripts/probes/set_problem_device.py [--parent DIR] [--reps N]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # (the numbers still stand; say why the card is unnamed)
        return f"nvidia-smi unavailable: {e}"


def set_problem_times(name, reps):
    import numpy as np
    import torch
    from scavislam_b200 import capi, synth
    import ctypes as C
    pb = synth.make_config(name)
    pb2 = synth.with_dropouts(pb, 0.02, seed=5)

    def cuda(p):
        kw = dict(p.__dict__)
        for k in ("pose_qt", "fixed", "psi", "e_point", "e_pose", "e_anchor", "e_obs", "e_info", "c_i", "c_j", "c_T", "c_Lambda"):
            kw[k] = torch.from_numpy(np.ascontiguousarray(kw[k])).cuda()
        return synth.BAProblem(**kw)

    out = {}
    for mode in ("host", "device"):
        ba = capi.BundleAdjuster()
        poses = np.zeros((pb.P, 7))
        wins = (pb, pb2) if mode == "host" else (cuda(pb), cuda(pb2))
        for case in ("new_structure", "same_structure"):
            ts = []
            for r in range(reps + 3):
                w = wins[r & 1] if case == "new_structure" else wins[0]
                t = time.perf_counter()
                ba.set_problem(w)
                capi.lib().svs_ba_get_poses(ba._h, poses.ctypes.data_as(C.POINTER(C.c_double)))
                if r >= 3:
                    ts.append(time.perf_counter() - t)
            out[f"{mode}_{case}_ms"] = 1e3 * float(np.median(ts))
        ba.close()
    return out


def make_tick_inputs(name, path):
    import numpy as np
    from scavislam_b200 import synth, synth_graph
    pb = synth.make_config(name)
    m, win, act = synth_graph.make_map(pb, seed=1)
    ptr, ids, T, Lm = synth_graph.make_pose_graph(m, seed=1)
    np.savez(path, win=win, ptr=ptr, ids=ids, T=T, Lm=Lm, **m)


def tick_times(name, reps, inputs):
    """One process: median wall time of a from-map back-end tick with whichever scavislam_b200 is first on sys.path."""
    import numpy as np
    from scavislam_b200 import capi, synth
    pb = synth.make_config(name)
    z = np.load(inputs)
    m, win, ptr, ids, T, Lm = z, z["win"], z["ptr"], z["ids"], z["T"], z["Lm"]
    dm, ba = capi.DeviceMap(), capi.BundleAdjuster()
    dm.set(m["poses"], m["point_anchor"], m["xyz_anchor"], m["vis_ptr"], m["vis_pose"], m["feat_center"], m["feat_level"])
    dm.set_graph(ptr, ids, T, Lm)
    root = int(win[pb.P // 2])
    ts = []
    for r in range(reps + 3):
        t = time.perf_counter()
        sel = dm.select_window(root, 10, pb.P)
        dm.set_problem(ba, sel["window_vertex"], sel["active_point"], pb.cam, c_i=sel["c_i"], c_j=sel["c_j"],
                       c_T=sel["c_T"], c_Lambda=sel["c_Lambda"])
        ba.optimize(2)
        dm.absorb(ba)
        if r >= 3:
            ts.append(time.perf_counter() - t)
    return {"P": len(sel["window_vertex"]), "L": len(sel["active_point"]), "tick_ms": 1e3 * float(np.median(ts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tick", default=None)     # internal: one tick measurement in this process
    ap.add_argument("--inputs", default=None)   # internal: the map and pose graph of that measurement (.npz)
    a = ap.parse_args()
    if a.tick:
        print(json.dumps(tick_times(a.tick, a.reps, a.inputs)))
        return
    sys.path.insert(0, ROOT)
    print("card:", card())
    for name in ("C2", "C5"):
        print(name, "set_problem", json.dumps(set_problem_times(name, a.reps)), flush=True)
    sides = [("this", ROOT)] + ([("parent", os.path.abspath(a.parent))] if a.parent else [])
    tmp_dir = tempfile.TemporaryDirectory()
    tmp = tmp_dir.name
    for name in ("C2", "C5"):
        inputs = os.path.join(tmp, name + ".npz")
        make_tick_inputs(name, inputs)
        res = {s: [] for s, _ in sides}
        for rnd in range(3):
            for s, path in (sides if rnd % 2 == 0 else sides[::-1]):
                env = dict(os.environ, PYTHONPATH=path)
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--tick", name, "--reps", str(a.reps),
                                    "--inputs", inputs],
                                   capture_output=True, text=True, env=env, cwd=path)
                if r.returncode:
                    raise RuntimeError(r.stderr[-2000:])
                res[s].append(json.loads(r.stdout.strip().splitlines()[-1]))
        print(name, "from-map tick", json.dumps(res), flush=True)
    print("card:", card())


if __name__ == "__main__":
    main()
