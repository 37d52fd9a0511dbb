"""Developer probe (GPU box): C2/C5 timing breakdown of the BA kernels + k_solve phase cycles.

With SVS_SOLVE_TIMING=1 (the default here) the library reports, for the last trial of a call, the phase boundaries of
both CTAs of k_solve (d.dbg[0..11], cycles since the end of the setup) and the setup itself (from the CTA's first
instruction past griddepcontrol.wait to the end of the setup).  This probe captures that report and prints it as a
table of phase lengths in microseconds at the SM clock nvidia-smi reports, with the GPU's name and power limit."""
import os
import re
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
from scavislam_b200 import synth, capi
from oracle import pyoracle as po

os.environ.setdefault("SVS_SOLVE_TIMING", "1")
PHASES = ("setup", "branch factored", "cluster sync #1", "separators factored", "separators solved + sync #2",
          "branch solved (with the pose update)", "reduction + sync #3")


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def captured_stderr(fn):
    """Runs fn() with file descriptor 2 redirected to a temporary file; returns (fn's result, the text written)."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        try:
            out = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return out, f.read().decode(errors="replace")


def phase_table(report, mhz):
    """Phase lengths (us) per CTA from the library's 'CTA g: b1 .. b6 setup s' lines."""
    rows = {}
    for g, rest in re.findall(r"CTA (\d): ([^\n]*)", report):
        nums = [int(v) for v in re.findall(r"-?\d+", rest)]
        if len(nums) < 7:
            continue
        bounds, setup = [0] + nums[:6], nums[6]
        rows[int(g)] = [setup] + [bounds[i + 1] - bounds[i] for i in range(6)]
    for g in sorted(rows):
        us = [c / mhz for c in rows[g]]
        print(f"    CTA {g}: " + ", ".join(f"{n} {u:.1f}" for n, u in zip(PHASES, us)) + f"; total {sum(us):.1f} us")
    return rows


ba = capi.BundleAdjuster()
mhz = float(re.sub(r"[^0-9.]", "", smi("clocks.max.sm")) or 1980.0)
print(capi.device_info(), "| power limit", smi("power.limit"), "| max SM clock", mhz, "MHz")
def rel(a, b): return np.abs(a - b).max() / np.abs(b).max()
for name in sys.argv[1:] or ("C2", "C5"):
    pb = synth.make_config(name)
    t = time.time(); ba.set_problem(pb); t_set = time.time() - t
    for rep in range(3):
        ba.reset_state()
        t = time.time(); (it, st), report = captured_stderr(lambda: ba.optimize(10)); dt = time.time() - t
    print(name, "P L E C", pb.P, pb.L, pb.E, pb.C, "set_problem s", t_set, "optimize wall s", dt, "iters", it)
    print("   ", {k: st[k] for k in ("ms_total", "ms_build", "ms_solve", "ms_update", "ms_control", "launches", "nnzb_S", "nnzb_L", "max_track", "trials_total")})
    print("    k_solve phases of the last trial (us at %.0f MHz):" % mhz)
    phase_table(report, mhz)
    print("    " + report.strip().replace("\n", "\n    "))
    t = time.time(); p_o, s_o, sto = po.optimize(pb, 10); dto = time.time() - t
    print("    oracle s", dto, "it/s", sto["iterations"] / dto, "pose rel", rel(ba.poses(), p_o), "psi rel", rel(ba.points(), s_o))
    print("    chi gpu", st["chi2_iter"][-1], "cpu", sto["chi2_iter"][-1])
