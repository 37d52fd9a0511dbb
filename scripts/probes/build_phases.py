"""Developer probe (GPU box): where k_build_wave's time goes, phase by phase, on C2 (or the configurations named).

With SVS_BUILD_TIMING set (the default here) every warp of k_build_wave reads clock64() at the end of each phase of a
task (a __syncwarp before each read) and adds the differences to d.dbg[48..54]; the library prints those sums, over all
warps and launches of a call, to stderr after the call.  This probe runs one 10-iteration call per configuration,
captures that line and prints each phase's share of the summed warp-cycles, with the GPU's name and power limit.  The
counters serialise the phases of a warp, so the shares say where a warp spends its cycles, not how the phases of
different warps overlap."""
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
os.environ.setdefault("SVS_BUILD_TIMING", "1")
from scavislam_b200 import synth, capi

PHASES = ("setup", "linearise", "landmark-sums", "inverse+Y+spill", "schur+direct", "gradients", "flush")


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


print(capi.device_info(), "| power limit", smi("power.limit"), "| max SM clock", smi("clocks.max.sm"))
ba = capi.BundleAdjuster()
for name in sys.argv[1:] or ("C2",):
    pb = synth.make_config(name)
    ba.set_problem(pb)
    ba.reset_state()
    captured_stderr(lambda: ba.optimize(10))   # warm-up: module load, first launches
    ba.reset_state()
    (it, st), report = captured_stderr(lambda: ba.optimize(10))
    m = re.search(r"k_build_wave warp-cycles[^\n]*", report)
    if not m:
        raise RuntimeError(f"no k_build_wave phase line in the library's report:\n{report}")
    cyc = dict(zip(PHASES, (int(v) for v in re.findall(r"(?<= )-?\d+", m.group(0)))))
    total = sum(cyc.values())
    print(f"{name}: P {pb.P} L {pb.L} E {pb.E}, {it} iterations, {st['trials_total']} trials, "
          f"ms_build per trial {st['ms_build'] / max(st['trials_total'], 1):.4f} (with the counters)")
    for k in PHASES:
        print(f"    {k:16s} {cyc[k]:>16d} warp-cycles  {100.0 * cyc[k] / total:5.1f} %")
