"""Developer probe (GPU box): the overlap timeline of one C2 trial -- when each block column of the reduced system became
complete in k_build_wave, and when k_solve's chain published it -- and what running the solve alongside the build could
gain (DESIGN.md 8, work list).

    python scripts/probes/overlap_timeline.py [--config C2] [--every 10]

Runs the library in a child process with SVS_SOLVE_TIMING=3 (the knob is read once, when the library loads) and parses
the timeline it prints for the last trial of a 10-iteration call.  Times are microseconds since the first k_build_wave
CTA entered (the solve runs after the build, so every chain time lies behind every ready time).  `head`: the moment the
first four columns of every branch are complete, which is the least a solve running alongside the build would wait
before its first column; per branch it also counts the columns that became complete before the one in front of them.
"""
import argparse
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CHILD = r"""
import sys
sys.path.insert(0, {root!r})
from scavislam_b200 import capi, synth
ba = capi.BundleAdjuster()
pb = synth.make_config({cfg!r})
ba.set_problem(pb)
for _ in range(3):
    ba.reset_state()
    it, st = ba.optimize(10)
print("STATS", st["ms_total"], st["ms_build"], st["ms_solve"], st["ms_update"], st["trials_total"], flush=True)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--every", type=int, default=10, help="print every n-th column of a branch")
    args = ap.parse_args()
    env = dict(os.environ, SVS_SOLVE_TIMING="3")
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=ROOT, cfg=args.config)], env=env,
                       capture_output=True, text=True, check=True)
    # the timeline of the LAST call (the library prints one per call)
    blocks = r.stderr.split("overlap timeline:")
    last = blocks[-1]
    head_line = last.splitlines()[0]
    m = re.search(r"branches (\d+) solve_entry_us (\S+)", head_line)
    nbranch, solve_entry = int(m.group(1)), float(m.group(2))
    cols = []
    for line in last.splitlines()[1:]:
        mm = re.match(r"\s+col (\d+) group (\d+) pos (\d+) ready_us (\S+) chain_us (\S+)", line)
        if not mm:
            break
        cols.append((int(mm.group(1)), int(mm.group(2)), int(mm.group(3)), float(mm.group(4)), float(mm.group(5))))
    stats = [ln for ln in r.stdout.splitlines() if ln.startswith("STATS")][-1].split()[1:]
    ms_total, ms_build, ms_solve, ms_update, trials = (float(x) for x in stats)
    print(f"{args.config}: branches={nbranch} solve entry {solve_entry:+.1f} us after the build's")
    print(f"per trial: ms_total {ms_total / trials:.4f}  ms_build {ms_build / trials:.4f}  ms_solve {ms_solve / trials:.4f}"
          f"  ms_update {ms_update / trials:.4f}  ({int(trials)} trials)")
    t0 = 0.0
    heads = []
    for g in range(nbranch + 1):
        part = [c for c in cols if c[1] == g]
        if not part:
            continue
        name = f"branch {g}" if g < nbranch else "separator"
        print(f"{name}: {len(part)} columns   pos  ready_us  chain_us  slack_us (chain - ready)")
        for c in part:
            if c[2] % args.every == 0 or c is part[-1]:
                print(f"    {c[2]:4d}  {c[3] - t0:8.1f}  {c[4] - t0:8.1f}  {c[4] - c[3]:8.1f}")
        if g < nbranch:
            heads.append(max(c[3] for c in part[:4]) - t0)
        ahead = sum(1 for a, b in zip(part, part[1:]) if b[3] < a[3])
        print(f"    columns complete before the column in front of them: {ahead} of {len(part) - 1}; last column complete "
              f"at {max(c[3] for c in part) - t0:.1f} us; chain from {part[0][4] - t0:.1f} to {part[-1][4] - t0:.1f} us")
    print(f"head (first four columns of every branch complete): {max(heads):.1f} us")


if __name__ == "__main__":
    main()
