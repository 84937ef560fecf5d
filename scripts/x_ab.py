"""A/B of two builds of the library: another tree (--base, e.g. a checkout of the parent commit with its library built)
against this one.

    python scripts/x_ab.py --out DIR --base TREE [--workload lidar512 ...] [--runs 3] [--steps 20] [--warmup 3] [--late-window 40]

For every workload, runs `bench.py --no-cpu-baseline --other-frames 0 --no-host-mirror` alternately from each tree (each
bench.py imports the fiesta_b200 next to it) with the same flags, `--runs` times per arm, in this one process tree (so both
arms see the same card and the same neighbours).  The first run
of each arm also writes `--dump-outputs`; the arrays of the two arms are compared for bit equality.  Prints the card, its
power limit and clocks, then one line per run and a summary per workload (min / max of EXACT ms per frame and of the late
window, expansions equal to the reference, arrays equal).  Writes the bench lines to DIR/ab.jsonl; the dumped arrays go
to a temporary directory that is removed at the end.  Needs a GPU.
"""
import argparse
import glob
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "nvidia-smi not found"


def run(wl, tree, args, dump):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--workload", wl, "--no-cpu-baseline", "--other-frames", "0", "--no-host-mirror", "--late-window", str(args.late_window)]
    if dump:
        cmd += ["--dump-outputs", dump]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=tree)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode or not lines:
        sys.stderr.write(p.stderr[-4000:])
        raise SystemExit("bench.py failed (%s, %s): exit %d" % (wl, tree, p.returncode))
    return json.loads(lines[-1])


def same_arrays(d0, d1):
    names = sorted(os.path.basename(f) for f in glob.glob(os.path.join(d0, "*.npy")))
    if not names or names != sorted(os.path.basename(f) for f in glob.glob(os.path.join(d1, "*.npy"))):
        return False, names
    diff = [n for n in names if not np.array_equal(np.load(os.path.join(d0, n)), np.load(os.path.join(d1, n)))]
    return not diff, diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--base", required=True, help="the other tree, with its library built")
    ap.add_argument("--workload", action="append")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--late-window", type=int, default=40)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card(), flush=True)
    log = open(os.path.join(args.out, "ab.jsonl"), "a")
    tmp = tempfile.mkdtemp(prefix="x_ab_")                   # the dumped arrays are large: compared here, then deleted
    trees = {"base": os.path.abspath(args.base), "head": ROOT}
    print("base:", trees["base"], "head:", ROOT, flush=True)
    for wl in args.workload or ["lidar512"]:
        res = {arm: [] for arm in trees}
        for k in range(args.runs):
            for arm, tree in trees.items():
                dump = os.path.join(tmp, "dump_%s_%s" % (wl, arm)) if k == 0 else None
                line = run(wl, tree, args, dump)
                line["arm"] = arm
                log.write(json.dumps(line) + "\n"); log.flush()
                lw = line.get("late_window") or {}
                res[arm].append((line["ms_per_step"], lw.get("ms_per_step"), line["expansions_equal_reference"], lw.get("expansions_equal_reference")))
                print("%s run %d %s: %.3f ms/frame, late_window %s ms/frame, expansions_equal_reference %s / %s, clocks %s" %
                      (wl, k, arm, line["ms_per_step"], "%.3f" % lw["ms_per_step"] if lw else "-", line["expansions_equal_reference"],
                       lw.get("expansions_equal_reference"), json.dumps(line.get("clocks"))), flush=True)
        eq, diff = same_arrays(os.path.join(tmp, "dump_%s_base" % wl), os.path.join(tmp, "dump_%s_head" % wl))
        for arm in trees:
            ms = [r[0] for r in res[arm]]
            late = [r[1] for r in res[arm] if r[1] is not None]
            print("%s %s: ms/frame min %.3f max %.3f; late_window min %s max %s; expansions equal %s" %
                  (wl, arm, min(ms), max(ms), "%.3f" % min(late) if late else "-", "%.3f" % max(late) if late else "-",
                   all(r[2] is not False and r[3] is not False for r in res[arm])), flush=True)
        print("%s dumped arrays bit-identical between the arms: %s%s" % (wl, eq, "" if eq else " (differ: %s)" % diff), flush=True)
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
