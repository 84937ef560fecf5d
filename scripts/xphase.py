"""Phase split of k_x_relax (EXACT UpdateESDF) over the frames bench.py times.

    python scripts/xphase.py [--workload lidar512] [--warmup 3] [--steps 20] [--out FILE]

Runs frames 0 .. warmup+steps-1 of the workload in EXACT mode with FIESTA_DEBUG_X=1 (the kernel then times its phases with
clock64; the library converts cycles with the device's SM clock) and sums, over the timed frames warmup .. warmup+steps-1:
the time of every phase, the evaluation rounds and the work-list entries evaluated and refreshed.  The re-seeding of the
dependants of deleted obstacles (k_x_reseed) is split into its stages: classify, closure, choose, resolve and the hand-over
to generation 0 (assemble); per frame it prints the dependants, those final after the classification, the closure rounds,
the closure list entries and the resolve passes.  It also prints, per frame, the (nE, rounds) list of every generation.  The numbers of generations and every nE
are fixed by the sequential result; rounds and list lengths vary from run to run (a round reads words flipped in the same
round).  For the evaluation-round categories it also splits the time into the summed longest CTA work time of every round
and the rest (grid barrier plus waiting for the slowest CTA), with a log2 histogram of the list lengths of SMALL
generations' later rounds, and it sums the counters of the asynchronous schedule (the work queue of BIG generations,
phase "async").  SMALL generations (at most
FIESTA_X_SMALL entries, default 32768) are summarised over the timed frames by log2 size bucket: count, rounds (a queue
phase counts as one) and time per generation.  The card, its power limit and the SM clock are printed first.  The output is
plain text, one item per line, so two runs can be diffed.  Needs a GPU, except with --from-trace FILE, which reads the
library's stderr trace of an earlier child run (python scripts/xphase.py --child ... 2> FILE with FIESTA_DEBUG_X=1).
"""
import argparse
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["S", "round1", "dense", "commit", "apply", "s.round1", "s.rounds", "s.commit", "s.apply", "top",
          "empty-barrier", "reseed.classify", "reseed.closure", "reseed.choose", "reseed.resolve", "reseed.assemble", "async",
          "refresh"]
ROUND_CATS = ["round1", "dense", "s.round1", "s.rounds"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "nvidia-smi not found"


def child(wl, nframes):
    """Runs the frames; the library writes its [x] lines to stderr, each frame is preceded by a marker line."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import bench
    import fiesta_b200
    from tests import scenes
    w = bench.WORKLOADS[wl]
    frames = bench.make_frames(wl, nframes)
    m = fiesta_b200.ESDFMap(w["origin"], w["res"], w["size"], device=0, mode="exact")
    m.SetParameters(*bench.wl_params(wl))
    if w["kind"] == "stress":
        allv = scenes.all_voxels(m.grid_size)
        m.SetOccupancyBatchVox(allv, np.zeros(len(allv), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    dparams = fiesta_b200.DepthParams(scenes.FX, scenes.FY, scenes.CX, scenes.CY, *w["filter"]) if w["kind"] == "depth" else None
    for f, fr in enumerate(frames):
        sys.stderr.write("[frame] %d\n" % f); sys.stderr.flush()
        if w["kind"] == "lidar":
            m.RaycastFrame(fr["pts"], fr["T"], w["min_len"], w["max_len"])
        elif w["kind"] == "depth":
            m.DepthFrame(fr["img"], dparams, fr["T"], fr["m_rel"], w["min_len"], w["max_len"])
        else:
            m.SetOccupancyBatchVox(fr["vox"], fr["occ"])
        if m.CheckUpdate():
            m.SetOriginalRange(); m.UpdateOccupancy(True); m.UpdateESDF()
        m.synchronize()
        sys.stderr.write("[expansions] %d\n" % m.stats()["expansions"]); sys.stderr.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="lidar512")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", help="also write the report to this file")
    ap.add_argument("--from-trace", help="summarise this saved trace instead of running the frames")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.workload, args.warmup + args.steps)
        return
    if args.from_trace:
        trace = open(args.from_trace).read()
    else:
        env = dict(os.environ, FIESTA_DEBUG_X="1")
        cmd = [sys.executable, os.path.abspath(__file__), "--child", "--workload", args.workload, "--warmup", str(args.warmup), "--steps", str(args.steps)]
        p = subprocess.run(cmd, env=env, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
        if p.returncode:
            sys.stderr.write(p.stderr[-4000:])
            raise SystemExit(p.returncode)
        trace = p.stderr
    lo, hi = args.warmup, args.warmup + args.steps
    small_max = int(os.environ.get("FIESTA_X_SMALL", "32768"))
    small = {}                                                 # log2 bucket of nE -> [generations, rounds, us]
    us = {k: 0.0 for k in PHASES}
    tot = dict(rounds=0, evaluated=0, refreshed=0, reseed_rounds=0, dependants=0, final_after_classify=0, closure_rounds=0,
               closure_entries=0, resolve_passes=0, generations=0, expansions=0)
    reseed = {}                                                # frame -> (dependants, final, closure rounds, entries, passes)
    work = {k: [0.0, 0] for k in ROUND_CATS}
    hist = {"s.rounds": {}}
    aq = dict(evaluations=0, dirty=0, pushes=0, spin_us=0.0)
    gens = {}
    f = -1
    for line in trace.splitlines():
        if line.startswith("[frame] "):
            f = int(line.split()[1]); gens[f] = []
            continue
        if not lo <= f < hi:
            if line.startswith("[x] gens "):
                gens[f] = [tuple(int(v) for v in t.split("/")[:2]) for t in line.split("|", 1)[1].split()]
            continue
        if line.startswith("[expansions] "):
            tot["expansions"] += int(line.split()[1])
        elif line.startswith("[x] reseed rounds"):
            tot["reseed_rounds"] += int(re.match(r"\[x\] reseed rounds (\d+)", line).group(1))
            for name, t, _ in re.findall(r" (\S+) ([\d.]+)/(\d+)", line.split(":", 1)[1]):
                us[name] += float(t)
        elif line.startswith("[x] round work"):
            for name, t, n in re.findall(r" (\S+) ([\d.]+)/(\d+)", line.split(":", 1)[1]):
                work[name][0] += float(t); work[name][1] += int(n)
        elif line.startswith("[x] list-length histogram "):
            name = line.split()[3]
            for b, c in re.findall(r" (\d+)=(\d+)", line.split(":", 1)[1]):
                hist[name][int(b)] = hist[name].get(int(b), 0) + int(c)
        elif line.startswith("[x] async:"):
            mm = re.search(r"evaluations (\d+) dirty (\d+) pushes (\d+) spin ([\d.]+)", line)
            aq["evaluations"] += int(mm.group(1)); aq["dirty"] += int(mm.group(2)); aq["pushes"] += int(mm.group(3))
            aq["spin_us"] += float(mm.group(4))
        elif line.startswith("[x] work-list entries:"):
            mm = re.search(r"evaluated (\d+) refreshed (\d+)", line)
            tot["evaluated"] += int(mm.group(1)); tot["refreshed"] += int(mm.group(2))
        elif line.startswith("[x] reseed:"):
            v = tuple(int(t) for t in re.findall(r"\d+", line))
            reseed[f] = v
            for k, n in zip(("dependants", "final_after_classify", "closure_rounds", "closure_entries", "resolve_passes"), v):
                tot[k] += n
        elif line.startswith("[x] gens "):
            mm = re.match(r"\[x\] gens (\d+) rounds (\d+)", line)
            tot["generations"] += int(mm.group(1)); tot["rounds"] += int(mm.group(2))
            gens[f] = [tuple(int(v) for v in t.split("/")[:2]) for t in line.split("|", 1)[1].split()]
            for t in line.split("|", 1)[1].split():
                n, r, t_us = t.split("/")
                if int(n) <= small_max:
                    b = small.setdefault(int(n).bit_length(), [0, 0, 0.0])
                    b[0] += 1; b[1] += int(r); b[2] += float(t_us[:-2])
    out = ["card: " + card() if not args.from_trace else "trace: " + args.from_trace,
           "workload %s, frames %d-%d, phase totals of k_x_relax (ms):" % (args.workload, lo, hi - 1)]
    for k in PHASES:
        if k != "empty-barrier":
            out.append("  %-16s %9.2f" % (k, us[k] / 1000.0))
    out.append("  %-16s %9.2f" % ("sum", sum(v for k, v in us.items() if k != "empty-barrier") / 1000.0))
    out.append("  %-16s %9.2f us per empty grid barrier (mean over the frames)" % ("empty-barrier", us["empty-barrier"] / max(1, hi - lo)))
    out.append("evaluation rounds (ms): wall = summed longest CTA work + barrier and idle; list entries")
    for k in ROUND_CATS:
        wall = us[k] / 1000.0
        wmax = work[k][0] / 1000.0
        out.append("  %-10s wall %9.2f work %9.2f barrier+idle %9.2f (%5.1f %%) entries %d" %
                   (k, wall, wmax, wall - wmax, 100.0 * (wall - wmax) / wall if wall else 0.0, work[k][1]))
    for name, h in hist.items():
        out.append("list lengths of %s, rounds per log2 bucket [2^(b-1), 2^b): %s" % (name, " ".join("%d:%d" % kv for kv in sorted(h.items()))))
    out.append("async: evaluations %d dirty re-runs %d pushes %d spin %.2f ms (summed over warps)" %
               (aq["evaluations"], aq["dirty"], aq["pushes"], aq["spin_us"] / 1000.0))
    out.append("SMALL generations (nE <= %d) per log2 bucket of nE [2^(b-1), 2^b): generations, rounds per generation, us per generation" % small_max)
    for b in sorted(small):
        g, r, t = small[b]
        out.append("  b %2d: %6d gens %6.2f rounds %8.1f us" % (b, g, r / g, t / g))
    g, r, t = (sum(v[k] for v in small.values()) for k in range(3))
    out.append("  all : %6d gens %6.2f rounds %8.1f us (%.2f ms)" % (g, r / max(1, g), t / max(1, g), t / 1000.0))
    for k in ("generations", "rounds", "evaluated", "refreshed", "reseed_rounds", "dependants", "final_after_classify",
              "closure_rounds", "closure_entries", "resolve_passes", "expansions"):
        out.append("total %s %d" % (k, tot[k]))
    for fr in sorted(reseed):
        out.append("frame %d reseed: dependants %d final after classify %d closure rounds %d list entries %d resolve passes %d" % ((fr,) + reseed[fr]))
    for fr in sorted(gens):
        out.append("frame %d nE %s" % (fr, " ".join(str(n) for n, _ in gens[fr])))
    for fr in sorted(gens):
        out.append("frame %d rounds %s" % (fr, " ".join(str(r) for _, r in gens[fr])))
    text = "\n".join(out) + "\n"
    sys.stdout.write(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text)


if __name__ == "__main__":
    main()
