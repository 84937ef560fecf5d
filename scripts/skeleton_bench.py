"""Topological skeleton time on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames) and times
fiesta_skeleton_compute at clearance --clearance, max_cos --max-cos and min_branch --min-branch (device time from the library's
CUDA events, the median of --repeats runs after one warm-up, split into init, thinning and graph) for
  * full   the whole 512^3 grid;
  * local  a 160^3 box (8 m) around the last sensor pose.
For each it prints ms per stage, the thinning iterations, the pruning rounds and the graph's size, with the GPU's name and power
limit.  The 160^3 result (mask, labels, vertices, edges, edge voxels, stats) is compared bit for bit with the CPU definition
(tests/skeletonref.py on export_distance() and export_closest_obstacle()).

  python scripts/skeleton_bench.py [--frames 10] [--clearance 0.3] [--max-cos 0.5] [--min-branch 8] [--repeats 7]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import segment_bench  # noqa: E402
from tests import scenes, skeletonref  # noqa: E402


def run_case(sk, name, box, args):
    kw = dict(clearance=args.clearance, max_cos=args.max_cos, min_branch=args.min_branch)
    sk.compute(box[0], box[1], **kw)                                       # warm-up (and the buffers grow here)
    runs = [sk.compute(box[0], box[1], **kw) for _ in range(args.repeats)]
    st = runs[-1]
    med = {k: round(float(np.median([x[k] for x in runs])), 3) for k in ("ms_compute", "ms_init", "ms_thin", "ms_graph")}
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]],
               **{k: st[k] for k in ("box_voxels", "traversable", "anchors", "iterations", "prune_rounds", "pruned_voxels",
                                     "skeleton_voxels", "vertices", "edges", "edge_voxels")},
               ms=med["ms_compute"], ms_init=med["ms_init"], ms_thin=med["ms_thin"], ms_graph=med["ms_graph"],
               ms_all=[round(x["ms_compute"], 3) for x in runs])
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the compute")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--max-cos", type=float, default=0.5)
    ap.add_argument("--min-branch", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("skeleton_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs = m.grid_size
    res, origin = w["res"], np.asarray(w["origin"])
    sk = m.Skeleton()
    rows = [run_case(sk, "full", ((0, 0, 0), tuple(g - 1 for g in gs)), args)]
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(np.floor((np.asarray(p) - origin) / res).astype(int) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    rows.append(run_case(sk, "local", box, args))

    # the last result (160^3) against the CPU definition
    t0 = time.perf_counter()
    want = skeletonref.skeleton(m.export_distance(), m.export_closest_obstacle(), gs, box, args.clearance, False, args.max_cos,
                                args.min_branch, res, origin)
    oracle_s = time.perf_counter() - t0
    mask, lab = sk.export()
    v, e = sk.vertices(), sk.edges()
    same = bool(np.array_equal(mask, want["mask"]) and np.array_equal(lab, want["labels"]) and
                all(np.array_equal(v[k], want["vertices"][k]) for k in v) and all(np.array_equal(e[k], want["edges"][k]) for k in e) and
                np.array_equal(sk.edge_voxels(), want["edge_voxels"]) and all(rows[-1][k] == x for k, x in want["stats"].items()))
    sk.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=args.clearance,
                          max_cos=args.max_cos, min_branch=args.min_branch, cases=rows, local_equals_skeletonref=same,
                          oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("skeleton_bench: the 160^3 result differs from the CPU definition")


if __name__ == "__main__":
    main()
