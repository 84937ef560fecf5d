"""Frontier extraction throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames) and times
fiesta_frontiers_compute at clearance --clearance and minimum cluster size --min-size (device time from the library's CUDA events,
the median of --repeats runs after one warm-up) for
  * full   the whole 512^3 grid;
  * local  a 160^3 box (8 m) around the last sensor pose.
For each it prints ms, frontier voxels, clusters before and after the size filter and kept members, with the GPU's name and power
limit.  The 160^3 result (labels, cluster arrays, member list, stats) is compared bit for bit with the CPU definition
(tests/frontierref.py on export_distance() and export_occupancy()).

  python scripts/frontier_bench.py [--frames 10] [--clearance 0.3] [--min-size 5] [--repeats 7]
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

import bench  # noqa: E402
import segment_bench  # noqa: E402
from tests import frontierref, scenes  # noqa: E402


def run_case(fr, name, box, r, min_size, repeats):
    fr.compute(box[0], box[1], r, min_size)                               # warm-up (and the buffers grow here)
    runs = [fr.compute(box[0], box[1], r, min_size) for _ in range(repeats)]
    st = runs[-1]
    ms = float(np.median([x["ms_compute"] for x in runs]))
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], box_voxels=st["box_voxels"],
               frontier_voxels=st["frontier_voxels"], clusters=st["clusters"], kept_clusters=st["kept_clusters"],
               kept_voxels=st["kept_voxels"], ms=round(ms, 3), ms_all=[round(x["ms_compute"], 3) for x in runs],
               box_voxels_per_s=st["box_voxels"] / (ms * 1e-3))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--min-size", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("frontier_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs, r = m.grid_size, args.clearance
    res, origin = w["res"], np.asarray(w["origin"])
    fr = m.Frontiers()
    rows = [run_case(fr, "full", ((0, 0, 0), tuple(g - 1 for g in gs)), r, args.min_size, args.repeats)]
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(np.floor((np.asarray(p) - origin) / res).astype(int) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    rows.append(run_case(fr, "local", box, r, args.min_size, args.repeats))

    # the last result (160^3) against the CPU definition
    t0 = time.perf_counter()
    l_occ = frontierref.l_occ(bench.wl_params("lidar512")[4])
    want = frontierref.extract(m.export_distance(), m.export_occupancy(), gs, box, r, l_occ, args.min_size, res, origin)
    oracle_s = time.perf_counter() - t0
    got = fr.clusters()
    same = bool(np.array_equal(fr.export(), want["labels"]) and np.array_equal(fr.voxels(), want["voxels"]) and
                all(np.array_equal(got[k], want[k]) for k in got) and
                all(rows[-1][k] == v for k, v in want["stats"].items()))
    fr.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r,
                          min_cluster_size=args.min_size, cases=rows, local_equals_frontierref=same, oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("frontier_bench: the 160^3 result differs from the CPU definition")


if __name__ == "__main__":
    main()
