"""Viewpoint coverage throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames), extracts
frontiers at clearance --clearance and minimum cluster size --min-size, and times fiesta_frontiers_score_viewpoints (device time
from the library's CUDA events, the median of --repeats runs after one warm-up) for
  * full   the whole 512^3 grid;
  * local  a 160^3 box (8 m) around the last sensor pose.
Candidates: 32 per kept cluster (radii 1.0, 1.5, 2.0 and 2.5 m x 8 angles, at the centroid's height); 8 yaw orientations; a
90 x 60 degree sensor of 4.5 m range.  For each case it prints candidates and the number scored, pairs walked and visible, and pairs
walked per second, with the GPU's name and power limit.  The 160^3 result (status, score, stats) is compared bit for bit with the
CPU definition (tests/viewref.py, line of sight from the host mirror's sequential walk); the script exits non-zero if it differs.

  python scripts/viewpoint_bench.py [--frames 10] [--clearance 0.3] [--min-size 5] [--repeats 7]
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
from tests import scenes, viewref  # noqa: E402

RADII = (1.0, 1.5, 2.0, 2.5)
MAX_RANGE, TAN = 4.5, (1.0, float(np.tan(np.pi / 6)))


def run_case(fr, name, box, r, min_size, repeats, R):
    fr.compute(box[0], box[1], r, min_size)
    cl, pos = viewref.rings(fr.clusters()["centroid"], RADII, 8)
    fr.score_viewpoints(cl, pos, R, MAX_RANGE, TAN, r)                      # warm-up (and the buffers grow here)
    runs = [fr.score_viewpoints(cl, pos, R, MAX_RANGE, TAN, r) for _ in range(repeats)]
    st = runs[-1][2]
    ms = float(np.median([x[2]["ms_compute"] for x in runs]))
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], kept_clusters=fr.stats["kept_clusters"],
               kept_voxels=fr.stats["kept_voxels"], candidates=len(cl), candidates_scored=st["candidates_scored"],
               pairs_walked=st["pairs_walked"], pairs_visible=st["pairs_visible"], ms=round(ms, 3),
               ms_all=[round(x[2]["ms_compute"], 3) for x in runs], pairs_walked_per_s=st["pairs_walked"] / (ms * 1e-3))
    print(json.dumps(row), flush=True)
    return row, (cl, pos), runs[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--min-size", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("viewpoint_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs, r = m.grid_size, args.clearance
    res, origin = w["res"], np.asarray(w["origin"])
    R = viewref.yaws(8)
    fr = m.Frontiers()
    rows = [run_case(fr, "full", ((0, 0, 0), tuple(g - 1 for g in gs)), r, args.min_size, args.repeats, R)[0]]
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(np.floor((np.asarray(p) - origin) / res).astype(int) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    row, (cl, pos), got = run_case(fr, "local", box, r, args.min_size, args.repeats, R)
    rows.append(row)

    # the 160^3 result against the CPU definition
    t0 = time.perf_counter()
    mirror = m.HostMirror()
    mirror.refresh()
    D = m.export_distance().reshape(gs)
    hi = origin + np.asarray(w["size"], np.float64)                        # PosInMap: [origin, origin + size]
    want = viewref.score(cl, pos, R, MAX_RANGE, TAN, r, fr.clusters()["size"], fr.voxels(), D, origin, res, origin, hi,
                         lambda ab: mirror.CheckSegments(ab, 0.0, False)[0])
    oracle_s = time.perf_counter() - t0
    mirror.close()
    same = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and all(got[2][k] == v for k, v in want[2].items()))
    fr.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r,
                          min_cluster_size=args.min_size, orientations=len(R), max_range_m=MAX_RANGE, tan_half_fov=TAN, cases=rows,
                          local_equals_viewref=same, oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("viewpoint_bench: the 160^3 result differs from the CPU definition")


if __name__ == "__main__":
    main()
