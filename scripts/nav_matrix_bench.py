"""Cost-matrix throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames) and times
fiesta_nav_matrix at clearance --clearance with K points used as both sources and targets:
  * random K   K random traversable voxels of the 160^3 box (8 m) around the last sensor pose, K = 16, 64, 256;
  * near K     K traversable voxels within --near metres of the sensor, in the same box (targets close to every source);
  * full 8     8 random traversable voxels of the whole 512^3 grid (more than one pass).
The matrix's device time is the library's CUDA-event time, the median of --repeats runs after one warm-up.  Each run alternates
with the baseline, K fiesta_nav_compute calls with one goal each over the same box (the sum of their device times).  It prints
both, generations, tile visits, passes and sources retired early, with the GPU's name and power limit.  The random K = 64 matrix
is compared bit for bit with the CPU definition (tests/navmatrixref.py: scipy's Dijkstra on export_distance()).

  python scripts/nav_matrix_bench.py [--frames 10] [--clearance 0.3] [--repeats 7] [--near 2.0]
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
from tests import navmatrixref, navref, scenes  # noqa: E402


def run_case(nav, name, box, pts, r, repeats):
    nav.matrix(box[0], box[1], pts, pts, r)                                # warm-up (the buffers grow here)
    nav.compute(box[0], box[1], pts[:1], r)
    mat, base = [], []
    for _ in range(repeats):                                               # matrix and baseline alternate
        cost, ss, _, st = nav.matrix(box[0], box[1], pts, pts, r)
        mat.append(st)
        base.append(sum(nav.compute(box[0], box[1], p[None], r)["ms_compute"] for p in pts))
    ms = float(np.median([x["ms_compute"] for x in mat]))
    ms_base = float(np.median(base))
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], K=len(pts),
               sources_placed=st["sources_placed"], ms=round(ms, 3), ms_all=[round(x["ms_compute"], 3) for x in mat],
               baseline_ms=round(ms_base, 3), baseline_ms_all=[round(x, 3) for x in base], speedup=round(ms_base / ms, 2),
               passes=st["passes"], generations=st["generations"], tile_visits=st["tile_visits"],
               sources_retired_early=st["sources_retired_early"], finite_entries=int(np.sum(np.isfinite(cost))),
               max_finite_cost=float(np.max(cost[np.isfinite(cost)])) if np.any(np.isfinite(cost)) else 0.0)
    print(json.dumps(row), flush=True)
    return row, cost


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--near", type=float, default=2.0, help="radius (m) of the near-the-robot cases")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("nav_matrix_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs, r = m.grid_size, args.clearance
    D = m.export_distance()
    T = navref.traversable(D.reshape(gs), r, False)
    nav = m.NavField()
    rng = np.random.default_rng(1)
    res, origin = w["res"], np.asarray(w["origin"])
    centre = lambda v: origin + (np.asarray(v) + 0.5) * res
    vox = lambda p: np.floor((np.asarray(p) - origin) / res).astype(int)

    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(vox(p) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    free = np.argwhere(T[navref.box_slices(box)]) + lo
    near = free[np.sum((free - vox(p)) ** 2, axis=1) <= (args.near / res) ** 2]
    rows, check = [], None
    for K in (16, 64, 256):
        pts = centre(free[rng.choice(len(free), K, replace=False)])
        row, cost = run_case(nav, "random%d" % K, box, pts, r, args.repeats)
        rows.append(row)
        if K == 64:
            check = (pts, cost)
    for K in (16, 64, 256):
        rows.append(run_case(nav, "near%d" % K, box, centre(near[rng.choice(len(near), K, replace=False)]), r, args.repeats)[0])
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    fr = np.argwhere(T)
    rows.append(run_case(nav, "full8", full, centre(fr[rng.choice(len(fr), 8, replace=False)]), r, args.repeats)[0])
    nav.close()

    # the random K = 64 matrix against the CPU definition
    t0 = time.perf_counter()
    pts, cost = check
    want = navmatrixref.matrix(D, gs, box, pts, pts, r, False, origin, res, origin, origin + np.asarray(w["size"]))[0]
    oracle_s = time.perf_counter() - t0
    same = bool(np.array_equal(cost, want, equal_nan=True))
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r, unknown_blocks=False,
                          near_radius_m=args.near, cases=rows, random64_matrix_equals_dijkstra=same, oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("nav_matrix_bench: the K = 64 matrix differs from the CPU definition")


if __name__ == "__main__":
    main()
