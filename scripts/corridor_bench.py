"""Safe flight corridor throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames), computes a
cost-to-go field over the 160^3 box (8 m) around the last sensor pose at clearance --clearance with one goal at the sensor, and
extracts --paths paths from random traversable voxels of the box (NavField.paths), reversed so that they run from the robot.  Then
it times fiesta_corridors with max_steps (40, 40, 20) (device time of the whole call from the library's CUDA events, the median of
--repeats runs after one warm-up) in three cases:
  * one     the longest of the paths alone, limit box = the 160^3 box;
  * paths   all the paths, limit box = the 160^3 box;
  * full    all the paths, limit box = the whole 512^3 grid.
The mask time of each limit box is the time of fiesta_inflate_boxes on one seed with max_steps 0, which tests no layer.  For each
case it prints boxes, layers tested and grown, the mask time and the total time, with the GPU's name and power limit.  The 160^3
result of all the paths is compared bit for bit with the CPU definition (tests/corridorref.py on export_distance()); the script
exits non-zero if it differs.

  python scripts/corridor_bench.py [--frames 10] [--clearance 0.3] [--paths 4096] [--repeats 7]
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
from nav_bench import centre, nearest_traversable  # noqa: E402
from tests import corridorref, navref, scenes  # noqa: E402

MAX_STEPS = (40, 40, 20)


def mask_ms(m, box, r, repeats):
    seed = [box[0]]
    m.InflateBoxes(seed, seed, box[0], box[1], (0, 0, 0), r)
    return float(np.median([m.InflateBoxes(seed, seed, box[0], box[1], (0, 0, 0), r)[3]["ms_compute"] for _ in range(repeats)]))


def run_case(m, name, box, paths, r, repeats):
    m.Corridors(paths, box[0], box[1], MAX_STEPS, r)                      # warm-up (and the buffers grow here)
    runs = [m.Corridors(paths, box[0], box[1], MAX_STEPS, r) for _ in range(repeats)]
    st = runs[-1][4]
    ms = float(np.median([x[4]["ms_compute"] for x in runs]))
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], paths=len(paths),
               path_voxels=int(sum(len(p) for p in paths)), status=np.bincount(runs[-1][0], minlength=3).tolist(), boxes=st["boxes"],
               layers_tested=st["layers_tested"], layers_grown=st["layers_grown"], mask_voxels=st["mask_voxels"],
               mask_ms=round(mask_ms(m, box, r, repeats), 3), ms=round(ms, 3), ms_all=[round(x[4]["ms_compute"], 3) for x in runs])
    print(json.dumps(row), flush=True)
    return row, runs[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--paths", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("corridor_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs, r = m.grid_size, args.clearance
    res, origin = w["res"], np.asarray(w["origin"])
    D = m.export_distance()
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    vox = np.floor((np.asarray(p) - origin) / res).astype(int)
    lo = np.clip(vox - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    Tb = navref.traversable(D.reshape(gs)[navref.box_slices(box)], r, False)
    goal = centre(w, lo + nearest_traversable(Tb, vox - lo))[None]
    nav = m.NavField()
    nav.compute(box[0], box[1], goal, r)
    free = np.argwhere(Tb)
    rng = np.random.default_rng(1)
    starts = centre(w, lo + free[rng.choice(len(free), args.paths, replace=False)])
    status, ln, _, pv = nav.paths(starts, 2048)
    nav.close()
    paths = [pv[i, :ln[i]][::-1].copy() for i in range(len(ln))]            # robot -> start
    longest = [paths[int(np.argmax(ln))]]
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    rows = [run_case(m, "one", box, longest, r, args.repeats)[0]]
    row, got = run_case(m, "paths", box, paths, r, args.repeats)
    rows.append(row)
    rows.append(run_case(m, "full", full, paths, r, args.repeats)[0])

    # the 160^3 result of all the paths against the CPU definition
    t0 = time.perf_counter()
    want = corridorref.corridors(corridorref.Limit(D, gs, box, r, False), paths, MAX_STEPS)
    oracle_s = time.perf_counter() - t0
    same = all(np.array_equal(got[k], want[k]) for k in range(3)) and \
        all(np.array_equal(x, y) for a, b in zip(got[3], want[3]) for x, y in zip(a, b)) and all(got[4][k] == v for k, v in want[4].items())
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r, unknown_blocks=False,
                          max_steps=MAX_STEPS, nav_path_status=np.bincount(status, minlength=4).tolist(),
                          mean_path_len=round(float(ln.mean()), 1), cases=rows, paths_equal_corridorref=bool(same),
                          oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("corridor_bench: the 160^3 result differs from the CPU definition")


if __name__ == "__main__":
    main()
