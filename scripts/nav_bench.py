"""Cost-to-go field throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames) and times
fiesta_nav_compute at clearance --clearance (device time from the library's CUDA events, the median of --repeats runs after one
warm-up) in three cases:
  * full     the whole 512^3 grid, one goal in the room's far corner;
  * local    a 160^3 box (8 m) around the last sensor pose, one goal at the sensor;
  * local64  the same box with 64 goals on random traversable voxels.
For each it prints ms, reached voxels per second, generations and tile visits, and the time of fiesta_nav_paths for 2^16 random
starts in the box (the synchronous host entry point, its copies included), with the GPU's name and power limit.  The 160^3 field
is compared bit for bit with the CPU definition (tests/navref.py: scipy's Dijkstra on export_distance()).

  python scripts/nav_bench.py [--frames 10] [--clearance 0.3] [--repeats 5] [--max-len 1024]
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
from tests import navref, scenes  # noqa: E402


def nearest_traversable(T, v, reach=32):
    """The traversable voxel of T nearest to voxel v, searched within `reach` voxels of it."""
    lo = np.maximum(np.asarray(v) - reach, 0)
    c = np.argwhere(T[tuple(slice(a, a + 2 * reach + 1) for a in lo)]) + lo
    return c[np.argmin(np.sum((c - np.asarray(v)) ** 2, axis=1))]


def centre(w, v):
    return np.asarray(w["origin"]) + (np.asarray(v) + 0.5) * w["res"]


def run_case(nav, name, box, goals, r, repeats, starts, max_len):
    nav.compute(box[0], box[1], goals, r)                                  # warm-up (and the buffers grow here)
    runs = [nav.compute(box[0], box[1], goals, r) for _ in range(repeats)]
    st = runs[-1]
    ms = float(np.median([x["ms_compute"] for x in runs]))
    nav.paths(starts[:1024], max_len)
    t0 = time.perf_counter()
    status, ln, _, _ = nav.paths(starts, max_len)
    path_ms = (time.perf_counter() - t0) * 1e3
    row = dict(case=name, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], goals=len(goals),
               goals_placed=st["goals_placed"], box_voxels=st["box_voxels"], blocked=st["blocked"], reached=st["reached"],
               ms=round(ms, 3), ms_all=[round(x["ms_compute"], 3) for x in runs], reached_voxels_per_s=st["reached"] / (ms * 1e-3),
               generations=st["generations"], tile_visits=st["tile_visits"], paths=len(starts), path_max_len=max_len,
               paths_ms=round(path_ms, 2), path_status=np.bincount(status, minlength=4).tolist(),
               mean_path_len=round(float(ln[status == 0].mean()), 1) if np.any(status == 0) else 0.0)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--max-len", type=int, default=1024)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("nav_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs, r = m.grid_size, args.clearance
    D = m.export_distance()
    Dg = D.reshape(gs)
    T = navref.traversable(Dg, r, False)
    nav = m.NavField()
    rng = np.random.default_rng(1)
    res, origin = w["res"], np.asarray(w["origin"])
    vox = lambda p: np.floor((np.asarray(p) - origin) / res).astype(int)
    rows = []

    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    corner = vox(np.asarray(w["room"]) * np.array([0.95, 0.95, -0.9]))
    g_full = centre(w, nearest_traversable(T, corner))[None]
    starts = rng.uniform(-np.asarray(w["room"]), np.asarray(w["room"]), (1 << 16, 3))
    rows.append(run_case(nav, "full", full, g_full, r, args.repeats, starts, args.max_len))

    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(vox(p) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    Tb = T[navref.box_slices(box)]
    g_one = centre(w, lo + nearest_traversable(Tb, vox(p) - lo))[None]
    free = np.argwhere(Tb)
    g_64 = centre(w, lo + free[rng.choice(len(free), 64, replace=False)])
    blo, bhi = origin + lo * res, origin + (lo + 160) * res
    starts = rng.uniform(blo, bhi, (1 << 16, 3))
    rows.append(run_case(nav, "local", box, g_one, r, args.repeats, starts, args.max_len))
    rows.append(run_case(nav, "local64", box, g_64, r, args.repeats, starts, args.max_len))

    # the last field (160^3, 64 goals) against the CPU definition
    t0 = time.perf_counter()
    want = navref.field(D, gs, box, np.floor((g_64 - origin) / res).astype(np.int64), r, False, res)
    oracle_s = time.perf_counter() - t0
    same = bool(np.array_equal(nav.export(), want))
    nav.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r, unknown_blocks=False,
                          cases=rows, local64_field_equals_dijkstra=same, oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("nav_bench: the 160^3 field differs from the CPU definition")


if __name__ == "__main__":
    main()
