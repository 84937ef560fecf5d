"""Surface mesh time on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames) and times
fiesta_mesh_compute (device time from the library's CUDA events, the median of --repeats runs after one warm-up, split into
classify (bitmap, counts and scans), vertices and faces) for
  * full   the whole 512^3 grid;
  * local  a 160^3 box (8 m) around the last sensor pose;
each at clearance 0.5 * resolution (the obstacle cubes' faces) and --clearance.  For each it prints ms per stage, the mesh's size and
the bytes floor: records read (4 bytes per box voxel) plus outputs written (12 bytes per vertex and per triangle) over 3.35 TB/s, with
the GPU's name and power limit.  The 160^3 results (vertices, triangles, stats) are compared bit for bit with the CPU definition
(tests/meshref.py on export_distance() and export_closest_obstacle()).

  python scripts/mesh_bench.py [--frames 10] [--clearance 0.3] [--repeats 7]
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
from tests import meshref, scenes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet


def run_case(me, name, box, r, args):
    me.compute(box[0], box[1], r)                                           # warm-up (and the buffers grow here)
    runs = [me.compute(box[0], box[1], r) for _ in range(args.repeats)]
    st = runs[-1]
    med = {k: round(float(np.median([x[k] for x in runs])), 3) for k in ("ms_compute", "ms_classify", "ms_vertices", "ms_faces")}
    floor_bytes = 4 * st["box_voxels"] + 12 * st["vertices"] + 12 * st["triangles"]
    row = dict(case=name, clearance_m=r, box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]],
               **{k: st[k] for k in ("box_voxels", "blocking", "vertices", "quads", "triangles")},
               ms=med["ms_compute"], ms_classify=med["ms_classify"], ms_vertices=med["ms_vertices"], ms_faces=med["ms_faces"],
               floor_ms=round(floor_bytes / HBM_BYTES_PER_S * 1e3, 3), ms_all=[round(x["ms_compute"], 3) for x in runs])
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the compute")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs = m.grid_size
    res, origin = w["res"], np.asarray(w["origin"])
    me = m.Mesh()
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(np.floor((np.asarray(p) - origin) / res).astype(int) - 80, 0, np.asarray(gs) - 160)
    local = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    rows, same, oracle_s = [], True, 0.0
    D, O = m.export_distance(), m.export_closest_obstacle()
    for r in (0.5 * res, args.clearance):
        rows.append(run_case(me, "full", full, r, args))
        rows.append(run_case(me, "local", local, r, args))
        # the last result (160^3) against the CPU definition
        t0 = time.perf_counter()
        want = meshref.mesh(D, O, gs, local, r, False, res, origin)
        oracle_s += time.perf_counter() - t0
        v = me.vertices()
        same &= bool(np.array_equal(v.view(np.uint32), want["vertices"].view(np.uint32)) and
                     np.array_equal(me.triangles(), want["triangles"]) and all(rows[-1][k] == x for k, x in want["stats"].items()))
    me.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, cases=rows, local_equals_meshref=same,
                          oracle_seconds=round(oracle_s, 1))))
    if not same:
        sys.exit("mesh_bench: a 160^3 result differs from the CPU definition")


if __name__ == "__main__":
    main()
