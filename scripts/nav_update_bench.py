"""Cost-to-go field updates against recomputes on the flagship map (H100 only; no CPU fallback).

Integrates the first --frames frames of bench.py's 512^3 LIDAR workload (EXACT mode, as scripts/segment_bench.py builds it) and
computes the two fields of scripts/nav_bench.py: the whole grid with one goal in the room's far corner, and a 160^3 box around
the sensor with 64 goals.  Then, for each of the next --steps frames, integrates the frame and times fiesta_nav_update on the
live fields against a fresh fiesta_nav_compute on a second field object (device time from the library's CUDA events), and
checks that the two exports are equal bit for bit; any difference exits non-zero.  Prints one JSON row per frame and case, then
the medians with the GPU's name and power limit.

  python scripts/nav_update_bench.py [--frames 10] [--steps 8] [--clearance 0.3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
import segment_bench  # noqa: E402
from nav_bench import centre, nearest_traversable  # noqa: E402
from tests import navref, scenes  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the fields are computed")
    ap.add_argument("--steps", type=int, default=8, help="frames integrated afterwards, each followed by an update")
    ap.add_argument("--clearance", type=float, default=0.3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("nav_update_bench: no CUDA device (there is no CPU fallback)")
    import fiesta_b200
    info = segment_bench.gpu_info()
    w = bench.WORKLOADS["lidar512"]
    frames = bench.make_frames("lidar512", args.frames + args.steps)
    m = fiesta_b200.ESDFMap(w["origin"], w["res"], w["size"], mode="exact")
    m.SetParameters(*bench.wl_params("lidar512"))

    def integrate(fr):
        m.RaycastFrame(fr["pts"], fr["T"], w["min_len"], w["max_len"])
        if m.CheckUpdate():
            m.SetOriginalRange(); m.UpdateOccupancy(True); m.UpdateESDF()
        m.synchronize()

    for fr in frames[:args.frames]:
        integrate(fr)
    gs, r, res, origin = m.grid_size, args.clearance, w["res"], np.asarray(w["origin"])
    T = navref.traversable(m.export_distance().reshape(gs), r, False)
    vox = lambda p: np.floor((np.asarray(p) - origin) / res).astype(int)
    rng = np.random.default_rng(1)
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    g_full = centre(w, nearest_traversable(T, vox(np.asarray(w["room"]) * np.array([0.95, 0.95, -0.9]))))[None]
    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(vox(p) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    free = np.argwhere(T[navref.box_slices(box)])
    g_64 = centre(w, lo + free[rng.choice(len(free), 64, replace=False)])
    cases = [("full", full, g_full), ("local64", box, g_64)]
    live = {}
    for name, b, g in cases:
        live[name] = (m.NavField(), m.NavField())
        live[name][0].compute(b[0], b[1], g, r)
        live[name][1].compute(b[0], b[1], g, r)                              # warm-up of the recompute object
    rows, ok = [], True
    for step, fr in enumerate(frames[args.frames:]):
        integrate(fr)
        for name, b, g in cases:
            nav, ref = live[name]
            st = nav.update()
            rs = ref.compute(b[0], b[1], g, r)
            same = bool(np.array_equal(nav.export(), ref.export()))
            ok &= same
            row = dict(frame=args.frames + step, case=name, update_ms=round(st["ms_compute"], 3), compute_ms=round(rs["ms_compute"], 3),
                       speedup=round(rs["ms_compute"] / max(st["ms_compute"], 1e-6), 2), equal=same,
                       **{k: v for k, v in st.items() if k != "ms_compute"}, compute_generations=rs["generations"],
                       compute_tile_visits=rs["tile_visits"])
            rows.append(row)
            print(json.dumps(row), flush=True)
    med = {}
    for name, _, _ in cases:
        rr = [x for x in rows if x["case"] == name]
        med[name] = dict(update_ms=float(np.median([x["update_ms"] for x in rr])), compute_ms=float(np.median([x["compute_ms"] for x in rr])),
                         withdrawn=float(np.median([x["withdrawn"] for x in rr])), tile_visits=float(np.median([x["tile_visits"] for x in rr])))
    for a, b in live.values():
        a.close(); b.close()
    print(json.dumps(dict(gpu=info, map="lidar512, fields computed after %d EXACT frames, %d updates" % (args.frames, args.steps),
                          clearance_m=r, unknown_blocks=False, medians=med, all_equal=ok)))
    if not ok:
        sys.exit("nav_update_bench: an updated field differs from the recomputed one")


if __name__ == "__main__":
    main()
