"""Signed distance throughput on the flagship map (H100 only; no CPU fallback).

Builds the map of scripts/segment_bench.py (bench.py's 512^3 LIDAR workload, 5 cm voxels, after --frames EXACT frames; the compute
reads only the records, so one mode is enough) and measures, with the GPU's name and power limit in the same run:
  * fiesta_signed_compute over the whole 512^3 grid and over a 160^3 box around the last sensor pose: device time from the
    library's CUDA events, the median of --repeats runs after two warm-ups;
  * 2^20 signed trilinear queries against 2^20 plain ones (fiesta_get_dist_grad_trilinear_batch_device) on the same positions, on
    device buffers, timed with CUDA events around --query-repeats back-to-back calls of each, alternated.
The 160^3 export is compared bit for bit with tests/signedref.py (scipy's EDT) on export_distance().
A floor from bytes for the whole grid: the passes move about 40 bytes per voxel (records in, q written and re-read, the scratch
written and re-read, the stacks) -> 5.4 GB at 3.35 TB/s = 1.6 ms.

  python scripts/signed_bench.py [--frames 10] [--repeats 20] [--query-repeats 20]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import segment_bench  # noqa: E402
from tests import scenes, signedref  # noqa: E402

BYTES_PER_VOXEL = 40


def time_compute(sf, box, repeats):
    for _ in range(2):
        sf.compute(box[0], box[1])
    runs = [sf.compute(box[0], box[1]) for _ in range(repeats)]
    st = runs[-1]
    ms = float(np.median([r["ms_compute"] for r in runs]))
    nv = st["box_voxels"]
    return dict(box_lo=[int(x) for x in box[0]], box_hi=[int(x) for x in box[1]], box_voxels=nv, obstacles=st["obstacles"],
                interior=st["interior"], max_depth_sq=st["max_depth_sq"], ms_median=round(ms, 3),
                ms_min=round(min(r["ms_compute"] for r in runs), 3), ms_max=round(max(r["ms_compute"] for r in runs), 3),
                floor_ms=round(nv * BYTES_PER_VOXEL / 3.35e12 * 1e3, 3), voxels_per_s=nv / (ms * 1e-3))


def time_queries(m, sf, pos, repeats):
    import torch
    tp = torch.from_numpy(pos).cuda()
    calls = {"signed": lambda: sf.GetDistWithGradTrilinearBatchDevice(tp), "plain": lambda: m.GetDistWithGradTrilinearBatchDevice(tp)}
    for f in calls.values():
        f()
    torch.cuda.synchronize()
    ms = {k: [] for k in calls}
    for _ in range(3):                                                       # alternate the two, three rounds
        for k, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(repeats):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / repeats)
    sd, sg = calls["signed"]()
    pd, pg = calls["plain"]()
    torch.cuda.synchronize()
    differ = int(torch.sum(sd != pd).item())
    return {k: dict(ms_per_call=round(float(np.median(v)), 4), queries_per_s=len(pos) / (np.median(v) * 1e-3)) for k, v in ms.items()}, differ


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the measurements")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--query-repeats", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("signed_bench: no CUDA device (there is no CPU fallback)")
    info = segment_bench.gpu_info()
    m, w = segment_bench.build_map(args.frames)
    gs = m.grid_size
    res, origin = w["res"], np.asarray(w["origin"])
    sf = m.SignedField()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    row_full = time_compute(sf, full, args.repeats)
    print(json.dumps(dict(case="full", **row_full)), flush=True)

    p, _ = scenes.pose_walk(args.frames, seed=w["pose_seed"], clamp=w["clamp"])[-1]
    lo = np.clip(np.floor((np.asarray(p) - origin) / res).astype(int) - 80, 0, np.asarray(gs) - 160)
    box = (tuple(int(x) for x in lo), tuple(int(x) + 159 for x in lo))
    row_local = time_compute(sf, box, args.repeats)
    print(json.dumps(dict(case="local160", **row_local)), flush=True)
    S, q = signedref.field(m.export_distance(), gs, box, res)
    same = bool(np.array_equal(sf.export().view(np.int64), S.view(np.int64)))

    # queries: 2^20 positions in the 160^3 box, half of them on obstacle voxels' neighbourhoods
    rng = np.random.default_rng(1)
    blo, bhi = origin + lo * res, origin + (lo + 160) * res
    pos = rng.uniform(blo, bhi, (1 << 20, 3))
    obst = np.argwhere(q > 0)
    if len(obst):
        k = len(pos) // 2
        pos[:k] = origin + (lo + obst[rng.integers(0, len(obst), k)] + rng.uniform(0, 1, (k, 3))) * res
    pos = np.ascontiguousarray(pos)
    qrows, differ = time_queries(m, sf, pos, args.query_repeats)
    sf.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, compute=[row_full, row_local],
                          queries=dict(n=len(pos), **qrows, distances_differing=differ), local160_export_equals_scipy=same)))
    if not same:
        sys.exit("signed_bench: the 160^3 field differs from the CPU definition")


if __name__ == "__main__":
    main()
