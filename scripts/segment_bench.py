"""Segment clearance throughput on the flagship map (H100 only; no CPU fallback).

Builds bench.py's default workload map (512^3 LIDAR, 5 cm voxels, same scene generator, seeds and frames), then times:
  * fiesta_check_segments_device (CUDA events on the current torch stream) on 2^16 and 2^20 segments for two workloads,
      "edges"          lengths U[0.05, 1] m (sampling-planner edges),
      "line_of_sight"  lengths U[1, 20] m (shortcuts, visibility);
  * fiesta_check_segments (host buffers, synchronous) on the same batches;
  * single-segment latency: the host mirror against a device call followed by a synchronise.
Segments start uniformly inside the room and are clipped to the map, so they never leave it.  It prints segments/s and voxels
walked per second (walked voxels counted with the exact definition of tests/segref.py on a subsample, scaled to the batch),
with the GPU's name and power limit.  Outputs of the device and host entry points are compared on every batch.

  python scripts/segment_bench.py [--frames 10] [--clearance 0.3] [--unknown-blocks] [--repeats 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tests import segref  # noqa: E402

WORKLOADS = {"edges": (0.05, 1.0), "line_of_sight": (1.0, 20.0)}


def gpu_info():
    import torch
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def build_map(frames):
    import fiesta_b200
    w = bench.WORKLOADS["lidar512"]
    m = fiesta_b200.ESDFMap(w["origin"], w["res"], w["size"], mode="exact")
    m.SetParameters(*bench.wl_params("lidar512"))
    for fr in bench.make_frames("lidar512", frames):
        m.RaycastFrame(fr["pts"], fr["T"], w["min_len"], w["max_len"])
        if m.CheckUpdate():
            m.SetOriginalRange(); m.UpdateOccupancy(True); m.UpdateESDF()
    m.synchronize()
    return m, w


def make_segments(w, n, lengths, seed):
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(w["origin"]), np.asarray(w["origin"]) + np.asarray(w["size"])
    room = np.asarray(w["room"])
    a = rng.uniform(-room, room, (n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    b = np.clip(a + d * rng.uniform(*lengths, n)[:, None], lo, hi)
    return np.ascontiguousarray(np.concatenate([a, b], 1))


def walked_voxels(ab, w, D, r, unknown_blocks, k=200):
    """Mean voxels the query walks per segment (up to and including the first blocking one), exact definition, k samples."""
    lo, hi = np.asarray(w["origin"]), np.asarray(w["origin"]) + np.asarray(w["size"])
    total = 0
    for s in ab[:k]:
        walk = segref.segment_walk(s, w["origin"], w["res"], lo, hi)
        st, ix, _, _ = segref.apply(walk, D, r, unknown_blocks)
        n = len(walk)
        if st == 1:
            gx, gy, gz = D.shape
            n = next(i for i, (v, _) in enumerate(walk) if (v[0] * gy + v[1]) * gz + v[2] == ix) + 1
        total += n
    return total / min(k, len(ab))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.3)
    ap.add_argument("--unknown-blocks", action="store_true")
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("segment_bench: no CUDA device (there is no CPU fallback)")
    info = gpu_info()
    m, w = build_map(args.frames)
    D = m.export_distance().reshape(m.grid_size)
    r, unk = args.clearance, args.unknown_blocks
    rows = []
    for name, lengths in WORKLOADS.items():
        for logn in (16, 20):
            n = 1 << logn
            ab = make_segments(w, n, lengths, seed=logn)
            ab_t = torch.from_numpy(ab).cuda()
            for _ in range(3):
                out = m.CheckSegments(ab_t, r, unknown_blocks=unk)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.repeats):
                out = m.CheckSegments(ab_t, r, unknown_blocks=unk)
            e1.record()
            e1.synchronize()
            dev_s = e0.elapsed_time(e1) * 1e-3 / args.repeats
            host = m.CheckSegments(ab, r, unknown_blocks=unk)
            t0 = time.perf_counter()
            reps = max(3, args.repeats // 4)
            for _ in range(reps):
                host = m.CheckSegments(ab, r, unknown_blocks=unk)
            host_s = (time.perf_counter() - t0) / reps
            same = all(np.array_equal(a.cpu().numpy(), b, equal_nan=True) for a, b in zip(out, host))
            vox = walked_voxels(ab, w, D, r, unk)
            st = np.bincount(host[0], minlength=3)
            rows.append(dict(workload=name, n=n, device_ms=round(dev_s * 1e3, 4), device_segments_per_s=n / dev_s,
                             device_voxels_per_s=n * vox / dev_s, host_entry_ms=round(host_s * 1e3, 3), host_entry_segments_per_s=n / host_s,
                             mean_voxels_walked=round(vox, 2), clear=int(st[0]), blocked=int(st[1]), outside=int(st[2]),
                             device_equals_host_entry=bool(same)))
            print(json.dumps(rows[-1]), flush=True)
    # single-segment latency: pinned host mirror (pure host code) against one device call + synchronise
    mir = m.HostMirror()
    one = make_segments(w, 1, WORKLOADS["edges"], seed=1)
    one_t = torch.from_numpy(one).cuda()
    for _ in range(100):
        mir.CheckSegments(one, r, unk); m.CheckSegments(one_t, r, unknown_blocks=unk)
    torch.cuda.synchronize()
    k = 2000
    t0 = time.perf_counter()
    for _ in range(k):
        mir.CheckSegments(one, r, unk)
    mirror_us = (time.perf_counter() - t0) / k * 1e6
    t0 = time.perf_counter()
    for _ in range(k):
        m.CheckSegments(one_t, r, unknown_blocks=unk)
        torch.cuda.synchronize()
    device_us = (time.perf_counter() - t0) / k * 1e6
    mir.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r, unknown_blocks=unk,
                          batches=rows, single_segment_us=dict(host_mirror=round(mirror_us, 2), device_call_and_sync=round(device_us, 2),
                                                                note="both through the Python binding (ctypes), so each includes its call overhead"))))


if __name__ == "__main__":
    main()
