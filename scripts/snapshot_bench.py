"""Map snapshots on the flagship map: size, save and load time, and the continuation check (H100 only; no CPU fallback).

Builds bench.py's 512^3 LIDAR map (lidar512) from its first --frames frames in each mode, then reports the stored tiles against
the grid's tiles and the stream bytes, and the median over --reps repetitions of:
  save   wall time of fiesta_snapshot_save into a preallocated host buffer (classification, pack, copy out; synchronous)
  load   wall time of fiesta_snapshot_load from that buffer (header checks, map creation, copy in, unpack, validation)
  floor  a plain pinned cudaMemcpy of the same byte count, device to host and host to device, timed with CUDA events in the
         same run
with the effective GB/s of each.  Then it integrates --steps more frames on the saved and the loaded map and exits non-zero on
any difference in the exports.  Prints one JSON row per mode with the GPU's name and power limit.

  python scripts/snapshot_bench.py [--frames 10] [--steps 3] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
import segment_bench  # noqa: E402


def memcpy_floor(nbytes, reps):
    import torch
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = {}
    for name, dst, src in (("d2h", h, d), ("h2d", d, h)):
        ts = []
        for _ in range(reps + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dst.copy_(src, non_blocking=True)
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = statistics.median(ts[1:])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the snapshot")
    ap.add_argument("--steps", type=int, default=3, help="frames integrated afterwards on both maps, compared bit for bit")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("snapshot_bench: no CUDA device (there is no CPU fallback)")
    import fiesta_b200
    info = segment_bench.gpu_info()
    w = bench.WORKLOADS["lidar512"]
    frames = bench.make_frames("lidar512", args.frames + args.steps)
    L = fiesta_b200.load_library()
    failed = False
    for mode in ("exact", "fast"):
        m = fiesta_b200.ESDFMap(w["origin"], w["res"], w["size"], mode=mode)
        m.SetParameters(*bench.wl_params("lidar512"))

        def integrate(mm, fr):
            mm.RaycastFrame(fr["pts"], fr["T"], w["min_len"], w["max_len"])
            if mm.CheckUpdate():
                mm.SetOriginalRange(); mm.UpdateOccupancy(True); mm.UpdateESDF()
            mm.synchronize()

        for fr in frames[:args.frames]:
            integrate(m, fr)
        size = C.c_int64(0)
        assert L.fiesta_snapshot_save(m._h, None, 0, C.byref(size)) == 0
        n = size.value
        buf = np.zeros(n, np.uint8)                                   # touched once: page faults are not part of the timing
        t_save, t_load = [], []
        for _ in range(args.reps + 1):
            t0 = time.perf_counter()
            assert L.fiesta_snapshot_save(m._h, buf.ctypes.data, C.c_int64(n), C.byref(size)) == 0
            t_save.append(time.perf_counter() - t0)
        for _ in range(args.reps + 1):
            t0 = time.perf_counter()
            h = C.c_void_p()
            rc = L.fiesta_snapshot_load(buf.ctypes.data, C.c_int64(n), C.c_int32(m.device), C.byref(h))
            t_load.append(time.perf_counter() - t0)
            assert rc == 0, L.fiesta_last_error().decode()
            L.fiesta_destroy(h)
        b = fiesta_b200.ESDFMap.load(buf, device=m.device)
        stored = int.from_bytes(buf[312:320].tobytes(), "little")
        gs = m.grid_size
        tiles = ((gs[0] + 7) // 8) * ((gs[1] + 7) // 8) * ((gs[2] + 7) // 8)
        floor = memcpy_floor(n, args.reps)
        ms_save, ms_load = 1e3 * statistics.median(t_save[1:]), 1e3 * statistics.median(t_load[1:])
        diffs = 0
        for fr in frames[args.frames:]:
            for mm in (m, b):
                integrate(mm, fr)
            for f in ("export_distance", "export_occupancy", "export_closest_obstacle"):
                diffs += int(getattr(m, f)().tobytes() != getattr(b, f)().tobytes())
            diffs += int(any(x.tobytes() != y.tobytes() for x, y in zip(m.export_counters(), b.export_counters())))
        failed = failed or diffs > 0
        print(json.dumps(dict(mode=mode, frames=args.frames, grid=list(gs), stored_tiles=stored, tiles=tiles, bytes=n,
                              save_ms=round(ms_save, 2), load_ms=round(ms_load, 2), save_GBps=round(n / ms_save / 1e6, 2),
                              load_GBps=round(n / ms_load / 1e6, 2), memcpy_d2h_ms=round(floor["d2h"], 2), memcpy_h2d_ms=round(floor["h2d"], 2),
                              memcpy_d2h_GBps=round(n / floor["d2h"] / 1e6, 2), memcpy_h2d_GBps=round(n / floor["h2d"] / 1e6, 2),
                              steps=args.steps, continuation_diffs=diffs, **info)), flush=True)
        b.close()
        m.close()
    if failed:
        sys.exit("snapshot_bench: the loaded map diverged from the saved one")


if __name__ == "__main__":
    main()
