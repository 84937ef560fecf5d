"""Robot-shaped collision check throughput on the flagship map (H100 only; no CPU fallback).

Builds bench.py's default workload map (512^3 LIDAR, 5 cm voxels, same scene generator, seeds and frames), then times:
  * fiesta_check_poses_device (CUDA events on the current torch stream) on 2^16 and 2^20 poses for two bodies,
      "drone"  half extents (0.25, 0.25, 0.1) m, uniformly random full rotations,
      "car"    half extents (2.25, 0.9, 0.75) m, random yaw only;
  * fiesta_check_poses (host buffers, synchronous) on the same batches;
  * single-pose latency: the host mirror against a device call followed by a synchronise.
Pose centres are uniform inside the room.  It prints poses/s and candidate voxels/s (the candidate range of every pose of a
subsample, counted exactly with tests/poseref.py and scaled to the batch), with the GPU's name and power limit.  The device and host
outputs are compared on every batch, and the host mirror's (pure host code) on the first --mirror-sample poses of every batch.

  python scripts/pose_bench.py [--frames 10] [--clearance 0.0] [--unknown-blocks] [--seconds 2] [--mirror-sample 2048]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.segment_bench import build_map, gpu_info  # noqa: E402
from tests import poseref  # noqa: E402

BODIES = {"drone": ((0.25, 0.25, 0.1), False), "car": ((2.25, 0.9, 0.75), True)}


def make_poses(w, n, yaw_only, seed):
    rng = np.random.default_rng(seed)
    room = np.asarray(w["room"])
    p = rng.uniform(-room, room, (n, 3))
    R = poseref.yaw_rotations(rng, n) if yaw_only else poseref.random_rotations(rng, n)
    return poseref.poses(p, R)


def candidates(P, h, w, k=4096):
    """Mean candidate voxels per pose (exact candidate ranges of k poses)."""
    tot = 0
    for pose in P[:k]:
        lo, hi = poseref.candidate_range(pose, h, w["origin"], w["res"])
        tot += int(np.prod(hi - lo + 1))
    return tot / min(k, len(P))


def timed(fn, seconds):
    """Warm up with one call, time a second, and return how many calls fill about `seconds` (3 to 50)."""
    fn()
    t0 = time.perf_counter()
    fn()
    one = time.perf_counter() - t0
    reps = int(max(3, min(50, seconds / max(one, 1e-6))))
    return reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="LIDAR frames integrated before the queries")
    ap.add_argument("--clearance", type=float, default=0.0)
    ap.add_argument("--unknown-blocks", action="store_true")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed window per measurement")
    ap.add_argument("--mirror-sample", type=int, default=2048)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("pose_bench: no CUDA device (there is no CPU fallback)")
    info = gpu_info()
    m, w = build_map(args.frames)
    mir = m.HostMirror()
    r, unk = args.clearance, args.unknown_blocks
    rows = []
    for name, (h, yaw_only) in BODIES.items():
        for logn in (16, 20):
            n = 1 << logn
            P = make_poses(w, n, yaw_only, seed=logn)
            P_t = torch.from_numpy(P).cuda()

            def dev_call():
                out = m.CheckPoses(P_t, h, r, unknown_blocks=unk)
                torch.cuda.synchronize()
                return out
            reps = timed(dev_call, args.seconds)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                out = m.CheckPoses(P_t, h, r, unknown_blocks=unk)
            e1.record()
            e1.synchronize()
            dev_s = e0.elapsed_time(e1) * 1e-3 / reps
            hreps = timed(lambda: m.CheckPoses(P, h, r, unknown_blocks=unk), args.seconds)
            t0 = time.perf_counter()
            for _ in range(hreps):
                host = m.CheckPoses(P, h, r, unknown_blocks=unk)
            host_s = (time.perf_counter() - t0) / hreps
            dev = [x.cpu().numpy() for x in out]
            same = all(np.array_equal(a, b) for a, b in zip(dev, host))
            k = min(args.mirror_sample, n)
            mirror = mir.CheckPoses(P[:k], h, r, unknown_blocks=unk)
            same_mirror = all(np.array_equal(a[:k], b) for a, b in zip(host, mirror))
            cand = candidates(P, h, w)
            st = np.bincount(host[0], minlength=4)
            rows.append(dict(body=name, half_extents_m=h, rotations="yaw" if yaw_only else "full", n=n, device_ms=round(dev_s * 1e3, 4),
                             device_poses_per_s=n / dev_s, device_candidate_voxels_per_s=n * cand / dev_s,
                             host_entry_ms=round(host_s * 1e3, 3), host_entry_poses_per_s=n / host_s,
                             mean_candidate_voxels=round(cand, 1), clear=int(st[0]), blocked=int(st[1]), invalid=int(st[2]),
                             leaves_map=int(st[3]), device_equals_host_entry=bool(same), mirror_equals_host_entry_on_first=k,
                             mirror_equal=bool(same_mirror)))
            print(json.dumps(rows[-1]), flush=True)
    # single-pose latency: pinned host mirror (pure host code) against one device call + synchronise
    latency = {}
    for name, (h, yaw_only) in BODIES.items():
        one = make_poses(w, 1, yaw_only, seed=1)
        one_t = torch.from_numpy(one).cuda()
        for _ in range(20):
            mir.CheckPoses(one, h, r, unk); m.CheckPoses(one_t, h, r, unknown_blocks=unk)
        torch.cuda.synchronize()
        k = 2000 if name == "drone" else 100
        t0 = time.perf_counter()
        for _ in range(k):
            mir.CheckPoses(one, h, r, unk)
        mirror_us = (time.perf_counter() - t0) / k * 1e6
        t0 = time.perf_counter()
        for _ in range(k):
            m.CheckPoses(one_t, h, r, unknown_blocks=unk)
            torch.cuda.synchronize()
        device_us = (time.perf_counter() - t0) / k * 1e6
        latency[name] = dict(host_mirror=round(mirror_us, 2), device_call_and_sync=round(device_us, 2))
    mir.close()
    print(json.dumps(dict(gpu=info, map="lidar512 after %d frames (EXACT mode)" % args.frames, clearance_m=r, unknown_blocks=unk,
                          batches=rows, single_pose_us=latency,
                          note="latencies go through the Python binding (ctypes), so each includes its call overhead")))


if __name__ == "__main__":
    main()
