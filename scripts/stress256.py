"""Dynamic-obstacle stress (BASELINE.json configs[4], SURVEY.md 8(d)-5): 256^3 grid, every voxel observed, then every frame a
uniformly random 20 % of the voxels is toggled occupied <-> free (toggle probabilities: one observation flips a voxel).

  python tests/golden/make_stress_nref.py 6      # CPU oracle -> tests/golden/stress_nref.json
  python scripts/stress256.py --frames 6         # GPU: FAST mode, events resident in HBM; prints one JSON line
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import scenes  # noqa: E402

ORIGIN, RES, SIZE = (-6.4, -6.4, -6.4), 0.05, (12.8, 12.8, 12.8)
NREF = os.path.join(ROOT, "tests", "golden", "stress_nref.json")


def frames(n, G=256):
    state = np.zeros(G * G * G, np.uint8)
    out = []
    for f in range(n):
        rng = np.random.default_rng(6 + f)
        idx = rng.choice(state.size, state.size // 5, replace=False)
        occ = (1 - state[idx]).astype(np.uint8)
        state[idx] = occ
        vox = np.stack([idx // (G * G), idx // G % G, idx % G], -1).astype(np.int32)
        out.append((vox, occ))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=6)
    a = ap.parse_args()
    import torch
    import fiesta_b200
    nref = json.load(open(NREF))["frames"] if os.path.exists(NREF) else []
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode="fast")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(m.grid_size)
    m.SetOccupancyBatchVox(allv, np.zeros(len(allv), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    fr = frames(a.frames)
    dev = [(torch.from_numpy(v).cuda(), torch.from_numpy(o).cuda()) for v, o in fr]
    torch.cuda.synchronize()
    per = []
    for f, (v, o) in enumerate(dev):
        t0 = time.perf_counter()
        m.SetOccupancyBatchVoxDevice(v.data_ptr(), o.data_ptr(), v.shape[0])
        m.UpdateOccupancy(True)
        m.UpdateESDF()
        m.synchronize()
        dt = time.perf_counter() - t0
        s = m.stats()
        per.append(dict(frame=f, ms=1000 * dt, inserts=s["inserts"], deletes=s["deletes"], changed=s["voxels_changed"], reset=s["voxels_reset"],
                        ms_esdf=s["ms_update_esdf"], ms_scan=s["ms_esdf_delete_scan"], ms_wave=s["ms_esdf_wavefront"], gens=s["generations"],
                        n_ref=nref[f]["expansions"] if f < len(nref) else None, cpu_s=nref[f]["cpu_update_s"] if f < len(nref) else None))
    timed = per[1:]                                            # frame 0 warms up
    tot = sum(p["ms"] for p in timed) / 1000
    ref = sum(p["n_ref"] for p in timed if p["n_ref"]) if all(p["n_ref"] for p in timed) else None
    print(json.dumps(dict(workload="stress256: 256^3, 20 % of the voxels toggled per frame (3 355 443 SetOccupancy events), FAST mode, events in HBM",
                          frames=len(timed), ms_per_frame=1000 * tot / len(timed), changed_per_s=sum(p["changed"] for p in timed) / tot,
                          n_ref_per_s=(ref / tot) if ref else None, cpu_reference_n_ref_per_s=(ref / sum(p["cpu_s"] for p in timed)) if ref else None,
                          per_frame=per)))


if __name__ == "__main__":
    main()
