import os, sys, json, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench, fiesta_b200
from tests import scenes
wl = sys.argv[1] if len(sys.argv) > 1 else 'lidar512'
nfr = int(sys.argv[2]) if len(sys.argv) > 2 else 8
w = bench.WORKLOADS[wl]
frames = bench.make_frames(wl, nfr)
m = fiesta_b200.ESDFMap(w['origin'], w['res'], w['size'], device=0, mode='exact')
m.SetParameters(*scenes.PARAMS_DEFAULT)
for f, fr in enumerate(frames):
    t0 = time.perf_counter()
    m.RaycastFrame(fr['pts'], fr['T'], w['min_len'], w['max_len'])
    if m.CheckUpdate():
        m.SetOriginalRange(); m.UpdateOccupancy(True); m.UpdateESDF()
    s = m.stats()
    print(f, round((time.perf_counter()-t0)*1e3, 1), {k: s[k] for k in ('ms_raycast','ms_update_occupancy','ms_update_esdf','expansions','inserts','deletes','generations','voxels_changed','voxels_reset')}, flush=True)
