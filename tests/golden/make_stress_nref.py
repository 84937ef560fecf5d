"""Fixture generator (CPU): the reference's expansion counts for the dynamic-obstacle stress frames of
scripts/stress256.py -> tests/golden/stress_nref.json.      python tests/golden/make_stress_nref.py [frames]"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from tests import scenes  # noqa: E402
from oracle import pyoracle  # noqa: E402
import stress256  # noqa: E402


def main(n):
    m = pyoracle.OracleMap(stress256.ORIGIN, stress256.RES, stress256.SIZE)
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(m.grid_size)
    m.SetOccupancyBatchVox(allv, np.zeros(len(allv), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    rows = []
    for f, (vox, occ) in enumerate(stress256.frames(n)):
        m.SetOccupancyBatchVox(vox, occ)
        t0 = time.perf_counter(); m.UpdateOccupancy(True); m.UpdateESDF(); dt = time.perf_counter() - t0
        s = m.stats()
        rows.append(dict(frame=f, expansions=s["expansions"], inserts=s["inserts"], deletes=s["deletes"], cpu_update_s=round(dt, 3)))
        print(rows[-1], flush=True)
    json.dump(dict(oracle=m.kind, frames=rows), open(stress256.NREF, "w"), indent=1)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 6)
