"""CPU: the segment traversal of fiesta_b200/csrc/fb_segment.h (compiled with g++ by tests/cpp/segment_test.cpp) against the exact
definition in tests/segref.py -- lattice endpoints, the walked voxels and their entry parameters voxel for voxel, the slab
partition the kernel's lanes walk, the kernel's combination of slab results, and the four outputs bit for bit -- on random and
adversarial segments over a synthetic record field holding every record kind."""
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from tests import segref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("seg") / "segment_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "segment_test.cpp"), "-o", out])
    return out


def records(gs, rng):
    """Packed records in device layout (z pitch rounded up to 4) with unknown, unreached, FB_DINF and finite entries."""
    gx, gy, gz = gs
    pz = (gz + 3) & ~3
    n = gx * gy * pz
    kind = rng.random(n)
    obs = np.stack([rng.integers(0, gs[k], n) for k in range(3)], -1).astype(np.uint64)
    code = ((obs[:, 0] + 1) << 20) | (obs[:, 1] << 10) | obs[:, 2]
    rec = np.where(kind < 0.2, 0, np.where(kind < 0.3, 1, code)).astype(np.uint64)
    rec = np.where((kind >= 0.3) & (kind < 0.4), rec | 0x80000000, rec)
    return rec.astype(np.uint32)


def distance_array(rec, gs, res):
    gx, gy, gz = gs
    pz = (gz + 3) & ~3
    R = rec.reshape(gx, gy, pz)[:, :, :gz]
    D = np.empty(gs)
    for x in range(gx):
        for y in range(gy):
            for z in range(gz):
                D[x, y, z] = segref.record_distance(int(R[x, y, z]), x, y, z, res)
    return D


def run(exe, gs, origin, res, size, rec, segs, r, flags):
    lo, hi = list(origin), [origin[k] + size[k] for k in range(3)]
    vals = list(gs) + list(origin) + [res] + lo + hi
    txt = [" ".join(float(v).hex() for v in vals), str(len(rec)), " ".join(str(int(c)) for c in rec),
           "%d %s %d" % (len(segs), float(r).hex(), flags)]
    txt += [" ".join(float(v).hex() for v in s) for s in segs]
    p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    lines = iter(p.stdout.splitlines())
    out = []
    for _ in segs:
        h = next(lines).split()
        walk = None
        if h[1] == "ok":
            q = [int(x) for x in h[2:8]]
            nslabs, slabs_equal, kernel_equal, nv = int(h[8]), h[9] == "1", h[10] == "1", int(h[11])
            vox = []
            for _ in range(nv):
                v = [int(x) for x in next(lines).split()[1:]]
                vox.append((tuple(v[:3]), Fraction(v[3], v[4])))
            walk = dict(qa=q[:3], qb=q[3:], nslabs=nslabs, slabs_equal=slabs_equal, kernel_equal=kernel_equal, voxels=vox)
        rr = next(lines).split()
        out.append((walk, (int(rr[1]), int(rr[2]), float.fromhex(rr[3]), float.fromhex(rr[4]))))
    return out


def verify(exe, gs, origin, res, size, segs, seed, clearances):
    rng = np.random.default_rng(seed)
    rec = records(gs, rng)
    D = distance_array(rec, gs, res)
    lo, hi = list(origin), [origin[k] + size[k] for k in range(3)]
    walked, seen = 0, set()
    for r in clearances:
        for flags in (0, 1):
            got = run(exe, gs, origin, res, size, rec, segs, r, flags)
            for s, (walk, res4) in zip(segs, got):
                want = segref.check(s, origin, res, lo, hi, D, r, flags == 1)
                if walk is not None:
                    qa, qb = segref.lattice(s[:3], origin, res), segref.lattice(s[3:], origin, res)
                    assert walk["qa"] == qa and walk["qb"] == qb, s
                    assert walk["voxels"] == segref.walk(qa, qb), s
                    assert walk["slabs_equal"] and walk["kernel_equal"], s
                    walked += len(walk["voxels"])
                else:
                    assert want[0] == 2, s
                assert segref.same(res4, want), (s, r, flags, res4, want)
                seen.add((want[0], flags))
    assert {(0, 0), (1, 0), (1, 1)} <= seen, seen                           # clear and blocked segments, with and without the flag
    return walked


def test_dyadic_grid_adversarial_and_random(exe):
    """res = 1/8 and a dyadic origin: voxel units are exact, so segments through exact edges and corners stay exact."""
    origin, res, size = (-4.0, -4.0, -2.0), 0.125, (8.0, 6.0, 3.75)
    gs = (64, 48, 30)
    rng = np.random.default_rng(1)
    units = segref.adversarial_voxel_units(gs, rng)
    segs = [list(np.concatenate([np.asarray(origin) + u[:3] * res, np.asarray(origin) + u[3:] * res])) for u in units]
    for _ in range(300):
        a = rng.uniform(origin, np.asarray(origin) + size)
        b = a + rng.normal(0, 1.5, 3)
        segs.append(list(np.concatenate([a, b])))                            # some leave the map: status 2
    segs.append([math.nan, 0, 0, 0, 0, 0])
    walked = verify(exe, gs, origin, res, size, segs, seed=2, clearances=(0.0, res, 0.3, 2.0))
    assert walked > 10000


def test_decimal_grid_random(exe):
    """res = 0.1, origin -3.2: endpoints land off the lattice planes through fp64 rounding like real planner queries."""
    origin, res, size = (-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.0)
    gs = (64, 64, 30)
    rng = np.random.default_rng(3)
    segs = []
    for _ in range(600):
        a = rng.uniform(np.asarray(origin) - 0.2, np.asarray(origin) + np.asarray(size) + 0.2)
        b = a + rng.normal(0, 0.3 if rng.random() < 0.5 else 3.0, 3)
        segs.append(list(np.concatenate([a, b])))
    hi = np.asarray(origin) + np.asarray(size)
    segs.append(list(np.concatenate([np.asarray(origin), hi])))             # lower corner to upper corner, both on the faces
    segs.append(list(np.concatenate([hi, hi])))
    verify(exe, gs, origin, res, size, segs, seed=4, clearances=(0.0, res, 0.45))


def test_full_length_axis(exe):
    """2046 voxels along x (the grid limit): segments across the whole axis exercise the largest lattice coordinates."""
    origin, res, size = (0.0, 0.0, 0.0), 1.0, (2046.0, 4.0, 4.0)
    gs = (2046, 4, 4)
    segs = [[0, 1.5, 2.5, 2046, 2.5, 0.5], [2046, 4, 4, 0, 0, 0], [0, 0, 0, 2046, 4, 4], [2046, 0.5, 0.5, 0, 0.5, 0.5],
            [0.1, 3.9, 0.1, 2045.9, 0.1, 3.9], [1023, 2, 2, 1023, 2, 2], [0, 2, 2, 2046, 2, 2]]
    walked = verify(exe, gs, origin, res, size, segs, seed=5, clearances=(0.0, 1.0, 3.0))
    assert walked > 2046 * 6
