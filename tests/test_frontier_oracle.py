"""CPU: the frontier definition (tests/frontierref.py) and the predicate and centroid of fiesta_b200/csrc/fb_frontier.h.

The GPU tests compare the device's labels with scipy's 26-connected labelling renumbered by smallest index.  That is only sound if
the device's schedule -- components inside each 8^3 tile, then unions across tiles in whatever order the hardware runs them -- always
reaches the same components with the same smallest members.  These tests check scipy against an independent BFS, run the tile /
union schedule on the CPU with random union orders, and include components that are joined only across a tile face, edge or corner
and a single-voxel diagonal chain through many tiles.  The header's predicate and centroid (compiled with g++) must give
frontierref's bits."""
import itertools
import os
import subprocess

import numpy as np
import pytest

from tests import frontierref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.1
ORIGIN = (-3.2, -3.2, -1.6)
L_OCC = frontierref.l_occ(0.8)


def synth(gs, rng, p_unknown=0.35, p_unreached=0.1):
    """export_distance() / export_occupancy()-like arrays: never observed (-10000), unreached (+10000), distances that are
    multiples of sqrt of integers times RES, and log-odds on both sides of l_occ."""
    n = int(np.prod(gs))
    d = np.sqrt(rng.integers(0, 40, n).astype(np.float64)) * RES
    kind = rng.random(n)
    D = np.where(kind < p_unknown, -10000.0, np.where(kind < p_unknown + p_unreached, 10000.0, d))
    O = rng.normal(0.0, 2.0, n)
    return D, O


CASES = [  # grid, box (lo, hi)
    ((24, 20, 17), ((0, 0, 0), (23, 19, 16))),
    ((13, 11, 9), ((2, 1, 0), (12, 10, 8))),
    ((10, 19, 12), ((4, 0, 0), (4, 18, 11))),          # 1 voxel thick in x
    ((17, 9, 21), ((0, 3, 2), (16, 3, 20))),           # 1 voxel thick in y
    ((9, 30, 7), ((1, 2, 3), (8, 27, 3))),             # 1 voxel thick in z
    ((19, 21, 18), ((0, 0, 17), (18, 20, 17))),        # on the grid's upper z face
    ((19, 21, 18), ((18, 0, 0), (18, 20, 17))),        # on the grid's upper x face
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_scipy_equals_bfs_and_tile_schedule(case):
    gs, box = CASES[case]
    rng = np.random.default_rng(case)
    seen = 0
    for p_unknown in (0.2, 0.5):
        D, O = synth(gs, rng, p_unknown)
        for r in (0.0, RES, 2.5 * RES):
            F = frontierref.frontier_mask(D, O, gs, box, r, L_OCC)
            lab = frontierref.label_scipy(F)
            assert np.array_equal(lab >= 0, F)
            assert np.array_equal(lab, frontierref.label_bfs(F)), (p_unknown, r)
            for seed in range(2):
                assert np.array_equal(lab, frontierref.label_schedule(F, np.random.default_rng(seed))), (p_unknown, r, seed)
            for min_size in (1, 2, 5):
                check_extract(D, O, gs, box, r, min_size, lab)
            seen += int(lab.max()) + 1
    assert seen > 0


def check_extract(D, O, gs, box, r, min_size, lab):
    """frontierref.extract's outputs against a direct per-cluster computation from the labels."""
    e = frontierref.extract(D, O, gs, box, r, L_OCC, min_size, RES, ORIGIN)
    lo = np.asarray(box[0])
    k = 0
    vox = []
    for c in range(int(lab.max()) + 1):
        m = np.argwhere(lab == c) + lo                                    # index order
        if len(m) < min_size:
            assert np.all(e["labels"][lab == c] == -1)
            continue
        assert np.all(e["labels"][lab == c] == k)
        assert e["size"][k] == len(m) and tuple(e["rep"][k]) == tuple(m[0])
        assert tuple(e["bbox_lo"][k]) == tuple(m.min(0)) and tuple(e["bbox_hi"][k]) == tuple(m.max(0))
        for a in range(3):
            s = int(sum(int(x) for x in m[:, a]))
            assert e["centroid"][k, a] == (float(s) / float(len(m)) + 0.5) * RES + ORIGIN[a]
        vox += [tuple(x) for x in m]
        k += 1
    assert e["stats"]["kept_clusters"] == k and [tuple(x) for x in e["voxels"]] == vox


def tile_boundary_masks():
    """Frontier masks of 24^3 whose components touch only across a tile face, an edge, a corner, and a diagonal chain of single
    voxels that crosses from tile to tile through corners only."""
    out = []
    for a, b in [((7, 3, 3), (8, 3, 3)), ((7, 7, 3), (8, 8, 3)), ((3, 7, 8), (3, 8, 7)), ((7, 7, 7), (8, 8, 8)),
                 ((15, 8, 16), (16, 7, 15))]:
        F = np.zeros((24, 24, 24), bool)
        F[a] = F[b] = True
        F[2, 20, 20] = True                                               # a separate cluster after them in index order
        out.append((F, 2))
    F = np.zeros((24, 24, 24), bool)
    for i in range(24):
        F[i, i, 23 - i] = True
    out.append((F, 1))
    F = np.zeros((40, 24, 8), bool)                                       # a serpentine through a row of tiles
    for y in range(0, 24, 2):
        F[:, y, 3] = True
        F[39 if y % 4 == 0 else 0, y + 1 if y + 1 < 24 else y, 3] = True
    out.append((F, 1))
    return out


@pytest.mark.parametrize("case", range(7))
def test_components_joined_only_across_tile_boundaries(case):
    F, clusters = tile_boundary_masks()[case]
    lab = frontierref.label_scipy(F)
    assert int(lab.max()) + 1 == clusters
    assert np.array_equal(lab, frontierref.label_bfs(F))
    for seed in range(4):
        assert np.array_equal(lab, frontierref.label_schedule(F, np.random.default_rng(seed)))
    # shifting the box shifts the tile lattice: the same components from the other side of each boundary
    for sh in itertools.product((0, 3), repeat=3):
        G = F[sh[0]:, sh[1]:, sh[2]:]
        assert np.array_equal(frontierref.label_schedule(G, np.random.default_rng(7)), frontierref.label_scipy(G))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("frontier") / "frontier_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "cpp", "frontier_test.cpp"), "-o", out])
    return out


def synth_records(gs, rng):
    """Packed records: never observed (0), observed without obstacle (1), local-map reset (bit 31) with or without an obstacle,
    and obstacles near the voxel."""
    n = int(np.prod(gs))
    v = np.stack(np.unravel_index(np.arange(n), gs), -1)
    ob = np.clip(v + rng.integers(-3, 4, v.shape), 0, np.asarray(gs) - 1)
    packed = ((ob[:, 0] + 1).astype(np.uint64) << 20) | (ob[:, 1].astype(np.uint64) << 10) | ob[:, 2].astype(np.uint64)
    kind = rng.random(n)
    rec = np.where(kind < 0.3, 0, np.where(kind < 0.4, 1, packed)).astype(np.uint64)
    rec = np.where((kind > 0.9) & (kind < 0.95), rec | (1 << 31), rec)
    return rec, rng.normal(0.0, 2.0, n)


def test_header_predicate_and_centroid(exe):
    rng = np.random.default_rng(12)
    total = 0
    for gs, box in CASES + [((16, 16, 30), ((0, 0, 0), (15, 15, 29)))]:   # Gz = 30: padded pitch
        rec, O = synth_records(gs, rng)
        for r in (0.0, RES, 2.5 * RES):
            sums = rng.integers(0, 2046 * 10**6, 200)
            cnt = rng.integers(1, 10**6, 200)
            txt = ["%d %d %d %s" % (*gs, float(RES).hex()), " ".join(float(x).hex() for x in ORIGIN),
                   "%s %s" % (float(L_OCC).hex(), float(r).hex()), " ".join(str(int(x)) for x in list(box[0]) + list(box[1])),
                   " ".join(str(int(x)) for x in rec), " ".join(float(x).hex() for x in O), str(len(sums))]
            txt += ["%d %d" % (s, c) for s, c in zip(sums, cnt)]
            p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr
            lines = p.stdout.splitlines()
            D = np.array([float.fromhex(x) for x in lines[0].split()])
            got = np.array([c == "1" for c in lines[1]]).reshape([b - a + 1 for a, b in zip(*box)])
            want = frontierref.frontier_mask(D, O, gs, box, r, L_OCC)
            assert np.array_equal(got, want), r
            total += int(want.sum())
            cen = [float.fromhex(x) for x in lines[2:]]
            ref = (sums.astype(np.float64) / cnt.astype(np.float64) + 0.5) * RES + ORIGIN[0]
            assert np.array_equal(np.array(cen), ref)
    assert total > 100
