"""CPU: safe flight corridors.  The sequential rule of fiesta_b200/csrc/fb_corridor.h (compiled with g++, traversability from
fb_seg_blocks voxel by voxel) equals tests/corridorref.py output for output, layer counts included, on random grids off the word
and tile lattices (Gz = 30 among them), limit boxes one voxel thick or on the grid's faces, three clearances, both flag settings and
max_steps of 0, asymmetric and binding.  On the same grids the boxes are traversable and maximal, consecutive boxes share a voxel
and every path voxel before blocked_at is covered; a crafted L-shaped obstacle pins the face order."""
import os
import subprocess

import numpy as np
import pytest

from tests import corridorref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.125
ORIGIN = (-2.0, -3.0, -1.0)
GRIDS = [(37, 35, 30), (9, 70, 33), (40, 3, 66)]
CLEARANCES = (0.0, RES, 0.3)
MAX_STEPS = [(0, 0, 0), (3, 1, 7), (1000, 1000, 1000), (2, 2, 0), (40, 40, 20)]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("corridor") / "corridor_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "corridor_test.cpp"), "-o", out])
    return out


def records(gs, rng, n_obstacles):
    """Packed records in device layout: the nearest of some random obstacles (walls among them), a few never-observed voxels, a
    few unreached ones and a few reset by a local-map update (bit 31)."""
    gx, gy, gz = gs
    pz = (gz + 3) & ~3
    v = np.stack(np.meshgrid(np.arange(gx), np.arange(gy), np.arange(pz), indexing="ij"), -1).reshape(-1, 3)
    ob = rng.integers(0, gs, (n_obstacles, 3))
    wall = rng.integers(0, gs)
    ob = np.concatenate([ob, [(wall[0], y, z) for y in range(gy // 3) for z in range(gz)]])
    best = np.full(len(v), np.iinfo(np.int64).max)
    code = np.zeros(len(v), np.uint64)
    for o in ob:
        d = np.sum((v - o) ** 2, axis=1)
        better = d < best
        best = np.where(better, d, best)
        code = np.where(better, ((np.uint64(o[0]) + 1) << 20) | (np.uint64(o[1]) << 10) | np.uint64(o[2]), code)
    kind = rng.random(len(v))
    rec = np.where(kind < 0.03, 0, np.where(kind < 0.04, 1, code)).astype(np.uint64)
    rec = np.where((kind >= 0.04) & (kind < 0.05), rec | 0x80000000, rec)
    rec = np.where(v[:, 2] >= gz, 0, rec)
    return rec.astype(np.uint32)


def distance_array(rec, gs):
    """export_distance() of the records: fb_record_distance's expression, -10000 never observed, +10000 unreached or reset."""
    gx, gy, gz = gs
    R = rec.reshape(gx, gy, (gz + 3) & ~3)[:, :, :gz].astype(np.int64)
    v = np.stack(np.meshgrid(np.arange(gx), np.arange(gy), np.arange(gz), indexing="ij"), -1)
    c = R & 0x7fffffff
    o = np.stack([(c >> 20) - 1, (c >> 10) & 1023, c & 1023], -1)
    d = (v - o).astype(np.float64)
    D = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]) * RES
    D = np.where((c == 1) | ((R & 0x80000000) != 0), 10000.0, D)
    return np.where(c == 0, -10000.0, D)


def limit_boxes(gs):
    gx, gy, gz = gs
    return [((0, 0, 0), (gx - 1, gy - 1, gz - 1)),                                   # the whole grid
            ((1, min(2, gy - 1), 3), (gx - 2, gy - 1, gz - 4)),                       # on the +y face
            ((gx // 2, 0, 0), (gx // 2, gy - 1, gz - 1)),                             # one voxel thick in x, on four faces
            ((0, gy // 3, gz - 1), (gx - 1, gy - 1, gz - 1))]                         # one voxel thick in z, on the +z face


def random_paths(L, rng, n):
    """Random 26-neighbour walks that start on a traversable voxel and may leave the traversable set (blocked seeds) or L (status
    2), jumps between distant voxels, repeated voxels, an empty path and 1-voxel paths."""
    free = np.argwhere(L.T) + L.lo
    paths = [np.zeros((0, 3), np.int64), L.lo[None].copy()]
    if len(free):
        paths.append(free[rng.integers(len(free))][None])
    for i in range(n):
        if not len(free):
            break
        p = [free[rng.integers(len(free))]]
        for _ in range(int(rng.integers(1, 60))):
            step = rng.integers(-1, 2, 3) if rng.random() < 0.9 else rng.integers(-4, 5, 3)
            q = p[-1] + step
            if i % 3 == 0 or np.all((q >= L.lo) & (q <= L.hi)):                  # a third of them may step outside L
                p.append(q)
            if rng.random() < 0.05:
                p.append(p[-1])
        paths.append(np.array(p))
    return paths


def run(exe, rec, gs, box, r, unk, ms, mode_lines):
    txt = ["%d %d %d" % gs, " ".join(float(x).hex() for x in list(ORIGIN) + [RES]), str(len(rec)), " ".join(str(int(c)) for c in rec),
           "%s %d" % (float(r).hex(), int(unk)), "%d %d %d %d %d %d" % (*box[0], *box[1]), "%d %d %d" % tuple(ms)] + mode_lines
    p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout.splitlines()


def ints(line):
    return [int(x) for x in line.split()]


def seed_of(P, j):
    P = np.asarray(P)
    return (P[0], P[0]) if j == 0 else (np.minimum(P[j - 1], P[j]), np.maximum(P[j - 1], P[j]))


def check_properties(L, ms, paths, want):
    status, nb, bl, boxes, _ = want
    for p, P in enumerate(paths):
        lo, hi, first = boxes[p]
        for k in range(nb[p]):
            assert L.free(lo[k], hi[k])
            s_lo, s_hi = seed_of(P, first[k])
            assert corridorref.maximal(L, ms, s_lo, s_hi, lo[k], hi[k])
            assert np.all(lo[k] <= s_lo) and np.all(s_hi <= hi[k])
            if k:
                shared = np.asarray(P)[first[k] - 1]
                for b in (k - 1, k):
                    assert np.all(lo[b] <= shared) and np.all(shared <= hi[b])
        covered = len(P) if status[p] == 0 else (bl[p] if status[p] == 1 else 0)
        for v in np.asarray(P)[:covered]:
            assert any(np.all(lo[k] <= v) and np.all(v <= hi[k]) for k in range(nb[p]))


@pytest.mark.parametrize("gs", GRIDS)
def test_header_equals_corridorref(exe, gs):
    rng = np.random.default_rng(sum(gs))
    rec = records(gs, rng, 12)
    D = distance_array(rec, gs)
    statuses, seeds_seen, grown, ci = set(), set(), 0, 0
    for box in limit_boxes(gs):
        for r in CLEARANCES:
            for unk in (False, True):
                ms = MAX_STEPS[ci % len(MAX_STEPS)]
                ci += 1
                L = corridorref.Limit(D, gs, box, r, unk)
                paths = random_paths(L, rng, 25)
                want = corridorref.corridors(L, paths, ms)
                lines = run(exe, rec, gs, box, r, unk, ms, ["paths", str(len(paths))] +
                            ["%d %s" % (len(P), " ".join(str(int(x)) for x in np.asarray(P).reshape(-1))) for P in paths])
                at = 0
                for p in range(len(paths)):
                    assert ints(lines[at]) == [want[0][p], want[1][p], want[2][p]], (box, r, unk, p)
                    got = np.array([ints(x) for x in lines[at + 1:at + 1 + want[1][p]]]).reshape(-1, 7)
                    lo, hi, first = want[3][p]
                    assert np.array_equal(got[:, :3], lo) and np.array_equal(got[:, 3:6], hi) and np.array_equal(got[:, 6], first)
                    at += 1 + want[1][p]
                st = want[4]
                assert ints(lines[at].split(None, 1)[1]) == [st["boxes"], st["layers_tested"], st["layers_grown"]]
                check_properties(L, ms, paths, want)
                statuses |= set(int(s) for s in want[0])
                grown += st["layers_grown"]
                # independent seeds: random boxes, inverted, outside L, blocked
                lo = rng.integers(np.asarray(box[0]) - 2, np.asarray(box[1]) + 3, (40, 3))
                hi = lo + rng.integers(-1, 3, (40, 3))
                free = np.argwhere(L.T) + L.lo
                if len(free):
                    f = free[rng.integers(len(free), size=20)]
                    lo, hi = np.concatenate([lo, f]), np.concatenate([hi, f])
                sw = corridorref.inflate_boxes(L, lo, hi, ms)
                lines = run(exe, rec, gs, box, r, unk, ms, ["inflate", str(len(lo))] +
                            ["%d %d %d %d %d %d" % (*a, *b) for a, b in zip(lo, hi)])
                got = np.array([ints(x) for x in lines[:len(lo)]])
                assert np.array_equal(got[:, 0], sw[0]) and np.array_equal(got[:, 1:4], sw[1]) and np.array_equal(got[:, 4:], sw[2])
                assert ints(lines[len(lo)].split(None, 1)[1]) == [sw[3]["boxes"], sw[3]["layers_tested"], sw[3]["layers_grown"]]
                for i in np.nonzero(sw[0] == 0)[0]:
                    assert L.free(sw[1][i], sw[2][i]) and corridorref.maximal(L, ms, lo[i], hi[i], sw[1][i], sw[2][i])
                seeds_seen |= set(int(s) for s in sw[0])
    assert statuses == {0, 1, 2} and seeds_seen == {0, 1, 2} and grown > 0


def test_max_steps_binds_in_open_space(exe):
    gs = (20, 21, 22)
    rec = np.ones(20 * 21 * 24, np.uint32)                                   # observed, no obstacle
    D = distance_array(rec, gs)
    box = ((0, 0, 0), (19, 20, 21))
    for ms in ((0, 0, 0), (3, 1, 7), (2, 0, 100)):
        L = corridorref.Limit(D, gs, box, 0.3, True)
        want = corridorref.inflate_boxes(L, [(10, 10, 10)], [(11, 10, 10)], ms)
        exp_lo = [max(0, 10 - ms[0]), max(0, 10 - ms[1]), max(0, 10 - ms[2])]
        exp_hi = [min(19, 11 + ms[0]), min(20, 10 + ms[1]), min(21, 10 + ms[2])]
        assert want[1][0].tolist() == exp_lo and want[2][0].tolist() == exp_hi
        lines = run(exe, rec, gs, box, 0.3, 1, ms, ["inflate", "1", "10 10 10 11 10 10"])
        assert ints(lines[0]) == [0] + exp_lo + exp_hi


def test_face_order_is_pinned_by_an_l_shaped_obstacle(exe):
    """Seed (5, 5, 1), max_steps (2, 2, 0) and an L of obstacles at (7, 7), (8, 7), (7, 8): growing x first claims the corner
    column x = 7 (box x 3..7, y 3..6); growing y first claims the row y = 7 instead (x 3..6, y 3..7)."""
    gs = (12, 12, 3)
    rec = np.ones(12 * 12 * 4, np.uint32).reshape(12, 12, 4)
    for x, y in ((7, 7), (8, 7), (7, 8)):
        rec[x, y, :3] = ((x + 1) << 20) | (y << 10) | np.arange(3)
    rec[:, :, 3] = 0
    rec = rec.reshape(-1)
    D = distance_array(rec, gs)
    box = ((0, 0, 0), (11, 11, 2))
    L = corridorref.Limit(D, gs, box, 0.0, False)
    seed = (5, 5, 1)
    lo, hi, _, _ = corridorref.inflate(L, (2, 2, 0), seed, seed)
    assert (lo, hi) == ([3, 3, 1], [7, 6, 1])
    y_first = ((1, False), (1, True), (0, False), (0, True), (2, False), (2, True))
    assert corridorref.inflate(L, (2, 2, 0), seed, seed, order=y_first)[:2] == ([3, 3, 1], [6, 7, 1])
    lines = run(exe, rec, gs, box, 0.0, 0, (2, 2, 0), ["inflate", "1", "5 5 1 5 5 1"])
    assert ints(lines[0]) == [0, 3, 3, 1, 7, 6, 1]
