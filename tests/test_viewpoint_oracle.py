"""CPU: viewpoint coverage.  The range and field-of-view predicates of fiesta_b200/csrc/fb_view.h (compiled with g++, no
contraction) give tests/viewref.py's bits on adversarial pairs; the kernel's chunk decomposition covers every (candidate, member)
pair exactly once; and viewref.score with tests/segref.py as its line of sight equals both a brute-force loop over pairs and the
header's own sequential run of the kernel's per-lane logic, on small random grids with and without FIESTA_SEGMENT_UNKNOWN_BLOCKS."""
import math
import os
import subprocess

import numpy as np
import pytest

from tests import segref, viewref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.125
ORIGIN = (-2.0, -3.0, -1.0)              # binary-exact: voxel centres and offsets are exact


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("view") / "viewpoint_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "cpp", "viewpoint_test.cpp"), "-o", out])
    return out


def hx(vals):
    return " ".join(float(v).hex() for v in vals)


def run(exe, txt):
    p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout.splitlines()


def sensor_lines(R, max_range, tan):
    R = np.asarray(R, np.float64).reshape(-1, 9)
    return [str(len(R)), hx(R.reshape(-1)), hx([max_range, tan[0], tan[1]])]


def adversarial_pairs(rng):
    """(member voxel, candidate position) pairs: exactly on a field-of-view plane and a hair inside or outside it, exactly at
    max_range and a hair beyond, s0 == 0, -0.0 coordinates, tiny and map-sized offsets, and random ones."""
    v0 = np.array([20, 30, 12])
    c0 = (v0 + 0.5) * RES + np.asarray(ORIGIN)
    ds = []
    for s in (1.0, 2.0, 0.375):
        for sg in (1, -1):
            ds += [(s, sg * 0.75 * s, 0.0), (s, 0.0, sg * 0.5 * s), (s, sg * 0.75 * s, sg * 0.5 * s)]   # on the planes (tan 0.75, 0.5)
    ds += [(0.375, 0.5, 0.0), (0.0, 0.375, 0.5), (0.3, 0.4, 0.0), (0.0, 0.0, 0.625), (-0.375, -0.5, 0.0)]   # |d| = 0.625 = max_range
    ds += [(0.0, 0.25, 0.0), (0.0, 0.0, 0.0), (0.0, -0.0, 0.0), (-0.0, 0.5, -0.25), (5e-324, 0.0, 0.0), (1e-300, 1e-300, -1e-300),
           (1e-17, 7.5e-18, 0.0), (150.0, 112.5, 75.0), (-300.0, 0.0, 1.0)]
    out = []
    for d in ds:
        d = np.array(d)
        out.append((v0, c0 - d))
        for eps in (1, -1):
            out.append((v0, np.nextafter(c0 - d, c0 - d + eps)))                    # a hair either way on every axis
    for _ in range(300):
        v = rng.integers(0, 40, 3)
        out.append((v, (v + rng.uniform(-8, 8, 3)) * RES + np.asarray(ORIGIN)))
    return out


def orientations(rng):
    R = [np.eye(3), viewref.yaw(0.0), viewref.yaw(np.pi / 2), viewref.yaw(np.pi), viewref.yaw_pitch(0.3, -0.4),
         -np.eye(3), np.array([[1.0, -0.0, 0.0], [-0.0, 1.0, -0.0], [0.0, 0.0, -1.0]])]
    R += [rng.normal(0, 1, (3, 3)) for _ in range(5)]                       # not orthonormal: used as given
    R += list(viewref.yaws(8)) + [viewref.yaw(a) for a in rng.uniform(0, 2 * np.pi, 12)]
    return np.stack(R[:32])


def test_predicates_match_viewref_on_adversarial_pairs(exe):
    rng = np.random.default_rng(1)
    pairs = adversarial_pairs(rng)
    R = orientations(rng)
    assert len(R) == 32
    inside = 0
    for max_range, tan in ((0.625, (0.75, 0.5)), (4.5, (1.0, math.tan(math.pi / 6))), (1e3, (0.75, 0.5))):
        txt = ["pairs", hx([RES] + list(ORIGIN))] + sensor_lines(R, max_range, tan) + [str(len(pairs))]
        txt += ["%d %d %d %s" % (*v, hx(p)) for v, p in pairs]
        lines = run(exe, txt)
        for (v, p), line in zip(pairs, lines):
            a, b = line.split()
            _, d = viewref.offsets(np.array([v]), p, ORIGIN, RES)
            want_r = bool(viewref.in_range(d, max_range)[0])
            m = viewref.view_mask(R, d, *tan)[0]
            want_m = int(sum(1 << j for j in range(len(R)) if m[j]))
            assert (a == "1", int(b)) == (want_r, want_m), (v, p, max_range, tan)
            inside += want_r and want_m != 0
    assert inside > 50
    # the exact boundaries are counted and a hair beyond is not (identity orientation, tan 0.75 / 0.5, range 0.625)
    v0 = np.array([20, 30, 12])
    c0 = (v0 + 0.5) * RES + np.asarray(ORIGIN)
    d = lambda p: viewref.offsets(np.array([v0]), p, ORIGIN, RES)[1]
    on_planes, at_range = d(c0 - np.array([1.0, 0.75, 0.5])), d(c0 - np.array([0.375, 0.5, 0.0]))
    assert np.array_equal(on_planes[0], [1.0, 0.75, 0.5]) and np.array_equal(at_range[0], [0.375, 0.5, 0.0])
    assert viewref.view_mask(np.eye(3), on_planes, 0.75, 0.5)[0, 0] and viewref.in_range(at_range, 0.625)[0]
    for k in (1, 2):
        p = c0 - np.array([1.0, 0.75, 0.5])
        p[k] -= 2.0 ** -40                                                  # |s_k| a hair above tan * s0 (exact)
        assert not viewref.view_mask(np.eye(3), d(p), 0.75, 0.5)[0, 0]
    p = c0 - np.array([0.375, 0.5, 0.0])
    p[1] -= 2.0 ** -40
    assert not viewref.in_range(d(p), 0.625)[0]


def test_chunk_decomposition_covers_every_pair_once(exe):
    rng = np.random.default_rng(2)
    for trial in range(6):
        n = int(rng.integers(1, 200))
        size = rng.choice([0, 1, 5, 31, 32, 33, 64, 65, 200], n)
        size[rng.random(n) < 0.2] = 0                                       # candidates that are not scored
        if trial == 0:
            size[:] = 0
        if trial == 1:
            size[n // 2] = 40000                                            # one cluster over many chunks
        if trial == 2:
            size[0], size[-1] = 0, 0                                        # zero work at both ends
        lines = run(exe, ["chunks", str(n), " ".join(str(int(s)) for s in size)])
        total = int(lines[0])
        assert total == int(sum((int(s) + 31) // 32 for s in size))
        seen = [np.zeros(int(s), np.int32) for s in size]
        for line in lines[1:]:
            i, lo, hi = (int(x) for x in line.split())
            assert 0 <= lo < hi <= size[i] and hi - lo <= 32
            seen[i][lo:hi] += 1
        assert all(np.all(s == 1) for s in seen)


def records(gs, rng):
    """Packed records in device layout (z pitch rounded up to 4): never observed, unreached, local-map reset (bit 31), obstacles
    at the voxel itself (distance 0: they block the line of sight) and obstacles nearby."""
    gx, gy, gz = gs
    pz = (gz + 3) & ~3
    v = np.stack(np.meshgrid(np.arange(gx), np.arange(gy), np.arange(pz), indexing="ij"), -1).reshape(-1, 3)
    ob = np.clip(v + rng.integers(-2, 3, v.shape), 0, np.asarray(gs) - 1)
    kind = rng.random(len(v))
    ob = np.where((kind < 0.12)[:, None], np.minimum(v, np.asarray(gs) - 1), ob).astype(np.uint64)
    code = ((ob[:, 0] + 1) << 20) | (ob[:, 1] << 10) | ob[:, 2]
    rec = np.where((kind >= 0.75) & (kind < 0.9), 0, np.where(kind >= 0.95, 1, code)).astype(np.uint64)
    rec = np.where((kind >= 0.9) & (kind < 0.95), rec | 0x80000000, rec)
    rec = np.where(v[:, 2] >= gz, 0, rec)                                   # padding words stay 0
    return rec.astype(np.uint32)


def distance_array(rec, gs):
    gx, gy, gz = gs
    R = rec.reshape(gx, gy, (gz + 3) & ~3)[:, :, :gz]
    D = np.empty(gs)
    for x in range(gx):
        for y in range(gy):
            for z in range(gz):
                D[x, y, z] = segref.record_distance(int(R[x, y, z]), x, y, z, RES)
    return D


def brute_force(cluster, pos, R, max_range, tan, clearance, sizes, members, D, lo, hi, unk):
    """One pair at a time in Python floats (IEEE doubles, one rounding per operation) with segref.check as the line of sight."""
    moff = np.concatenate([[0], np.cumsum(sizes)])
    n = len(pos)
    st = np.zeros(n, np.int32)
    sc = np.zeros((n, len(R)), np.int32)
    walked = visible = 0
    for i in range(n):
        p = [float(x) for x in pos[i]]
        if any(math.isnan(x) for x in p) or not segref.in_map(p, lo, hi):
            st[i] = 2
            continue
        v = [math.floor((p[k] - ORIGIN[k]) / RES) for k in range(3)]
        if not all(0 <= v[k] < D.shape[k] for k in range(3)) or D[tuple(v)] == -10000 or D[tuple(v)] <= clearance:
            st[i] = 1
            continue
        k = cluster[i]
        for m in members[moff[k]:moff[k + 1]]:
            c = [(float(m[a]) + 0.5) * RES + ORIGIN[a] for a in range(3)]
            d = [c[a] - p[a] for a in range(3)]
            if not (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= max_range * max_range:
                continue
            bits = []
            for Rj in R:
                s = [(Rj[r][0] * d[0] + Rj[r][1] * d[1]) + Rj[r][2] * d[2] for r in range(3)]
                bits.append(s[0] > 0 and abs(s[1]) <= tan[0] * s[0] and abs(s[2]) <= tan[1] * s[0])
            if not any(bits):
                continue
            walked += 1
            if segref.check(p + c, ORIGIN, RES, lo, hi, D, 0.0, unk)[0] != 0:
                continue
            visible += 1
            sc[i] += np.array(bits, np.int32)
    return st, sc, dict(candidates_scored=int(np.sum(st == 0)), pairs_walked=walked, pairs_visible=visible)


@pytest.mark.parametrize("gs", [(14, 12, 9), (10, 13, 30)])                 # Gz = 30: padded z pitch
def test_score_equals_brute_force_and_header(exe, gs):
    rng = np.random.default_rng(sum(gs))
    rec = records(gs, rng)
    D = distance_array(rec, gs)
    size = np.asarray(gs) * RES
    lo, hi = np.asarray(ORIGIN), np.asarray(ORIGIN) + size
    K = 6
    sizes = rng.integers(1, 70, K)
    sizes[2] = 1
    members = np.concatenate([rng.integers(0, gs, (int(s), 3)) for s in sizes]).astype(np.int32)
    n = 90
    cluster = rng.integers(0, K, n)
    pos = rng.uniform(lo, hi, (n, 3))
    pos[:4] = [lo - 0.01, hi + 0.01, [np.nan, 0.0, 0.0], hi]                 # outside, NaN, on the upper faces (status 1)
    stand = np.argwhere((D > 0.3) & (D < 10000))[:20]
    pos[4:4 + len(stand)] = (stand + 0.5) * RES + lo                        # observed voxels beyond the largest clearance
    R = np.stack([viewref.yaw(a) for a in (0.0, 1.0, 2.5, 4.0)] + [viewref.yaw_pitch(0.5, 0.6), np.eye(3)])
    seen = set()
    for clearance in (0.0, 0.15):
        for unk in (False, True):
            for max_range, tan in ((1.2, (1.0, 0.6)), (4.0, (0.4, 0.3))):
                los = lambda ab: [segref.check(s, ORIGIN, RES, lo, hi, D, 0.0, unk)[0] for s in ab]
                want = viewref.score(cluster, pos, R, max_range, tan, clearance, sizes, members, D, ORIGIN, RES, lo, hi, los)
                bf = brute_force(cluster, pos, R, max_range, tan, clearance, sizes, members, D, lo, hi, unk)
                assert np.array_equal(want[0], bf[0]) and np.array_equal(want[1], bf[1]) and want[2] == bf[2]
                txt = ["score %d %d %d" % gs, hx(list(ORIGIN) + [RES] + list(lo) + list(hi)), str(len(rec)),
                       " ".join(str(int(c)) for c in rec), "%s %d" % (float(clearance).hex(), int(unk))]
                txt += sensor_lines(R, max_range, tan) + [str(K), " ".join(str(int(s)) for s in sizes)]
                txt += [" ".join(str(int(x)) for x in members.reshape(-1)), str(n)]
                txt += ["%d %s" % (int(c), hx(p)) for c, p in zip(cluster, pos)]
                lines = run(exe, txt)
                got = np.array([[int(x) for x in line.split()] for line in lines[:n]])
                assert np.array_equal(got[:, 0], want[0]) and np.array_equal(got[:, 1:], want[1])
                assert [int(x) for x in lines[n].split()[1:]] == [want[2][k] for k in ("candidates_scored", "pairs_walked", "pairs_visible")]
                seen |= set(int(s) for s in want[0])
                assert want[2]["pairs_visible"] < want[2]["pairs_walked"]             # some lines of sight are blocked
                assert want[1].sum() > 0
    assert seen == {0, 1, 2}
