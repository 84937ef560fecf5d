"""CPU: the signed field's definition.  tests/signedref.py (scipy's exact EDT indices turned into integer squared distances) equals
the O(n^2) brute-force minimum on random masks of small boxes and on the corner cases: no obstacle, all obstacle (-inf), a single
free voxel, a solid cube with a one-voxel tunnel, boxes one voxel thick on each axis.  The header fiesta_b200/csrc/fb_signed.h,
compiled with g++, classifies records and computes the first pass's 1-D distance and the envelope of one line exactly as numpy does,
on random lines up to 2046 voxels long and on lines of all obstacles and all free voxels."""
import os
import subprocess

import numpy as np
import pytest

from tests import signedref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = signedref.NONE


def check_model(obst, res=0.1):
    q = signedref.depth_sq(obst)
    assert np.array_equal(q, signedref.brute_q(obst))
    S = signedref.signed_values(q, np.full(obst.shape, 0.3), res)
    assert np.all(S[~obst] == 0.3)
    return q, S


@pytest.mark.parametrize("shape", [(5, 6, 7), (1, 9, 8), (9, 1, 8), (9, 8, 1), (1, 1, 12), (12, 1, 1), (1, 12, 1), (3, 3, 3)])
@pytest.mark.parametrize("density", [0.3, 0.7, 0.95])
def test_model_equals_brute_force_on_random_masks(shape, density):
    rng = np.random.default_rng(hash((shape, density)) % 2**32)
    for _ in range(4):
        check_model(rng.random(shape) < density)


def test_no_obstacle():
    q, S = check_model(np.zeros((4, 5, 6), bool))
    assert np.all(q == 0)
    assert signedref.stats(q) == dict(box_voxels=120, obstacles=0, interior=0, max_depth_sq=0)


def test_all_obstacle_is_minus_infinity():
    q, S = check_model(np.ones((4, 3, 2), bool))
    assert np.all(q == NONE) and np.all(S == -np.inf)
    assert signedref.stats(q) == dict(box_voxels=24, obstacles=24, interior=24, max_depth_sq=-1)


def test_single_free_voxel():
    obst = np.ones((6, 5, 7), bool)
    obst[1, 4, 2] = False
    q, S = check_model(obst)
    g = np.indices(obst.shape)
    assert np.array_equal(q, (g[0] - 1) ** 2 + (g[1] - 4) ** 2 + (g[2] - 2) ** 2)
    st = signedref.stats(q)
    assert st["max_depth_sq"] == 4 ** 2 + 4 ** 2 + 4 ** 2 and st["obstacles"] == obst.size - 1


def test_solid_cube_with_tunnel():
    obst = np.zeros((15, 15, 15), bool)
    obst[2:13, 2:13, 2:13] = True
    obst[7, 7, :] = False                                                  # a one-voxel tunnel through the cube along z
    q, S = check_model(obst)
    assert q[7, 6, 7] == 1 and q[7, 8, 7] == 1                            # beside the tunnel: surface
    assert q[4, 4, 7] == 3 ** 2                                           # 3 voxels from the outside, 3 + 3 from the tunnel
    assert q[6, 6, 7] == 2 and q[7, 5, 7] == 4                            # diagonal and straight from the tunnel
    assert S[7, 6, 7] == 0.0 and not np.signbit(S[7, 6, 7])               # q == 1 is +0.0
    assert np.all(S[obst & (q > 1)] < 0)


def test_signed_value_formula():
    q = np.array([0, 1, 2, 4, 9, 6275083, NONE], np.int64)
    S = signedref.signed_values(q, np.array([-10000.0, 0, 0, 0, 0, 0, 0]), 0.05)
    assert S[0] == 10000.0                                                 # never observed reads +10000
    assert S[1] == 0.0 and not np.signbit(S[1])
    assert S[2] == (1.0 - np.sqrt(2.0)) * 0.05 and S[3] == -0.05 and S[4] == (1.0 - 3.0) * 0.05
    assert S[6] == -np.inf


# ---- the header, compiled with g++
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("signed") / "signed_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "cpp", "signed_test.cpp"), "-o", out])
    return out


def run(exe, text):
    out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
    return out


def pack(x, y, z):
    return ((x + 1) << 20) | (y << 10) | z


def record_distance(c, x, y, z, res=0.1):
    """fb_record_distance restated: what fiesta_export_distance writes for record c at voxel (x, y, z)."""
    if c & 0x7fffffff == 0:
        return -10000.0
    if c & 0x7fffffff == 1 or c >> 31:
        return 10000.0
    c &= 0x7fffffff
    ox, oy, oz = (c >> 20) - 1, (c >> 10) & 1023, c & 1023
    return float(np.sqrt(float((ox - x) ** 2 + (oy - y) ** 2) + float((oz - z) ** 2)) * res)


def random_records(rng, x, y, m, p_obst):
    """Records of a z-line: obstacles (own coordinates), reset obstacles (bit 31), other voxels' obstacles, +10000, unknown."""
    recs = []
    for z in range(m):
        r = rng.random()
        if r < p_obst:
            recs.append(pack(x, y, z))
        else:
            k = rng.integers(0, 4)
            recs.append([pack(x, y, z) | 0x80000000, pack(x, y, (z + 1 + int(rng.integers(0, 5))) % 1024), 1, 0][k])
    return recs


def line_model(obst):
    m = len(obst)
    free = np.nonzero(~obst)[0]
    if len(free) == 0:
        return np.full(m, NONE)
    return np.min((np.arange(m)[:, None] - free[None, :]) ** 2, axis=1)


def test_header_classification_and_first_pass(exe):
    rng = np.random.default_rng(11)
    cases = []
    for m in [1, 2, 31, 32, 33, 64, 95, 100, 1000, 1024]:
        for p in (0.0, 0.5, 0.9, 0.99, 1.0):
            x, y = int(rng.integers(0, 2046)), int(rng.integers(0, 1024))
            cases.append((x, y, random_records(rng, x, y, m, p)))
    text = "".join("line %d %d %d %s\n" % (x, y, len(r), " ".join(str(c) for c in r)) for x, y, r in cases)
    out = run(exe, text)
    pos = 0
    for x, y, r in cases:
        obst = np.array([record_distance(c, x, y, z) == 0.0 for z, c in enumerate(r)])
        got = np.array([int(v) for v in out[pos:pos + len(r)]])
        pos += len(r)
        assert np.array_equal(got, line_model(obst)), (x, y, len(r))


def envelope_model(F):
    F = np.asarray(F, np.int64)
    ok = np.nonzero(F != NONE)[0]
    m = len(F)
    if len(ok) == 0:
        return np.full(m, NONE)
    return np.min((np.arange(m)[:, None] - ok[None, :]) ** 2 + F[ok][None, :], axis=1)


def test_header_envelope(exe):
    rng = np.random.default_rng(12)
    lines = [np.full(7, NONE), np.zeros(9, np.int64), np.full(2046, NONE), np.zeros(2046, np.int64), [NONE], [0], [5]]
    for m in [2, 3, 17, 100, 1024, 2046]:
        for p_none in (0.0, 0.5, 0.99):
            for hi in (4, 1023 ** 2 + 1, 2 * 1023 ** 2 + 1):
                F = rng.integers(0, hi, m)
                F[rng.random(m) < p_none] = NONE
                lines.append(F)
    lines.append(np.array([2 * 1023 ** 2] + [NONE] * 2044 + [2 * 1023 ** 2]))    # the largest values at the longest distance
    text = "".join("env %d %s\n" % (len(F), " ".join(str(int(v)) for v in F)) for F in lines)
    out = run(exe, text)
    pos = 0
    for F in lines:
        want = envelope_model(F)
        got = np.array([int(v) for v in out[pos:pos + len(F)]])
        acc = out[pos + len(F)].split()
        pos += len(F) + 1
        assert np.array_equal(got, want), len(F)
        fin = want[want != NONE]
        assert acc == ["acc", str(int(np.sum(want > 0))), str(int(np.sum(want > 1))), str(int(fin.max()) if len(fin) and fin.max() > 0 else 0)]
