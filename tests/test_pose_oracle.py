"""CPU: robot-shaped collision checks.  fiesta_b200/csrc/fb_pose.h, compiled with g++ without contraction, accepts exactly the voxels
tests/poseref.py's separating-axis test accepts, bit for bit, on adversarial and random poses; every touched voxel lies in the
candidate range (brute force over a window 3 voxels wider); and fb_pose_check's status, count and first index equal poseref's on
synthetic records, with and without FIESTA_SEGMENT_UNKNOWN_BLOCKS."""
import os
import subprocess

import numpy as np
import pytest

from tests import poseref, segref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.125
ORIGIN = (-2.0, -3.0, -1.0)              # binary-exact voxel centres
DRONE, CAR = (0.25, 0.25, 0.1), (0.55, 0.225, 0.1875)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("pose") / "pose_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "cpp", "pose_test.cpp"), "-o", out])
    return out


def hx(vals):
    return " ".join(float(v).hex() for v in vals)


def run(exe, txt):
    p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout.splitlines()


def bounds(gs):
    lo = np.asarray(ORIGIN)
    return lo, lo + np.asarray(gs) * RES


def touch_lines(exe, P, h, gs, margin=3):
    lo, hi = bounds(gs)
    txt = ["touch", hx([RES] + list(ORIGIN) + list(lo) + list(hi) + list(h)), str(margin), str(len(P))] + [hx(p) for p in P]
    return run(exe, txt)


def assert_touch_matches(exe, P, h, gs):
    """The header's touched set and candidate range equal poseref's; nothing outside the candidate range is touched."""
    lo, hi = bounds(gs)
    lines = touch_lines(exe, P, h, gs)
    assert len(lines) == len(P)
    n_valid = n_touched = 0
    for pose, line in zip(P, lines):
        f = [int(x) for x in line.split()]
        if not poseref.valid(pose, lo, hi):
            assert f == [0], pose
            continue
        n_valid += 1
        wlo, hit, (clo, chi) = poseref.touched(pose, h, ORIGIN, RES, margin=3)
        assert f[0] == 1 and f[1:4] == list(clo) and f[4:7] == list(chi), pose
        got = np.array(f[8:], np.int64).reshape(-1, 3)
        want = np.argwhere(hit) + wlo
        assert f[7] == len(want) and np.array_equal(got, want), pose
        assert np.all((want >= clo) & (want <= chi)), pose                  # the candidate range is a superset
        n_touched += len(want) > 0
    return n_valid, n_touched


def test_touch_adversarial(exe):
    rng = np.random.default_rng(1)
    gs = (40, 36, 24)
    for h in (DRONE, CAR, (0.25, 0.0, 0.125), (0.0, 0.375, 0.0), (0.0, 0.0, 0.0), (0.5, 0.5, 0.5)):
        P = poseref.adversarial(rng, ORIGIN, RES, gs, h)
        n_valid, n_touched = assert_touch_matches(exe, P, h, gs)
        assert n_valid > 40 and n_touched == n_valid                       # a valid pose always touches the voxels at its centre


def test_touch_faces_on_voxel_faces():
    """R = I, a centre on a voxel corner and h a whole number of voxels: the closed box touches exactly the voxels its faces bound
    plus the ring whose faces it touches."""
    c = np.asarray(ORIGIN) + np.array([20, 18, 12]) * RES
    for nh in ((2, 1, 3), (1, 1, 1), (0, 2, 0)):
        h = tuple(k * RES for k in nh)
        wlo, hit, _ = poseref.touched(poseref.poses(c, np.eye(3))[0], h, ORIGIN, RES)
        got = np.argwhere(hit) + wlo
        want_lo, want_hi = np.array([20, 18, 12]) - np.array(nh) - 1, np.array([20, 18, 12]) + np.array(nh)
        assert np.array_equal(got.min(0), want_lo) and np.array_equal(got.max(0), want_hi)
        assert len(got) == int(np.prod(want_hi - want_lo + 1))
        # 2^-30 m inside on every axis drops the touching ring (one ulp would round away in T_L)
        hin = tuple(x - 2.0 ** -30 if x > 0 else x for x in h)
        wlo, hit, _ = poseref.touched(poseref.poses(c, np.eye(3))[0], hin, ORIGIN, RES)
        assert len(np.argwhere(hit)) < len(got) or min(nh) == 0


def test_touch_random_and_r_limits(exe):
    rng = np.random.default_rng(2)
    gs = (40, 36, 24)
    lo, hi = bounds(gs)
    n = 150
    p = rng.uniform(lo - 0.2, hi + 0.2, (n, 3))
    R = poseref.random_rotations(rng, n)
    R[:20] *= rng.uniform(0.999, poseref.R_MAX, (20, 1, 1))                 # not orthonormal: used as given
    R[20:30] = rng.normal(0, 0.5, (10, 3, 3)).clip(-1, 1)
    P = poseref.poses(p, R)
    for h in (DRONE, CAR, (0.0, 0.3, 0.0)):
        n_valid, _ = assert_touch_matches(exe, P, h, gs)
        assert 50 < n_valid < n
    base = poseref.poses(lo + np.array([2.0, 2.0, 1.0]), np.eye(3))[0]
    at, above = base.copy(), base.copy()
    at[3] = -poseref.R_MAX
    above[7] = np.nextafter(poseref.R_MAX, 2.0)
    assert poseref.valid(at, lo, hi) and not poseref.valid(above, lo, hi)
    assert [line.split()[0] for line in touch_lines(exe, [at, above], DRONE, gs)] == ["1", "0"]


def test_touch_largest_body(exe):
    """h0 + h1 + h2 == 256 voxels, the largest body the library accepts."""
    gs = (40, 36, 24)
    lo, _ = bounds(gs)
    c = lo + np.array([2.5, 2.25, 1.5])
    P = poseref.poses(np.stack([c] * 3), np.stack([np.eye(3), poseref.rot_z(np.pi / 4), poseref.rot_z(0.3)]))
    for h in ((256 * RES, 0.0, 0.0), (128 * RES, 0.0, 128 * RES)):
        assert (h[0] + h[1]) + h[2] == 256 * RES
        n_valid, n_touched = assert_touch_matches(exe, P, h, gs)
        assert n_valid == n_touched == 3


def records(gs, rng):
    """Packed records in device layout (z pitch rounded up to 4): never observed, unreached, local-map reset (bit 31), obstacles
    at the voxel itself and nearby."""
    gx, gy, gz = gs
    pz = (gz + 3) & ~3
    v = np.stack(np.meshgrid(np.arange(gx), np.arange(gy), np.arange(pz), indexing="ij"), -1).reshape(-1, 3)
    ob = np.clip(v + rng.integers(-3, 4, v.shape), 0, np.asarray(gs) - 1)
    kind = rng.random(len(v))
    ob = np.where((kind < 0.01)[:, None], np.minimum(v, np.asarray(gs) - 1), ob).astype(np.uint64)
    code = ((ob[:, 0] + 1) << 20) | (ob[:, 1] << 10) | ob[:, 2]
    rec = np.where((kind >= 0.85) & (kind < 0.9), 0, np.where(kind >= 0.95, 1, code)).astype(np.uint64)
    rec = np.where((kind >= 0.9) & (kind < 0.95), rec | 0x80000000, rec)
    rec = np.where(v[:, 2] >= gz, 0, rec)
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


@pytest.mark.parametrize("gs", [(24, 20, 16), (18, 22, 13)])                 # Gz = 13: padded z pitch
def test_check_equals_poseref(exe, gs):
    rng = np.random.default_rng(sum(gs))
    rec = records(gs, rng)
    D = distance_array(rec, gs)
    lo, hi = bounds(gs)
    settings = [(0.0, False), (0.0, True), (0.2, False), (0.4, True)]
    seen = set()
    for h in (DRONE, CAR, (0.0, 0.0, 0.0), (0.3, 0.0, 0.0), (128 * RES, 0.0, 128 * RES)):
        n = 30
        p = rng.uniform(lo, hi, (n, 3))
        P = np.concatenate([poseref.poses(p, poseref.random_rotations(rng, n)), poseref.adversarial(rng, ORIGIN, RES, gs, h)])
        if sum(h) > 1:
            P = P[::6]                                                      # the largest body: ~10^5 window voxels per pose
        want = poseref.check_all(P, h, ORIGIN, RES, lo, hi, D, settings)
        for (r, unk) in settings:
            txt = ["check %d %d %d" % gs, hx(list(ORIGIN) + [RES] + list(lo) + list(hi)), str(len(rec)),
                   " ".join(str(int(c)) for c in rec), hx(h), "%s %d" % (float(r).hex(), int(unk)), str(len(P))] + [hx(q) for q in P]
            got = np.array([[int(x) for x in line.split()] for line in run(exe, txt)])
            w = want[(r, unk)]
            assert np.array_equal(got[:, 0], w[0]) and np.array_equal(got[:, 1], w[1]) and np.array_equal(got[:, 2], w[2]), (h, r, unk)
            seen |= set(int(s) for s in w[0])
    assert seen == {0, 1, 2, 3}
