"""GPU: safe flight corridors (fiesta_inflate_boxes / fiesta_corridors) against tests/corridorref.py on export_distance() of the same
map -- every array and statistic with np.array_equal -- on ray-cast maps in both modes with paths from a cost-to-go field over the
same box, clearance and flags (none of which may be blocked), cross-checked with the segment query; on crafted maps (a 1-voxel
corridor, seeds on the limit box's faces, an unknown voxel beside a seed, a path through an obstacle, a voxel outside the box, empty,
1-voxel and repeated paths, open space where max_steps binds); after a map update that follows the nav compute; and on thousands of
paths, random seeds, determinism, permutation, isolation and every invalid and limit path."""
import ctypes as C

import numpy as np
import pytest

from tests import corridorref, scenes
from tests.test_gpu_nav import ORIGIN, RES, SIZES, boxes, raycast_map
from tests.test_gpu_viewpoints import block, crafted_map

pytestmark = pytest.mark.gpu

MS = (40, 40, 20)


def as_list(paths):
    _, ln, _, vox = paths
    return [vox[i, :int(ln[i])] for i in range(len(ln))]


def check(m, paths, box, ms, r, unk):
    """Corridors on the device == corridorref on export_distance(); returns the result."""
    got = m.Corridors(paths, box[0], box[1], ms, r, unk)
    L = corridorref.Limit(m.export_distance(), m.grid_size, box, r, unk)
    want = corridorref.corridors(L, as_list(paths) if isinstance(paths, tuple) else paths, ms)
    for k in range(3):
        assert np.array_equal(got[k], want[k]), (k, int(np.sum(got[k] != want[k])))
    for p, (a, b) in enumerate(zip(got[3], want[3])):
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), p
    assert {k: got[4][k] for k in want[4]} == want[4], (got[4], want[4])
    return got


def check_inflate(m, lo, hi, box, ms, r, unk):
    got = m.InflateBoxes(lo, hi, box[0], box[1], ms, r, unk)
    L = corridorref.Limit(m.export_distance(), m.grid_size, box, r, unk)
    want = corridorref.inflate_boxes(L, lo, hi, ms)
    for k in range(3):
        assert np.array_equal(got[k], want[k]), k
    assert {k: got[3][k] for k in want[3]} == want[3], (got[3], want[3])
    return got


def centre(m, v):
    return np.asarray(m.origin) + (np.asarray(v, np.float64) + 0.5) * m.resolution


def segments_clear(m, res, paths, r, unk, rng, pairs=4):
    """Random pairs of voxel centres inside each box, and the polyline through one shared voxel per junction, are clear."""
    status, nb, _, bx, _ = res
    ab = []
    for p, P in enumerate(paths):
        lo, hi, first = bx[p]
        for k in range(nb[p]):
            for _ in range(pairs):
                ab.append(np.concatenate([centre(m, rng.integers(lo[k], hi[k] + 1)), centre(m, rng.integers(lo[k], hi[k] + 1))]))
        if status[p] == 0 and nb[p]:
            pts = [P[0]] + [P[j - 1] for j in first[1:]] + [P[-1]]
            ab += [np.concatenate([centre(m, a), centre(m, b)]) for a, b in zip(pts[:-1], pts[1:])]
    if ab:
        assert np.all(m.CheckSegments(np.array(ab), r, unk)[0] == 0)
    return len(ab)


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_nav_paths_on_raycast_maps(kind, mode, size):
    m, _ = raycast_map(mode, kind, SIZES[size])
    m.origin = ORIGIN
    nav = m.NavField()
    rng = np.random.default_rng(7)
    boxes_seen, segs = 0, 0
    for box in boxes(m.grid_size)[:2]:                                     # the whole grid and a local box
        lo, hi = np.asarray(box[0]), np.asarray(box[1])
        for r, unk in ((RES, False), (RES, True), (2.5 * RES, False)):
            L = corridorref.Limit(m.export_distance(), m.grid_size, box, r, unk)
            free = np.argwhere(L.T) + lo
            goal = centre(m, free[rng.integers(len(free))])[None]
            nav.compute(box[0], box[1], goal, r, unknown_blocks=unk)
            starts = centre(m, free[rng.integers(len(free), size=60)])
            paths = nav.paths(starts, 400)
            assert np.sum(paths[0] == 0) > 10
            for ms in (MS, (3, 0, 5)):
                res = check(m, paths, box, ms, r, unk)
                assert not np.any(res[0] == 1)                            # nav paths are never blocked
                assert np.all(res[0] == 0)
                boxes_seen += int(res[1].sum())
            segs += segments_clear(m, res, as_list(paths), r, unk, rng)
            check(m, [P[::-1] for P in as_list(paths)], box, MS, r, unk)  # reversed: start to goal
    assert boxes_seen > 100 and segs > 100
    nav.close()


def crafted():
    """24 x 24 x 12, all observed free except: a wall x = 12 with a one-voxel hole at (12, 12, 6), and (4, 4, 7) never observed."""
    gs = (24, 24, 12)
    wall = [v for v in map(tuple, block((12, 0, 0), (12, 23, 11))) if v != (12, 12, 6)]
    free = [v for v in map(tuple, block((0, 0, 0), (23, 23, 11))) if v not in set(wall) and v != (4, 4, 7)]
    m, mirror = crafted_map(gs, free, wall)
    mirror.close()
    m.origin = m.origin_m
    return m


def test_crafted_cases():
    m = crafted()
    full = ((0, 0, 0), (23, 23, 11))
    line = np.array([(x, 12, 6) for x in range(8, 17)])
    # a 1-voxel corridor through the hole: the box across the wall is the line itself
    st, nb, bl, bx, _ = check(m, [line], full, MS, 0.0, False)
    assert st[0] == 0
    lo, hi, _ = bx[0]
    through = [k for k in range(nb[0]) if lo[k][0] <= 12 <= hi[k][0]]
    assert through and all(lo[k][1] == hi[k][1] == 12 and lo[k][2] == hi[k][2] == 6 for k in through)
    # a user path through the wall: status 1 at the wall voxel, the boxes before it kept
    wallpath = np.array([(x, 5, 6) for x in range(6, 16)])
    st, nb, bl, bx, _ = check(m, [wallpath], full, MS, 0.0, False)
    assert st[0] == 1 and bl[0] == 6 and nb[0] >= 1
    # a voxel outside the limit box: status 2, no boxes
    small = ((0, 0, 0), (10, 23, 11))
    st, nb, bl, _, _ = check(m, [np.array([(2, 2, 2), (11, 2, 2)])], small, MS, 0.0, False)
    assert st[0] == 2 and nb[0] == 0 and bl[0] == -1
    # empty, 1-voxel and repeated paths
    st, nb, bl, bx, _ = check(m, [np.zeros((0, 3), np.int32), [(3, 3, 3)], [(3, 3, 3)] * 5 + [(4, 3, 3)] * 3], small, MS, 0.0, False)
    assert st.tolist() == [0, 0, 0] and nb.tolist() == [0, 1, 1]
    # an unknown voxel above a seed: blocks the +z face only with the flag
    for unk, top in ((False, 8), (True, 6)):
        s, lo, hi, _ = check_inflate(m, [(4, 4, 6)], [(4, 4, 6)], full, (0, 0, 2), 0.0, unk)
        assert s[0] == 0 and hi[0][2] == top
    s, _, _, _ = check_inflate(m, [(4, 4, 7)], [(4, 4, 7)], full, MS, 0.0, True)
    assert s[0] == 1
    # seeds on the limit box's faces and corners, and open space where max_steps binds
    lim = ((2, 3, 1), (9, 20, 10))
    seeds = [(2, 3, 1), (9, 20, 10), (2, 10, 5), (9, 10, 5), (5, 3, 5), (5, 20, 5), (5, 10, 1), (5, 10, 10), (5, 10, 5)]
    s, lo, hi, _ = check_inflate(m, seeds, seeds, lim, (2, 1, 0), 0.0, False)
    assert np.all(s == 0) and np.all(lo >= lim[0]) and np.all(hi <= lim[1])
    assert (hi - lo)[0].tolist() == [2, 1, 0] and (hi - lo)[8].tolist() == [4, 2, 0]
    s, lo, hi, _ = check_inflate(m, seeds, seeds, lim, (1000, 1000, 1000), 0.3, False)
    assert np.all(lo >= lim[0]) and np.all(hi <= lim[1]) and np.all(hi[:, 0] <= 9)


def test_map_updated_after_the_nav_compute():
    m, _ = raycast_map("exact", "lidar", SIZES["gz32"], frames=2)
    m.origin = ORIGIN
    box = boxes(m.grid_size)[1]
    nav = m.NavField()
    L = corridorref.Limit(m.export_distance(), m.grid_size, box, RES, True)
    free = np.argwhere(L.T) + np.asarray(box[0])
    rng = np.random.default_rng(11)
    nav.compute(box[0], box[1], centre(m, free[rng.integers(len(free))])[None], RES, unknown_blocks=True)
    paths = nav.paths(centre(m, free[rng.integers(len(free), size=200)]), 400)
    before = check(m, paths, box, MS, RES, True)
    assert np.all(before[0] == 0)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=8, edge=(0.3, 0.8))
    pts, T = scenes.lidar_frame(sc, np.array([0.5, 0.4, 0.0]), 1.1, beams=16, azimuths=360)
    m.RaycastFrame(pts, T, 0.3, 4.0)
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    after = check(m, paths, box, MS, RES, True)                           # old paths, new records
    assert not all(np.array_equal(a, b) for a, b in zip(before[:3], after[:3])) or before[4] != after[4]
    nav.close()


def test_many_paths_seeds_determinism_and_isolation():
    m, _ = raycast_map("fast", "lidar", SIZES["gz30"], frames=3)
    m.origin = ORIGIN
    gs = m.grid_size
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    rng = np.random.default_rng(12)
    L = corridorref.Limit(m.export_distance(), gs, box, RES, False)
    free = np.argwhere(L.T)
    paths = []
    for i in range(3000):                                                  # mixed lengths: 0 .. 300 voxels, some off the box
        n = int(rng.choice([0, 1, 2, 5, 30, 300], p=[0.05, 0.1, 0.15, 0.3, 0.3, 0.1]))
        p = np.cumsum(rng.integers(-1, 2, (n, 3)), axis=0) + free[rng.integers(len(free))]
        paths.append(np.clip(p, -1, np.asarray(gs)) if i % 10 == 0 else np.clip(p, 0, np.asarray(gs) - 1))
    D0, O0, C0 = m.export_distance(), m.export_occupancy(), m.export_closest_obstacle()
    a = check(m, paths, box, MS, RES, False)
    assert set(a[0].tolist()) == {0, 1, 2} and a[4]["boxes"] > 2000
    b = m.Corridors(paths, box[0], box[1], MS, RES, False)
    assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3]))         # determinism
    assert all(np.array_equal(x, y) for P, Q in zip(a[3], b[3]) for x, y in zip(P, Q))
    perm = rng.permutation(len(paths))
    c = m.Corridors([paths[i] for i in perm], box[0], box[1], MS, RES, False)
    assert all(np.array_equal(x[perm], y) for x, y in zip(a[:3], c[:3]))
    assert all(np.array_equal(x, y) for i, Q in zip(perm, c[3]) for x, y in zip(a[3][i], Q))
    assert {k: c[4][k] for k in ("boxes", "layers_tested", "layers_grown")} == {k: a[4][k] for k in ("boxes", "layers_tested", "layers_grown")}
    # independent seeds: random, inverted, outside, blocked
    lo = rng.integers(-2, np.asarray(gs) + 2, (4000, 3))
    hi = lo + rng.integers(-2, 4, (4000, 3))
    f = free[rng.integers(len(free), size=2000)]
    lo, hi = np.concatenate([lo, f]), np.concatenate([hi, f])
    s = check_inflate(m, lo, hi, box, MS, RES, False)
    assert set(s[0].tolist()) == {0, 1, 2}
    s2 = check_inflate(m, lo, hi, boxes(gs)[1], (5, 2, 3), 2.5 * RES, True)
    assert set(s2[0].tolist()) == {0, 1, 2}
    # isolation: the map is unchanged
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert np.array_equal(m.export_closest_obstacle(), C0)


def test_invalid_and_limit_arguments_write_nothing():
    import fiesta_b200
    assert C.sizeof(fiesta_b200.CorridorStats) == 4 * 8 + 2 * 4
    m, _ = raycast_map("fast", "lidar", SIZES["gz30"], frames=1)
    Lb = m._L
    gs = m.grid_size
    n = 4
    I = lambda *v: np.array(v, np.int32)
    seeds = np.tile(I(10, 10, 5), (n, 1))
    out = [np.full(n, -7, np.int32), np.full((n, 3), -7, np.int32), np.full((n, 3), -7, np.int32)]
    ptr = lambda a: None if a is None else a.ctypes
    box_hi = I(*[g - 1 for g in gs])

    def inflate(lo=I(0, 0, 0), hi=box_hi, s_lo=seeds, s_hi=seeds, nn=n, ms=I(4, 4, 4), r=RES, flags=0, o=out, h=None):
        return Lb.fiesta_inflate_boxes(m._h if h is None else h, ptr(lo), ptr(hi), ptr(s_lo), ptr(s_hi), C.c_int64(nn), ptr(ms), C.c_double(r),
                                       flags, *(ptr(x) for x in o), None)

    bad = [inflate(lo=I(-1, 0, 0)), inflate(hi=I(gs[0], 3, 3)), inflate(lo=I(5, 0, 0), hi=I(4, 9, 9)), inflate(lo=None), inflate(hi=None),
           inflate(ms=I(1, -1, 1)), inflate(ms=None), inflate(r=np.nan), inflate(r=-0.1), inflate(r=10000.0), inflate(flags=2),
           inflate(nn=-1), inflate(s_lo=None), inflate(s_hi=None), inflate(o=[None, out[1], out[2]]), inflate(o=[out[0], None, out[2]]),
           inflate(o=[out[0], out[1], None]), inflate(h=C.c_void_p(0))]
    assert bad == [1] * len(bad), bad                                        # FIESTA_ERR_INVALID
    assert inflate(nn=0x7fffffff) == 4                                       # FIESTA_ERR_LIMIT
    assert all(np.all(x == -7) for x in out)

    P = np.tile(I(10, 10, 5), (6, 1))
    cout = [np.full(3, -7, np.int32) for _ in range(3)] + [np.full((6, 3), -7, np.int32), np.full((6, 3), -7, np.int32), np.full(6, -7, np.int32)]

    def corr(off=np.array([0, 2, 2, 6], np.int64), np_=3, vox=P, ms=I(4, 4, 4), r=RES, flags=0, lo=I(0, 0, 0), o=cout):
        return Lb.fiesta_corridors(m._h, ptr(lo), ptr(box_hi), ptr(vox), ptr(off), C.c_int64(np_), ptr(ms), C.c_double(r), flags,
                                   *(ptr(x) for x in o), None)

    bad = [corr(off=np.array([1, 2, 2, 6], np.int64)), corr(off=np.array([0, 3, 2, 6], np.int64)), corr(off=None), corr(np_=-1),
           corr(vox=None), corr(ms=I(0, 0, -3)), corr(r=np.nan), corr(flags=4), corr(lo=I(0, 0, gs[2])),
           corr(o=[None] + cout[1:]), corr(o=cout[:3] + [None] + cout[4:]), corr(o=cout[:5] + [None])]
    assert bad == [1] * len(bad), bad
    assert corr(off=np.array([0, 2, 2, 0x7fffffff], np.int64)) == 4
    assert all(np.all(x == -7) for x in cout)
    assert corr(off=None, np_=0, vox=None, o=[None] * 6) == 0               # no paths: nothing to do
    assert corr(off=np.array([0, 0, 0, 0], np.int64), vox=None, o=cout[:3] + [None] * 3) == 0   # only empty paths
    assert cout[0].tolist() == [0, 0, 0] and cout[1].tolist() == [0, 0, 0] and cout[2].tolist() == [-1, -1, -1]
    with pytest.raises(fiesta_b200.FiestaError):
        m.InflateBoxes([(0, 0, 0)], [(0, 0, 0)], (0, 0, 0), gs, MS, RES)
    assert corr() == 0 and set(cout[0].tolist()) <= {0, 1}                    # still usable
