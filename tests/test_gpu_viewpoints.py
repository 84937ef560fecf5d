"""GPU: viewpoint coverage (fiesta_frontiers_score_viewpoints) against tests/viewref.py, whose line of sight is the sequential host
walk of the pinned mirror (fiesta_host_mirror_check_segments at clearance 0), independent of the scoring kernel -- status, score
and stats with np.array_equal -- on ray-cast maps in both modes (whole grid and a local box), on crafted maps with exact fp64
boundaries (members on the field-of-view planes and at max_range, a hair beyond, lines of sight through an edge shared by two
diagonal obstacles, unknown voxels on the line of sight), on a cluster of more than 10^5 members with thousands of tiny clusters
beside it, and after a map update that follows the frontier compute.  Also: determinism, permuted candidates, score <= size,
status-0 candidates traversable in a cost-to-go field, isolation from the map and the frontier result, and every invalid path."""
import ctypes as C

import numpy as np
import pytest

from tests import scenes, segref, viewref
from tests.test_gpu_nav import ORIGIN, RES, SIZES, boxes, raycast_map

pytestmark = pytest.mark.gpu

SENSORS = [(4.5, (1.0, np.tan(np.pi / 6))), (1.5, (0.4, 0.3))]            # 90 x 60 degrees at 4.5 m; a narrow, short one
ORIENTS = np.stack(list(viewref.yaws(8)) + [viewref.yaw_pitch(0.7, 0.5), np.eye(3)])


def map_box(m):
    """The PosInMap box [origin, origin + size]."""
    o = np.asarray(m.origin_m, np.float64)
    return o, o + np.asarray(m.size_m, np.float64)


def check(m, fr, mirror, cluster, pos, R, sensor, clearance=0.0, unk=False, subset=0):
    """Score on the device and compare everything with viewref; `subset` lines of sight are also checked against segref on
    export_distance().  Returns (status, score, stats)."""
    mirror.refresh()
    max_range, tan = sensor
    st, sc, stats = fr.score_viewpoints(cluster, pos, R, max_range, tan, clearance, unk)
    D = m.export_distance().reshape(m.grid_size)
    lo, hi = map_box(m)
    seen = []

    def los(ab):
        s = mirror.CheckSegments(ab, 0.0, unk)[0]
        seen.append((ab, s))
        return s

    want = viewref.score(cluster, pos, R, max_range, tan, clearance, fr.clusters()["size"], fr.voxels(), D, m.origin_m, m.resolution,
                         lo, hi, los)
    assert np.array_equal(st, want[0]), int(np.sum(st != want[0]))
    assert np.array_equal(sc, want[1]), int(np.sum(sc != want[1]))
    assert {k: stats[k] for k in want[2]} == want[2], (stats, want[2])
    if subset and seen:
        ab, s = seen[0]
        for k in np.random.default_rng(0).choice(len(ab), min(subset, len(ab)), replace=False):
            assert segref.check(ab[k], m.origin_m, m.resolution, lo, hi, D, 0.0, unk)[0] == s[k]
    return st, sc, stats


def candidates(m, fr, rng, n_random=200):
    """Rings around every centroid (radii 0.5 and 1.0 m, 8 angles), random positions in the map, and bad ones: outside, NaN, on
    the upper faces, on unknown, obstacle and near-obstacle voxels."""
    cen = fr.clusters()["centroid"]
    K = len(cen)
    cl, pos = viewref.rings(cen, (0.5, 1.0), 8)
    lo, hi = map_box(m)
    D = m.export_distance().reshape(m.grid_size)
    centre = lambda v: np.asarray(m.origin_m) + (np.asarray(v) + 0.5) * m.resolution
    bad = [lo - 0.01, hi + 0.01, [np.nan, 0.0, 0.0], hi, [lo[0], hi[1], lo[2]]]
    for sel in (D == -10000, D == 0, (D > 0) & (D <= 2.5 * RES)):
        bad += [centre(v) for v in np.argwhere(sel)[:5]]
    extra = np.concatenate([rng.uniform(lo, hi, (n_random, 3)), np.asarray(bad, np.float64)])
    return np.concatenate([cl, rng.integers(0, K, len(extra))]), np.concatenate([pos, extra])


def prepare(m):
    m.origin_m = ORIGIN
    return m, m.HostMirror()


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_raycast_maps(kind, mode, size):
    m, mirror = prepare(raycast_map(mode, kind, SIZES[size])[0])
    fr = m.Frontiers()
    rng = np.random.default_rng(3)
    statuses, walked, visible = set(), 0, 0
    for bi, box in enumerate(boxes(m.grid_size)[:2]):                      # the whole grid and a local box
        fr.compute(box[0], box[1], RES, 3)
        assert fr.stats["kept_clusters"] > 0
        cl, pos = candidates(m, fr, rng)
        for si, sensor in enumerate(SENSORS):
            for unk in (False, True):
                st, sc, stats = check(m, fr, mirror, cl, pos, ORIENTS, sensor, RES, unk, subset=200 if si == 0 else 0)
                statuses |= set(int(s) for s in st)
                walked += stats["pairs_walked"]
                visible += stats["pairs_visible"]
        check(m, fr, mirror, cl, pos, viewref.yaws(32), SENSORS[0], 0.0, False)   # n_orient = 32
        check(m, fr, mirror, cl, pos, ORIENTS[:1], SENSORS[0], 2.5 * RES, True)   # n_orient = 1
    assert statuses == {0, 1, 2}
    assert 0 < visible < walked
    fr.close(); mirror.close()


def crafted_map(gs, free, occupied=()):
    """A map of 0.125 m voxels with a binary-exact origin (every voxel centre and offset below is exact) that has observed only the
    voxels `free` (free) and `occupied`; everything else is unknown."""
    import fiesta_b200
    origin = (-2.0, -2.0, -1.0)
    m = fiesta_b200.ESDFMap(origin, 0.125, tuple(g * 0.125 for g in gs), mode="fast")
    assert m.grid_size == tuple(gs)
    m.size_m, m.origin_m = tuple(g * 0.125 for g in gs), origin
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    free, occ = np.asarray(free, np.int32).reshape(-1, 3), np.asarray(occupied, np.int32).reshape(-1, 3)
    m.SetOccupancyBatchVox(np.concatenate([free, occ]), np.concatenate([np.zeros(len(free), np.uint8), np.ones(len(occ), np.uint8)]))
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    return m, m.HostMirror()


def block(lo, hi):
    return np.stack(np.meshgrid(*[np.arange(a, b + 1) for a, b in zip(lo, hi)], indexing="ij"), -1).reshape(-1, 3)


def test_exact_boundaries_diagonal_obstacles_and_unknown_on_the_line():
    """Observed free space x <= 15 of a 32^3 grid, unknown beyond: the plane x = 15 is one frontier cluster.  A candidate at the
    centre of voxel (7, 16, 16) sees member (15, 16 + a, 16 + b) at d = (1, a/8, b/8), exactly."""
    gs = (32, 32, 32)
    obstacles = [(8, 16, 8), (7, 17, 8)]                                   # share the edge the diagonal line of sight crosses
    hole = (11, 16, 24)                                                    # never observed, on a line of sight
    free = [v for v in map(tuple, block((0, 0, 0), (15, 31, 31))) if v not in obstacles and v != hole]
    m, mirror = crafted_map(gs, free, obstacles)
    fr = m.Frontiers()
    fr.compute((0, 0, 0), (31, 31, 31), 0.0, 1)
    vox, size = fr.voxels(), fr.clusters()["size"]
    plane = int(np.searchsorted(np.cumsum(size), np.argmax(vox[:, 0] == 15), side="right"))
    assert size[plane] == 32 * 32 and len(size) == 2                       # the plane, and the six neighbours of the hole
    centre = lambda v: np.asarray(m.origin_m) + (np.asarray(v, np.float64) + 0.5) * 0.125
    p = centre((7, 16, 16))
    hair = 2.0 ** -30
    cl = np.full(3, plane)
    for unk in (False, True):
        # field of view: |a| <= 6 (tan 0.75) and |b| <= 4 (tan 0.5) counted on the planes; a hair off-centre loses one plane
        st, sc, _ = check(m, fr, mirror, cl, [p, p + [0, hair, 0], p + [0, 0, -hair]], np.eye(3)[None], (10.0, (0.75, 0.5)), 0.0, unk)
        assert np.array_equal(st, [0, 0, 0]) and sc[:, 0].tolist() == [13 * 9, 12 * 9, 13 * 8]
        # range: a^2 + b^2 <= 36 at max_range 1.25 exactly (113 lattice points); a hair further loses the four at radius 6
        st, sc, _ = check(m, fr, mirror, cl[:2], [p, p - [hair, 0, 0]], np.eye(3)[None], (1.25, (10.0, 10.0)), 0.0, unk)
        assert sc[:, 0].tolist() == [113, 109]
    # the diagonal from (7, 16, 8) to (15, 24, 8) crosses the edge between the obstacles (8, 16, 8) and (7, 17, 8): the walk steps
    # through the shared corner and never enters either, so the member is visible
    q = centre((7, 16, 8))
    st, sc, stats = check(m, fr, mirror, cl[:1], [q], viewref.yaw(np.pi / 4)[None], (2.0, (1e-3, 1e-3)), 0.0, False)
    assert st[0] == 0 and sc[0, 0] == 1 and stats["pairs_walked"] == 1
    # the hole on the axis from (7, 16, 24) to (15, 16, 24) blocks only with the unknown flag
    r = centre((7, 16, 24))
    for unk, want in ((False, 1), (True, 0)):
        st, sc, stats = check(m, fr, mirror, cl[:1], [r], np.eye(3)[None], (2.0, (1e-3, 1e-3)), 0.0, unk)
        assert sc[0, 0] == want and stats["pairs_walked"] == 1
    # candidates that cannot stand: an obstacle, the hole, within the clearance, unknown space beyond the plane, the upper faces
    bad = [centre(obstacles[0]), centre(hole), centre((9, 16, 8)), centre((20, 5, 5)), np.asarray(m.origin_m) + np.asarray(m.size_m)]
    st, sc, _ = check(m, fr, mirror, np.full(len(bad), plane), bad, np.eye(3)[None], SENSORS[0], 0.2, False)
    assert st.tolist() == [1, 1, 1, 1, 1] and not sc.any()
    fr.close(); mirror.close()


def test_large_cluster_and_thousands_of_tiny_clusters():
    """A 320 x 320 frontier plane (102 400 members, 3 200 chunks per candidate) scored by many candidates, beside 5 000+ clusters
    of six voxels around single unknown voxels."""
    gs = (20, 320, 320)
    holes = block((2, 0, 0), (8, 319, 319))
    holes = holes[(holes[:, 0] % 6 == 2) & (holes[:, 1] % 6 == 2) & (holes[:, 2] % 6 == 2)]
    V = block((0, 0, 0), (15, 319, 319))
    keep = np.ones(len(V), bool)
    keep[(holes[:, 0] * 320 + holes[:, 1]) * 320 + holes[:, 2]] = False
    m, mirror = crafted_map(gs, V[keep])
    fr = m.Frontiers()
    fr.compute((0, 0, 0), tuple(g - 1 for g in gs), 0.0, 1)
    cls = fr.clusters()
    size = cls["size"]
    assert len(size) > 5000 and size.max() == 320 * 320
    big = int(np.argmax(size))
    rng = np.random.default_rng(9)
    lo = np.asarray(m.origin_m)
    pos = lo + rng.uniform([0.2, 0.5, 0.5], [1.9, 39.5, 39.5], (48, 3))
    tiny = np.nonzero(size == 6)[0]
    cl = np.concatenate([np.full(len(pos), big), tiny])
    pos = np.concatenate([pos, cls["centroid"][tiny] + [0.25, 0.0, 0.0]])
    for unk in (False, True):
        st, sc, stats = check(m, fr, mirror, cl, pos, ORIENTS, (6.0, (1.0, 0.6)), 0.0, unk)
        assert np.all(sc <= size[cl][:, None]) and np.sum(st == 0) > len(st) - 5
        assert sc[:48].max() > 100 and sc[48:].max() > 0
    fr.close(); mirror.close()


def test_map_updated_after_the_frontier_compute():
    m, mirror = prepare(raycast_map("exact", "lidar", SIZES["gz32"], frames=2)[0])
    fr = m.Frontiers()
    fr.compute((0, 0, 0), tuple(g - 1 for g in m.grid_size), RES, 3)
    cl, pos = candidates(m, fr, np.random.default_rng(4))
    before = check(m, fr, mirror, cl, pos, ORIENTS, SENSORS[0], RES, True)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=8, edge=(0.3, 0.8))
    pts, T = scenes.lidar_frame(sc, np.array([0.5, 0.4, 0.0]), 1.1, beams=16, azimuths=360)
    m.RaycastFrame(pts, T, 0.3, 4.0)
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    after = check(m, fr, mirror, cl, pos, ORIENTS, SENSORS[0], RES, True)  # old members, new records
    assert not np.array_equal(before[1], after[1]) or not np.array_equal(before[0], after[0])
    fr.close(); mirror.close()


def test_properties_and_isolation():
    m, mirror = prepare(raycast_map("fast", "lidar", SIZES["gz30"], frames=3)[0])
    gs = m.grid_size
    fr = m.Frontiers()
    box = ((4, 7, 1), (49, 55, 26))
    fr.compute(box[0], box[1], RES, 2)
    rng = np.random.default_rng(6)
    cl, pos = candidates(m, fr, rng)
    D0, O0, C0 = m.export_distance(), m.export_occupancy(), m.export_closest_obstacle()
    L0, K0, V0 = fr.export(), fr.clusters(), fr.voxels()
    a = fr.score_viewpoints(cl, pos, ORIENTS, *SENSORS[0], RES)
    b = check(m, fr, mirror, cl, pos, ORIENTS, SENSORS[0], RES)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])           # determinism
    perm = rng.permutation(len(cl))
    c = fr.score_viewpoints(cl[perm], pos[perm], ORIENTS, *SENSORS[0], RES)
    assert np.array_equal(c[0], a[0][perm]) and np.array_equal(c[1], a[1][perm])
    assert np.all(a[1] <= K0["size"][cl][:, None])
    assert {k: c[2][k] for k in ("candidates_scored", "pairs_walked", "pairs_visible")} == {k: a[2][k] for k in ("candidates_scored", "pairs_walked", "pairs_visible")}
    # every status-0 candidate is a traversable voxel of a cost-to-go field at the same clearance, with or without the flag
    nav = m.NavField()
    ok = a[0] == 0
    v = np.floor((pos[ok] - np.asarray(ORIGIN)) / m.resolution).astype(int)
    for unk in (False, True):
        nav.compute((0, 0, 0), tuple(g - 1 for g in gs), np.zeros((0, 3)), RES, unknown_blocks=unk)
        F = nav.export()
        assert np.all(F[tuple(v.T)] >= 0) and ok.sum() > 0
    nav.close()
    # isolation: the map and the frontier result are unchanged
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert np.array_equal(m.export_closest_obstacle(), C0)
    assert np.array_equal(fr.export(), L0) and np.array_equal(fr.voxels(), V0)
    assert all(np.array_equal(fr.clusters()[k], K0[k]) for k in K0)
    fr.close(); mirror.close()


def test_invalid_arguments_write_nothing():
    import fiesta_b200
    m, mirror = prepare(raycast_map("fast", "lidar", SIZES["gz30"], frames=1)[0])
    L = m._L
    fr = m.Frontiers()
    n = 6
    cl0 = np.zeros(n, np.int32)
    pos0 = np.tile(np.asarray(ORIGIN) + 3.0, (n, 1))
    R0 = np.ascontiguousarray(ORIENTS[:4])
    status, score = np.full(n, -7, np.int32), np.full((n, 40), -7, np.int32)
    sm = lambda r=4.5, th=1.0, tv=0.5: fiesta_b200.SensorModel(r, (C.c_double * 2)(th, tv))

    def call(h=None, cl=cl0, pos=pos0, nn=n, R=R0, k=4, s="ok", r=RES, flags=0, st=status, sc=score):
        s = sm() if s == "ok" else s
        ptr = lambda a: None if a is None else a.ctypes
        return L.fiesta_frontiers_score_viewpoints(fr._h if h is None else h, ptr(cl), ptr(pos), C.c_int64(nn), ptr(R), C.c_int32(k),
                                                   None if s is None else C.byref(s), C.c_double(r), flags, ptr(st), ptr(sc), None)

    assert call() == 1                                                      # before any compute
    fr.compute((0, 0, 0), tuple(g - 1 for g in m.grid_size), RES, 2)
    K = fr.stats["kept_clusters"]
    L0, V0 = fr.export(), fr.voxels()
    nanR = R0.copy(); nanR[2, 1, 1] = np.nan
    infR = R0.copy(); infR[0, 0, 0] = np.inf
    bad = [call(cl=np.full(n, K, np.int32)), call(cl=np.full(n, -1, np.int32)), call(k=0), call(k=-2),
           call(s=sm(r=0.0)), call(s=sm(r=-1.0)), call(s=sm(r=np.nan)), call(s=sm(r=np.inf)),
           call(s=sm(th=0.0)), call(s=sm(tv=-0.5)), call(s=sm(th=np.nan)), call(s=sm(tv=np.inf)), call(s=None),
           call(R=nanR), call(R=infR), call(R=None), call(r=np.nan), call(r=-0.1), call(r=10000.0), call(flags=2),
           call(cl=None), call(pos=None), call(st=None), call(sc=None), call(nn=-1), call(h=C.c_void_p(0))]
    assert bad == [1] * len(bad), bad                                       # FIESTA_ERR_INVALID
    R33 = np.ascontiguousarray(viewref.yaws(33))
    assert call(R=R33, k=33) == 4                                           # FIESTA_ERR_LIMIT
    assert np.all(status == -7) and np.all(score == -7)                     # nothing written
    assert np.array_equal(fr.export(), L0) and np.array_equal(fr.voxels(), V0)
    assert call(cl=None, pos=None, nn=0, st=None, sc=None) == 0             # no candidates: nothing to do
    with pytest.raises(fiesta_b200.FiestaError):
        fr.score_viewpoints([K], [pos0[0]], ORIENTS, *SENSORS[0])
    check(m, fr, mirror, cl0, pos0, ORIENTS, SENSORS[0], RES)                # still usable
    fr.close(); mirror.close()
