"""GPU: frontier extraction (fiesta_frontiers_*) against tests/frontierref.py evaluated on export_distance() and
export_occupancy() of the same map -- labels, cluster arrays, member lists and stats with np.array_equal -- on ray-cast maps in
both modes, between UpdateOccupancy and UpdateESDF, after an EXACT local-map reset, and on crafted maps: clusters joined only across
tile faces, edges and corners, a serpentine and a diagonal chain through many tiles, thousands of small clusters, empty results and
a 1-voxel box.  Also: determinism, isolation from the map, agreement with the cost-to-go field, cap truncation and argument
validation."""
import ctypes as C

import numpy as np
import pytest

from tests import frontierref, scenes
from tests.test_gpu_nav import ORIGIN, RES, SIZES, boxes, raycast_map

pytestmark = pytest.mark.gpu

L_OCC = frontierref.l_occ(scenes.PARAMS_TOGGLE[4])


def check(m, fr, box, r, min_size, D=None, O=None):
    """Compute on the device and compare every output with frontierref; returns the expected dict."""
    D = m.export_distance() if D is None else D
    O = m.export_occupancy() if O is None else O
    st = fr.compute(box[0], box[1], r, min_size)
    want = frontierref.extract(D, O, m.grid_size, box, r, L_OCC, min_size, m.resolution, ORIGIN)
    assert {k: st[k] for k in want["stats"]} == want["stats"], (box, r, min_size, st, want["stats"])
    assert np.array_equal(fr.export(), want["labels"]), (box, r, min_size)
    got = fr.clusters()
    for k in ("size", "rep", "bbox_lo", "bbox_hi", "centroid"):
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), (k, box, r, min_size)
    assert np.array_equal(fr.voxels(), want["voxels"]), (box, r, min_size)
    return want


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_raycast_maps(kind, mode, size):
    m, _ = raycast_map(mode, kind, SIZES[size])
    fr = m.Frontiers()
    D, O = m.export_distance(), m.export_occupancy()
    gs = m.grid_size
    kept = 0
    for box in boxes(gs) + [((0, 0, 0), (gs[0] - 1, gs[1] - 1, 0)), ((0, 0, gs[2] - 1), (gs[0] - 1, gs[1] - 1, gs[2] - 1)),
                            ((gs[0] - 1, 0, 0), (gs[0] - 1, gs[1] - 1, gs[2] - 1)), ((0, gs[1] - 1, 0), (gs[0] - 1, gs[1] - 1, gs[2] - 1))]:
        for r in (0.0, RES, 2.5 * RES):
            for min_size in (1, 5):
                kept += check(m, fr, box, r, min_size, D, O)["stats"]["kept_clusters"]
    assert kept > 0
    fr.close()


def test_between_update_occupancy_and_esdf_and_pending_counters():
    m, _ = raycast_map("exact", "lidar", SIZES["gz32"], frames=2)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=8, edge=(0.3, 0.8))
    pts, T = scenes.lidar_frame(sc, np.array([0.5, 0.4, 0.0]), 1.1, beams=16, azimuths=360)
    fr = m.Frontiers()
    full = ((0, 0, 0), tuple(g - 1 for g in m.grid_size))
    m.RaycastFrame(pts, T, 0.3, 4.0)
    check(m, fr, full, RES, 1)                                             # pending counters: not part of the snapshot
    m.UpdateOccupancy(True)                                                # log-odds integrated, distances not yet updated
    check(m, fr, full, RES, 1)
    m.UpdateESDF()
    check(m, fr, full, RES, 1)
    fr.close()


def test_exact_local_map_reset():
    """UpdateOccupancy(false) with a moving local box leaves voxels whose distance reads +10000 while they keep their obstacle
    (FB_DINF) until UpdateESDF rewrites them: they are observed."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZES["gz32"], mode="exact")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    radius = np.array([1.5, 1.5, 1.0])
    poses = scenes.pose_walk(4, seed=2, clamp=0.5)
    for i, (p, yaw) in enumerate(poses):
        if i:
            m.SetUpdateRange(p - radius, p + radius)
        pts, T = scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=360)
        m.RaycastFrame(pts, T, 0.3, 4.0)
        m.UpdateOccupancy(i == 0)
        if i + 1 < len(poses):
            m.UpdateESDF()
        sc.step()
    D = m.export_distance()
    cobs = m.export_closest_obstacle()
    assert np.any((D == 10000) & (cobs[:, 0] >= 0)), "no local-map reset voxel"
    fr = m.Frontiers()
    for box in boxes(m.grid_size)[:2]:
        for r in (0.0, RES):
            check(m, fr, box, r, 1, D)
    m.UpdateESDF()
    check(m, fr, boxes(m.grid_size)[0], RES, 1)
    fr.close()


def crafted_map(gs, free, occupied=()):
    """A map of 0.125 m voxels (sizes exact in binary) that has observed only the voxels `free` (free) and `occupied`; everything
    else is unknown."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, 0.125, tuple(g * 0.125 for g in gs), mode="fast")
    assert m.grid_size == tuple(gs)
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    free = np.asarray(free, np.int32).reshape(-1, 3)
    occ = np.asarray(occupied, np.int32).reshape(-1, 3)
    v = np.concatenate([free, occ])
    if len(v):
        m.SetOccupancyBatchVox(v, np.concatenate([np.zeros(len(free), np.uint8), np.ones(len(occ), np.uint8)]))
        m.UpdateOccupancy(True)
        m.UpdateESDF()
    return m


def test_clusters_joined_across_tile_faces_edges_and_corners():
    gs = (40, 40, 40)
    # pairs of voxels that touch only across a tile boundary of the box starting at 0, and of the box starting at 4
    pairs = []
    for off in (0, 4):
        b = 8 + off - 1
        pairs += [[(b, 2 + off, 2 + off), (b + 1, 2 + off, 2 + off)],           # face (x)
                  [(2 + off, b, 20), (2 + off, b + 1, 20)],                      # face (y)
                  [(20, 2 + off, b), (20, 2 + off, b + 1)],                      # face (z)
                  [(b, b, 30), (b + 1, b + 1, 30)],                              # edge (xy)
                  [(30, b, b), (30, b + 1, b + 1)],                              # edge (yz)
                  [(b + 8, 30, b + 8), (b + 9, 30, b + 7)],                      # edge (xz), the other diagonal
                  [(b + 16, b + 16, b + 16), (b + 17, b + 17, b + 17)],          # corner
                  [(b + 8, b + 17, b + 8), (b + 9, b + 16, b + 9)]]              # corner, mixed signs
    m = crafted_map(gs, np.concatenate(pairs))
    fr = m.Frontiers()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    w = check(m, fr, full, 0.0, 1)
    assert w["stats"]["frontier_voxels"] == 2 * len(pairs) and w["stats"]["clusters"] == len(pairs)
    assert np.all(w["size"] == 2)
    check(m, fr, ((4, 4, 4), tuple(g - 1 for g in gs)), 0.0, 2)          # the second set on the tile lattice of this box
    check(m, fr, ((4, 4, 4), (27, 27, 27)), 0.0, 1)                       # pairs cut by the box's faces stay cut
    fr.close()


def test_serpentine_and_diagonal_chain_through_many_tiles():
    gs = (64, 64, 64)
    v = []
    for i, y in enumerate(range(0, gs[1], 2)):                             # rows along x joined at alternating ends
        v += [(x, y, 5) for x in range(gs[0])]
        if y + 1 < gs[1]:
            v.append((gs[0] - 1 if i % 2 == 0 else 0, y + 1, 5))
    chain = [(i, i, i) for i in range(8, 64)]                              # crosses tiles only through their corners
    m = crafted_map(gs, np.array(v + chain))
    fr = m.Frontiers()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    w = check(m, fr, full, 0.0, 1)
    assert w["stats"]["clusters"] == 2 and sorted(w["size"]) == [len(chain), len(v)]
    check(m, fr, ((3, 5, 0), (60, 61, 40)), 0.0, 1)
    check(m, fr, full, 0.0, 20)
    fr.close()


def test_thousands_of_small_clusters():
    gs = (96, 96, 24)
    rng = np.random.default_rng(4)
    base = np.stack(np.meshgrid(*[np.arange(0, g - 1, 3) for g in gs], indexing="ij"), -1).reshape(-1, 3)
    extra = base + rng.integers(0, 2, base.shape)                          # a second voxel in the same 2^3 block, sometimes
    extra2 = base + rng.integers(0, 2, base.shape)
    v = np.unique(np.concatenate([base, extra[rng.random(len(base)) < 0.5], extra2[rng.random(len(base)) < 0.3]]), axis=0)
    m = crafted_map(gs, v)
    fr = m.Frontiers()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    for min_size in (1, 2, 3, 5):
        w = check(m, fr, full, 0.0, min_size)
        if min_size == 1:
            assert w["stats"]["clusters"] > 5000
    check(m, fr, ((5, 7, 2), (77, 90, 20)), 0.0, 2)
    fr.close()


def test_empty_results_and_single_voxel_box():
    gs = (24, 24, 16)
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    m = crafted_map(gs, [])                                                # nothing observed
    fr = m.Frontiers()
    w = check(m, fr, full, 0.0, 1)
    assert w["stats"]["frontier_voxels"] == 0 and w["stats"]["kept_clusters"] == 0
    fr.close()
    m = crafted_map(gs, scenes.all_voxels(gs))                             # nothing unknown
    fr = m.Frontiers()
    w = check(m, fr, full, 0.0, 1)
    assert w["stats"]["frontier_voxels"] == 0
    fr.close()
    m = crafted_map(gs, [(5, 5, 5), (5, 5, 6), (9, 9, 9)], occupied=[(12, 12, 12)])
    fr = m.Frontiers()
    for v in ((5, 5, 5), (9, 9, 9), (12, 12, 12), (0, 0, 0)):
        check(m, fr, (v, v), 0.0, 1)
    w = check(m, fr, ((5, 5, 5), (5, 5, 5)), 0.0, 1)
    assert w["stats"]["kept_voxels"] == 1
    check(m, fr, full, 2.5 * RES, 1)                                       # the obstacle blocks the free voxels next to it
    check(m, fr, full, 0.0, 10**12)                                        # every cluster dropped
    fr.close()


def test_determinism_isolation_nav_and_cap():
    m, _ = raycast_map("exact", "lidar", SIZES["gz30"], frames=3)
    gs = m.grid_size
    box = ((4, 7, 1), (49, 55, 26))
    D0, O0, S0 = m.export_distance(), m.export_occupancy(), m.stats()
    fr = m.Frontiers()
    w = check(m, fr, box, RES, 1)
    outs = lambda: (fr.export(), fr.clusters(), fr.voxels())
    a = outs()
    fr.compute(box[0], box[1], RES, 1)
    b = outs()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])
    check(m, fr, ((0, 0, 0), tuple(g - 1 for g in gs)), RES, 5)            # a larger box, then the small one again
    check(m, fr, box, RES, 1)
    # every frontier voxel is a traversable voxel of a cost-to-go field at the same clearance
    nav = m.NavField()
    nav.compute(box[0], box[1], np.zeros((0, 3)), RES)
    F = nav.export()
    assert np.all(F[a[0] >= 0] >= 0) and w["stats"]["kept_voxels"] > 0
    nav.close()
    # cap truncation
    K, M = w["stats"]["kept_clusters"], w["stats"]["kept_voxels"]
    for cap in (0, 1, K // 2):
        got = fr.clusters(cap)
        assert all(np.array_equal(got[k], w[k][:cap]) for k in got)
    for cap in (0, 1, M // 3):
        assert np.array_equal(fr.voxels(cap), w["voxels"][:cap])
    big = np.full((K + 5, 3), -7, np.int32)
    L = m._L
    args = [np.empty(K + 5, np.int64), big, np.empty((K + 5, 3), np.int32), np.empty((K + 5, 3), np.int32), np.empty((K + 5, 3))]
    assert L.fiesta_frontiers_clusters(fr._h, K + 5, *(x.ctypes for x in args)) == 0
    assert np.array_equal(big[:K], w["rep"]) and np.all(big[K:] == -7)
    # the map is untouched, apart from the launch counter, and its next update is the same as without the extraction
    S1 = m.stats()
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert {k: v for k, v in S0.items() if k != "kernel_launches"} == {k: v for k, v in S1.items() if k != "kernel_launches"}
    m2, _ = raycast_map("exact", "lidar", SIZES["gz30"], frames=3)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=4, edge=(0.3, 0.8))
    pts, T = scenes.lidar_frame(sc, np.array([0.4, -0.3, 0.1]), 0.7, beams=16, azimuths=360)
    for mm in (m, m2):
        mm.RaycastFrame(pts, T, 0.3, 4.0); mm.UpdateOccupancy(True); mm.UpdateESDF()
    assert np.array_equal(m.export_distance(), m2.export_distance())
    assert np.array_equal(m.export_closest_obstacle(), m2.export_closest_obstacle())
    assert np.array_equal(m.export_occupancy(), m2.export_occupancy())
    assert np.array_equal(fr.export(), w["labels"])                        # a snapshot until recomputed
    fr.close()


def test_invalid_arguments_change_nothing():
    import fiesta_b200
    m, _ = raycast_map("fast", "lidar", SIZES["gz30"], frames=1)
    gs = m.grid_size
    L = m._L
    fr = m.Frontiers()
    box = ((2, 3, 4), (40, 50, 20))
    w = check(m, fr, box, RES, 1)
    I3 = lambda v: np.ascontiguousarray(v, np.int32)
    st = fiesta_b200.FrontierStats()

    def compute(lo, hi, r=RES, ms=1):
        return L.fiesta_frontiers_compute(fr._h, I3(lo).ctypes, I3(hi).ctypes, C.c_double(r), C.c_int64(ms), C.byref(st))

    buf = [np.empty(10, np.int64), np.empty((10, 3), np.int32), np.empty((10, 3), np.int32), np.empty((10, 3), np.int32), np.empty((10, 3))]
    bad = [compute((5, 3, 4), (4, 50, 20)), compute((-1, 3, 4), (40, 50, 20)), compute((2, 3, 4), (gs[0], 50, 20)),
           compute((2, 3, 4), (40, gs[1], 20)), compute((2, 3, 4), (40, 50, gs[2])),
           compute((2, 3, 4), (40, 50, 20), r=float("nan")), compute((2, 3, 4), (40, 50, 20), r=-0.1),
           compute((2, 3, 4), (40, 50, 20), r=10000.0), compute((2, 3, 4), (40, 50, 20), ms=0), compute((2, 3, 4), (40, 50, 20), ms=-3),
           L.fiesta_frontiers_compute(fr._h, None, I3((40, 50, 20)).ctypes, C.c_double(RES), 1, None),
           L.fiesta_frontiers_compute(fr._h, I3((2, 3, 4)).ctypes, None, C.c_double(RES), 1, None),
           L.fiesta_frontiers_compute(None, I3((2, 3, 4)).ctypes, I3((40, 50, 20)).ctypes, C.c_double(RES), 1, None),
           L.fiesta_frontiers_export(fr._h, None), L.fiesta_frontiers_export(None, np.empty(10, np.int32).ctypes),
           L.fiesta_frontiers_voxels(fr._h, 10, None), L.fiesta_frontiers_voxels(fr._h, -1, buf[1].ctypes),
           L.fiesta_frontiers_voxels(None, 10, buf[1].ctypes),
           L.fiesta_frontiers_clusters(fr._h, -1, *(b.ctypes for b in buf)),
           L.fiesta_frontiers_clusters(None, 10, *(b.ctypes for b in buf))]
    for i in range(5):
        bad.append(L.fiesta_frontiers_clusters(fr._h, 10, *(None if j == i else b.ctypes for j, b in enumerate(buf))))
    assert bad == [1] * len(bad), bad                                       # FIESTA_ERR_INVALID
    assert np.array_equal(fr.export(), w["labels"]) and np.array_equal(fr.voxels(), w["voxels"])
    assert np.array_equal(fr.clusters()["centroid"], w["centroid"])
    fresh = m.Frontiers()                                                  # reads before any compute
    assert L.fiesta_frontiers_export(fresh._h, np.empty(10, np.int32).ctypes) == 1
    assert L.fiesta_frontiers_voxels(fresh._h, 10, buf[1].ctypes) == 1
    assert L.fiesta_frontiers_clusters(fresh._h, 10, *(b.ctypes for b in buf)) == 1
    fresh.close()
    with pytest.raises(fiesta_b200.FiestaError):
        fr.compute((0, 0, 0), (gs[0], 1, 1), RES)
    assert np.array_equal(fr.export(), w["labels"])                        # a refused compute changes nothing
    check(m, fr, box, RES, 1)                                              # still usable
    fr.close()
