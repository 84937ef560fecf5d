"""GPU: the cost-to-go field (fiesta_nav_*) against tests/navref.py evaluated on export_distance() of the same map -- every field
with np.array_equal, every path voxel for voxel with the same status, length and cost -- on ray-cast maps in both modes, on a
serpentine maze that takes hundreds of generations, and in the corner cases of goals, clearances and boxes.  Also: determinism,
isolation from the map, and argument validation."""
import ctypes as C

import numpy as np
import pytest

from tests import navref, scenes

pytestmark = pytest.mark.gpu

ORIGIN, RES = (-3.2, -3.2, -1.6), 0.1
SIZES = {"gz32": (6.4, 6.4, 3.2), "gz30": (6.4, 6.4, 3.0)}     # Gz = 30: padded z pitch Pz = 32 != Gz


def raycast_map(mode, kind, size, frames=4):
    """A ray-cast map with moving boxes (TOGGLE parameters: a box that moves away is deleted at once)."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, size, mode=mode)
    m.size_m = size                                                         # PosInMap range of path starts: ORIGIN + size
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    deletes = 0
    for p, yaw in scenes.pose_walk(frames, seed=2, clamp=0.5):
        if kind == "lidar":
            pts, T = scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=360)
        else:
            pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
        m.RaycastFrame(pts, T, 0.3, 4.0)
        if m.CheckUpdate():
            m.UpdateOccupancy(True)
            m.UpdateESDF()
            deletes += m.stats()["deletes"]
        for _ in range(3):
            sc.step()
    return m, deletes


def goal_positions(m, box, k, rng):
    """k random goal positions inside the box (voxel centres jittered inside the voxel)."""
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    v = np.stack([rng.integers(lo[i], hi[i] + 1, k) for i in range(3)], -1)
    return np.asarray(ORIGIN) + (v + rng.uniform(0.05, 0.95, v.shape)) * m.resolution


def expected(m, D, box, goals, r, unk):
    gv = np.floor((np.asarray(goals).reshape(-1, 3) - np.asarray(ORIGIN)) / m.resolution)
    gv = np.where(np.isfinite(gv), gv, -1).astype(np.int64)
    return navref.field(D, m.grid_size, box, gv, r, unk, m.resolution)


def placed(m, D, box, goals, r, unk):
    v, ok = navref.locate(goals, ORIGIN, m.resolution, box)
    T = navref.traversable(D.reshape(m.grid_size)[navref.box_slices(box)], r, unk)
    return int(np.sum(ok & T[tuple(v.T)]))


def check_field(m, nav, box, goals, r, unk, D=None):
    """Compute on the device, compare with navref bit for bit; returns the field."""
    D = m.export_distance() if D is None else D
    st = nav.compute(box[0], box[1], goals, r, unknown_blocks=unk)
    got = nav.export()
    want = expected(m, D, box, goals, r, unk)
    assert got.shape == want.shape
    assert np.array_equal(got, want), (box, r, unk, int(np.sum(got != want)))
    assert st["box_voxels"] == want.size and st["blocked"] == int(np.sum(want < 0))
    assert st["reached"] == int(np.sum((want >= 0) & (want < np.inf)))
    assert st["goals_placed"] == placed(m, D, box, goals, r, unk)
    return want, st


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def check_paths(m, nav, F, box, starts, max_len):
    lo, hi = np.asarray(ORIGIN), np.asarray(ORIGIN) + np.asarray(m.size_m)
    got = nav.paths(starts, max_len)
    v, ok = navref.locate(starts, ORIGIN, m.resolution, box, lo, hi)
    want = navref.paths(F, box, m.resolution, v, ok, max_len)
    for name, a, b in zip(("status", "len", "cost", "vox"), got, want):
        assert same(a, b), (name, int(np.sum(np.asarray(a) != np.asarray(b))))
    st, ln, cost, vox = got
    for i in np.nonzero(st == 0)[0][:300]:
        assert navref.fold(F, box, m.resolution, vox[i, :ln[i]]) == cost[i]
    return set(int(s) for s in st)


def starts_for(m, box, n, rng, goals):
    """Starts in and around the box (some outside the map), a NaN, and the goals themselves."""
    lo = np.asarray(ORIGIN) + np.asarray(box[0]) * m.resolution
    hi = np.asarray(ORIGIN) + (np.asarray(box[1]) + 1) * m.resolution
    s = rng.uniform(lo - 0.3, hi + 0.3, (n, 3))
    return np.concatenate([s, [[np.nan, 0.0, 0.0]], np.asarray(goals).reshape(-1, 3)])


def boxes(gs):
    gx, gy, gz = gs
    return [((0, 0, 0), (gx - 1, gy - 1, gz - 1)),                  # the whole grid
            ((10, 12, 3), (50, 47, gz - 5)),                          # a local box, not aligned to tiles
            ((0, 5, 0), (gx - 1, 40, gz - 1)),                        # touches the x and z faces
            ((3, 0, 1), (37, gy - 1, gz - 2))]                        # touches the y faces


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_field_and_paths_on_raycast_maps(kind, mode, size):
    m, deletes = raycast_map(mode, kind, SIZES[size])
    assert deletes > 0
    nav = m.NavField()
    rng = np.random.default_rng(5)
    D = m.export_distance()
    statuses = set()
    generations = 0
    for bi, box in enumerate(boxes(m.grid_size)):
        for r in (0.0, RES, 2.5 * RES):
            for unk in (False, True):
                goals = goal_positions(m, box, 4, rng)
                F, st = check_field(m, nav, box, goals, r, unk, D)
                generations = max(generations, st["generations"])
                if r == RES and bi < 2:
                    for max_len in (4, 64):                               # the short one truncates most paths
                        statuses |= check_paths(m, nav, F, box, starts_for(m, box, 1000, rng, goals), max_len)
    assert statuses == {0, 1, 2, 3}, statuses
    assert generations > 3
    nav.close()


def maze_map(gs=(96, 96, 12), size=(9.6, 9.6, 1.2)):
    """A fully observed serpentine maze: walls along x on every third y row, each with a 2-voxel gap at alternating ends, through
    the whole height.  The one corridor runs back and forth across the x tiles about 32 times."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, size, mode="fast")
    m.size_m = size
    assert m.grid_size == gs
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(gs)
    m.SetOccupancyBatchVox(allv, np.zeros(len(allv), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    walls = []
    for i, y in enumerate(range(2, gs[1] - 1, 3)):
        xs = range(0, gs[0] - 2) if i % 2 == 0 else range(2, gs[0])
        walls += [(x, y, z) for x in xs for z in range(gs[2])]
    walls = np.array(walls, np.int32)
    m.SetOccupancyBatchVox(walls, np.ones(len(walls), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    return m


def test_maze_takes_hundreds_of_generations():
    m = maze_map()
    gs = m.grid_size
    nav = m.NavField()
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    goal = np.asarray(ORIGIN) + (np.array([1, 0, 5]) + 0.5) * RES
    F, st = check_field(m, nav, box, goal[None], 0.0, False)
    assert st["generations"] > 200, st
    far = F[:, -1, :]
    assert np.all(far[far >= 0] > 80 * 32 * RES * 0.9)                     # the far end is reached the long way round
    rng = np.random.default_rng(3)
    statuses = check_paths(m, nav, F, box, starts_for(m, box, 500, rng, goal[None]), 4000)
    assert 0 in statuses
    # several goals, including both ends of the corridor
    goals = np.concatenate([goal[None], np.asarray(ORIGIN) + (np.array([[90, 94, 2], [40, 45, 7]]) + 0.5) * RES])
    check_field(m, nav, box, goals, 0.0, False)
    nav.close()


def test_goal_on_tile_face_or_corner():
    """Goals connected to the rest of free space only across a tile face or a tile corner (tests/test_nav_oracle.py's boundary
    grid, written with SetOccupancyBatchVox): the tiles behind the goal must be relaxed too."""
    import fiesta_b200
    from tests.test_nav_oracle import BOUNDARY_CASES, boundary_grid
    gs, D0 = boundary_grid()
    res = 0.125
    size = tuple(g * res for g in gs)                                      # exact in binary
    m = fiesta_b200.ESDFMap(ORIGIN, res, size, mode="fast")
    m.size_m = size
    assert m.grid_size == gs
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(gs)
    free = D0.reshape(gs)[tuple(allv.T)] > 0
    m.SetOccupancyBatchVox(allv, (~free).astype(np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    nav = m.NavField()
    for lo, goal, far in BOUNDARY_CASES:
        box = (lo, tuple(g - 1 for g in gs))
        F, st = check_field(m, nav, box, (np.asarray(ORIGIN) + (np.asarray(goal) + 0.5) * res)[None], 0.0, False)
        assert st["goals_placed"] == 1
        assert np.isfinite(F[tuple(np.asarray(far) - np.asarray(lo))]), (goal, far)
    nav.close()


def test_goal_and_clearance_corner_cases():
    m, _ = raycast_map("fast", "lidar", SIZES["gz32"], frames=2)
    nav = m.NavField()
    gs = m.grid_size
    box = ((5, 6, 2), (58, 57, 29))
    D = m.export_distance()
    Db = D.reshape(gs)[navref.box_slices(box)]
    free = np.argwhere((Db > 0.5) & (Db < 100)) + np.asarray(box[0])
    blocked = np.argwhere((Db >= 0) & (Db <= 0.05)) + np.asarray(box[0])
    assert len(free) and len(blocked)
    centre = lambda v: np.asarray(ORIGIN) + (np.asarray(v) + 0.5) * RES
    g_free = centre(free[[0, len(free) // 2, -1]])
    g_block = centre(blocked[:1])
    g_out = centre([[1, 1, 1]])                                              # in the grid, outside the box
    # duplicates, a blocked goal and one outside the box: only the free ones are placed (duplicates counted)
    goals = np.concatenate([g_free, g_free[:1], g_block, g_out])
    F, st = check_field(m, nav, box, goals, 0.1, False, D)
    assert st["goals_placed"] == 4
    # no goal placed: all blocked or outside -> +inf everywhere that is traversable
    F, st = check_field(m, nav, box, np.concatenate([g_block, g_out]), 0.1, False, D)
    assert st["goals_placed"] == 0 and st["reached"] == 0 and np.all((F == -1) | (F == np.inf))
    F, st = check_field(m, nav, box, np.zeros((0, 3)), 0.1, False, D)    # no goals at all
    assert st["reached"] == 0
    # a clearance that blocks every voxel with a finite distance, with unknown space blocking too: only unreached (+10000) voxels
    # stay traversable, and no goal lies on one
    F, st = check_field(m, nav, box, g_free, 9999.0, True, D)
    assert st["blocked"] == int(np.sum(Db != 10000)) and st["goals_placed"] == 0 and st["reached"] == 0
    # the unknown flag: on and off, with goals in unknown space
    unknown = np.argwhere(Db == -10000) + np.asarray(box[0])
    assert len(unknown)
    g_unk = centre(unknown[:2])
    _, st_off = check_field(m, nav, box, np.concatenate([g_unk, g_free]), 0.1, False, D)
    _, st_on = check_field(m, nav, box, np.concatenate([g_unk, g_free]), 0.1, True, D)
    assert st_off["goals_placed"] == 5 and st_on["goals_placed"] == 3 and st_on["blocked"] > st_off["blocked"]
    # a single-voxel box and 1-voxel-thick boxes
    v = free[0]
    check_field(m, nav, (tuple(v), tuple(v)), centre(v)[None], 0.1, False, D)
    check_field(m, nav, ((v[0], 0, 0), (v[0], gs[1] - 1, gs[2] - 1)), centre(v)[None], 0.1, False, D)
    check_field(m, nav, ((0, 0, v[2]), (gs[0] - 1, gs[1] - 1, v[2])), centre(v)[None], 0.1, False, D)
    nav.close()


def test_determinism_and_isolation():
    m, _ = raycast_map("exact", "lidar", SIZES["gz30"], frames=3)
    gs = m.grid_size
    rng = np.random.default_rng(9)
    box = ((4, 7, 1), (49, 55, 26))
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    goals = goal_positions(m, box, 6, rng)
    D0, O0, S0 = m.export_distance(), m.export_occupancy(), m.stats()
    nav = m.NavField()
    F1, _ = check_field(m, nav, box, goals, RES, False)
    F2, _ = check_field(m, nav, box, goals, RES, False)
    assert np.array_equal(F1, F2)
    check_field(m, nav, full, goals, RES, True)                            # a larger box on the same object ...
    F3, _ = check_field(m, nav, box, goals, RES, False)                    # ... then the small one again
    assert np.array_equal(F1, F3)
    other = m.NavField()
    other.compute(box[0], box[1], goals, RES)
    assert np.array_equal(other.export(), F1)
    other.close()
    starts = starts_for(m, box, 500, rng, goals)
    P1 = nav.paths(starts, 64)
    assert all(same(a, b) for a, b in zip(P1, nav.paths(starts, 64)))
    # the map is untouched, apart from the launch counter
    S1 = m.stats()
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert {k: v for k, v in S0.items() if k != "kernel_launches"} == {k: v for k, v in S1.items() if k != "kernel_launches"}
    assert S1["kernel_launches"] > S0["kernel_launches"]
    # the field keeps its bits across a map update until it is recomputed
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=4, edge=(0.3, 0.8))
    for _ in range(4):
        sc.step()
    pts, T = scenes.lidar_frame(sc, np.array([0.4, -0.3, 0.1]), 0.7, beams=16, azimuths=360)
    m.RaycastFrame(pts, T, 0.3, 4.0); m.UpdateOccupancy(True); m.UpdateESDF()
    assert not np.array_equal(m.export_distance(), D0)
    assert np.array_equal(nav.export(), F1)
    assert all(same(a, b) for a, b in zip(P1, nav.paths(starts, 64)))
    F4, _ = check_field(m, nav, box, goals, RES, False)                    # recomputed: navref on the new records
    assert not np.array_equal(F4, F1)
    nav.close()


def test_invalid_arguments_change_nothing():
    import fiesta_b200
    m, _ = raycast_map("fast", "lidar", SIZES["gz30"], frames=1)
    gs = m.grid_size
    L = m._L
    nav = m.NavField()
    rng = np.random.default_rng(2)
    box = ((2, 3, 4), (40, 50, 20))
    goals = goal_positions(m, box, 3, rng)
    F, _ = check_field(m, nav, box, goals, RES, False)
    starts = starts_for(m, box, 200, rng, goals)
    P = nav.paths(starts, 32)
    I3 = lambda v: np.ascontiguousarray(v, np.int32)
    g = np.ascontiguousarray(goals)
    st = fiesta_b200.NavStats()

    def compute(lo, hi, gp=g.ctypes, n=len(g), r=RES, flags=0):
        return L.fiesta_nav_compute(nav._h, I3(lo).ctypes, I3(hi).ctypes, gp, n, C.c_double(r), flags, C.byref(st))

    bad = [compute((5, 3, 4), (4, 50, 20)),                                 # inverted
           compute((-1, 3, 4), (40, 50, 20)),                               # below the grid
           compute((2, 3, 4), (gs[0], 50, 20)),                             # beyond the grid
           compute((2, 3, 4), (40, 50, gs[2])),
           compute((2, 3, 4), (40, 50, 20), r=float("nan")),
           compute((2, 3, 4), (40, 50, 20), r=-0.1),
           compute((2, 3, 4), (40, 50, 20), r=10000.0),
           compute((2, 3, 4), (40, 50, 20), flags=2),
           compute((2, 3, 4), (40, 50, 20), gp=None),
           compute((2, 3, 4), (40, 50, 20), n=-1),
           L.fiesta_nav_compute(nav._h, None, I3((40, 50, 20)).ctypes, g.ctypes, len(g), C.c_double(RES), 0, None),
           L.fiesta_nav_compute(None, I3((2, 3, 4)).ctypes, I3((40, 50, 20)).ctypes, g.ctypes, len(g), C.c_double(RES), 0, None),
           L.fiesta_nav_export(nav._h, None),
           L.fiesta_nav_export(None, np.empty(10).ctypes)]
    s = np.ascontiguousarray(starts)
    outs = [np.empty(len(s), np.int32), np.empty(len(s), np.int32), np.empty(len(s)), np.empty((len(s), 32, 3), np.int32)]
    bad += [L.fiesta_nav_paths(nav._h, s.ctypes, len(s), 0, *(o.ctypes for o in outs)),
            L.fiesta_nav_paths(nav._h, s.ctypes, len(s), -3, *(o.ctypes for o in outs)),
            L.fiesta_nav_paths(nav._h, s.ctypes, -1, 32, *(o.ctypes for o in outs)),
            L.fiesta_nav_paths(nav._h, None, len(s), 32, *(o.ctypes for o in outs)),
            L.fiesta_nav_paths(nav._h, s.ctypes, len(s), 32, None, *(o.ctypes for o in outs[1:]))]
    assert bad == [1] * len(bad), bad                                       # FIESTA_ERR_INVALID
    assert np.array_equal(nav.export(), F)
    assert all(same(a, b) for a, b in zip(P, nav.paths(starts, 32)))
    fresh = m.NavField()                                                    # export / paths before any compute
    assert L.fiesta_nav_export(fresh._h, np.empty(10).ctypes) == 1
    assert L.fiesta_nav_paths(fresh._h, s.ctypes, len(s), 32, *(o.ctypes for o in outs)) == 1
    fresh.close()
    with pytest.raises(fiesta_b200.FiestaError):
        nav.compute((0, 0, 0), (gs[0], 1, 1), goals, RES)
    check_field(m, nav, box, goals, RES, False)                            # still usable
    nav.close()
