"""GPU: the cost-to-go field update (fiesta_nav_update).  After every map change, update() must give the bits of compute() on a
second NavField with the same box, goals, clearance and flags, and of tests/navref.py on export_distance(); its withdrawn count
must be the model's (tests/navupdref.py), its other statistics the fresh compute's or the numpy diff of the traversability, and its
paths navref's voxel for voxel.  Covered: chained ray-cast LIDAR and depth frames with moving boxes in both modes (full grid, a
local box, boxes on the grid faces, Gz = 30, the unknown flag with newly observed voxels), single-voxel edits on a serpentine maze
and a diagonal gap, a local-map reset, an update with nothing changed, a matrix between compute and update, a compute on another
box, an update before any compute, and the map left untouched."""
import ctypes as C

import numpy as np
import pytest

from tests import navref, navupdref, scenes
from tests.test_gpu_nav import ORIGIN, RES, SIZES, check_paths, expected, goal_positions, maze_map, placed, starts_for

pytestmark = pytest.mark.gpu


class Tracked:
    """A field kept up to date by update(), its reference twin recomputed from scratch, and what the checks need."""

    def __init__(self, m, box, goals, r, unk):
        self.m, self.box, self.goals, self.r, self.unk = m, box, goals, r, unk
        self.nav, self.ref = m.NavField(), m.NavField()
        st = self.nav.compute(box[0], box[1], goals, r, unknown_blocks=unk)
        self.F = self.nav.export()
        assert np.array_equal(self.F, expected(m, m.export_distance(), box, goals, r, unk))
        self.placed0 = st["goals_placed"]

    def check(self, paths=False, rng=None):
        m, box, goals, r, unk = self.m, self.box, self.goals, self.r, self.unk
        st = self.nav.update()
        got = self.nav.export()
        rs = self.ref.compute(box[0], box[1], goals, r, unknown_blocks=unk)
        assert np.array_equal(got, self.ref.export())
        D = m.export_distance()
        want = expected(m, D, box, goals, r, unk)
        assert np.array_equal(got, want), (box, r, unk, int(np.sum(got != want)))
        Told = self.F >= 0
        Tnew = navref.traversable(D.reshape(m.grid_size)[navref.box_slices(box)], r, unk)
        for k in ("box_voxels", "blocked", "reached", "goals_placed"):
            assert st[k] == rs[k], (k, st[k], rs[k])
        assert st["became_blocked"] == int(np.sum(Told & ~Tnew)) and st["became_free"] == int(np.sum(Tnew & ~Told))
        assert st["withdrawn"] == int(navupdref.withdrawn(self.F, Tnew, m.resolution).sum())
        v, ok = navref.locate(goals, ORIGIN, m.resolution, box)
        assert st["goals_new"] == int(np.sum(ok & Tnew[tuple(v.T)] & ~Told[tuple(v.T)]))
        assert st["goals_placed"] == placed(m, D, box, goals, r, unk)
        if st["became_blocked"] + st["became_free"] == 0:
            assert st["seed_tiles"] == st["generations"] == st["tile_visits"] == st["withdraw_generations"] == 0
        if paths:
            check_paths(m, self.nav, want, box, starts_for(m, box, 400, rng, goals), 64)
        self.F = got
        return st

    def close(self):
        self.nav.close(); self.ref.close()


def cast(m, sc, p, yaw, kind):
    if kind == "lidar":
        pts, T = scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=360)
    else:
        pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
    m.RaycastFrame(pts, T, 0.3, 4.0)


@pytest.mark.parametrize("kind,mode,size", [("lidar", "exact", "gz32"), ("depth", "fast", "gz32"), ("lidar", "fast", "gz30"),
                                            ("depth", "exact", "gz30")])
def test_update_follows_raycast_frames(kind, mode, size):
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZES[size], mode=mode)
    m.size_m = SIZES[size]
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    poses = scenes.pose_walk(8, seed=2, clamp=0.5)
    p, yaw = poses[0]
    cast(m, sc, p, yaw, kind)
    m.UpdateOccupancy(True); m.UpdateESDF()
    gx, gy, gz = m.grid_size
    rng = np.random.default_rng(7)
    tracked = []
    for box, r, unk in [(((0, 0, 0), (gx - 1, gy - 1, gz - 1)), RES, False),          # the whole grid
                        (((10, 12, 3), (50, 47, gz - 5)), 2.5 * RES, True),          # a local box, unknown space blocking
                        (((0, 5, 0), (gx - 1, 40, gz - 1)), 0.0, False)]:            # touches the x and z faces
        tracked.append(Tracked(m, box, goal_positions(m, box, 4, rng), r, unk))
    totals = {}
    for f, (p, yaw) in enumerate(poses[1:]):                                         # 7 chained frames, no compute in between
        for _ in range(3):
            sc.step()
        cast(m, sc, p, yaw, kind)
        if m.CheckUpdate():
            m.UpdateOccupancy(True)
            m.UpdateESDF()
        for i, t in enumerate(tracked):
            st = t.check(paths=(f % 3 == 0 and i < 2), rng=rng)
            for k in ("became_blocked", "became_free", "withdrawn"):
                totals[(i, k)] = totals.get((i, k), 0) + st[k]
    assert all(totals[(i, "became_blocked")] + totals[(i, "became_free")] > 0 for i in range(3)), totals
    assert sum(totals[(i, "withdrawn")] for i in range(3)) > 0, totals
    assert totals[(1, "became_free")] > 0                                            # newly observed voxels, unknown flag on
    for t in tracked:
        t.close()


def test_single_voxel_edits_on_the_maze():
    m = maze_map()
    gs = m.grid_size
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    centre = lambda v: np.asarray(ORIGIN) + (np.asarray(v) + 0.5) * RES
    goals = centre([[1, 0, 5], [60, 40, 3]])
    t = Tracked(m, box, goals, 0.0, False)
    rng = np.random.default_rng(4)

    def edit(vox, occ):
        vox = np.asarray(vox, np.int32).reshape(-1, 3)
        m.SetOccupancyBatchVox(vox, np.full(len(vox), occ, np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
        return t.check(paths=True, rng=rng)

    door = [(40, 5, z) for z in range(gs[2])]                                          # in the second wall (y = 5)
    st = edit(door, 0)
    assert st["became_free"] == len(door) and st["withdrawn"] == 0
    st = edit(door, 1)
    assert st["became_blocked"] == len(door) and st["withdrawn"] > 0
    st = edit([(1, 0, 5)], 1)                                                            # block a goal voxel ...
    assert st["goals_placed"] == 1 and st["withdrawn"] > 0
    st = edit([(1, 0, 5)], 0)                                                            # ... and free it again
    assert st["goals_placed"] == 2 and st["goals_new"] == 1
    st = t.check()                                                                       # nothing changed since
    assert st["became_blocked"] == st["became_free"] == st["withdrawn"] == 0
    assert st["generations"] == st["tile_visits"] == st["seed_tiles"] == 0
    t.close()


def test_freed_voxel_opens_a_diagonal_gap():
    """Two corridors touch only diagonally across a tile corner; freeing one voxel of the 2x2 between them allows the diagonal
    move between two unchanged voxels (tests/test_nav_update_oracle.py's case, written with SetOccupancyBatchVox)."""
    import fiesta_b200
    gs, res = (17, 17, 3), 0.125
    size = tuple(g * res for g in gs)
    m = fiesta_b200.ESDFMap(ORIGIN, res, size, mode="fast")
    m.size_m = size
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    free = np.zeros(gs, bool)
    free[:8, 7, 1] = True
    free[8, 8:, 1] = True
    allv = scenes.all_voxels(gs)
    m.SetOccupancyBatchVox(allv, (~free[tuple(allv.T)]).astype(np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    t = Tracked(m, box, (np.asarray(ORIGIN) + (np.array([0, 7, 1]) + 0.5) * res)[None], 0.0, False)
    assert t.F[8, 16, 1] == np.inf
    m.SetOccupancyBatchVox(np.array([[8, 7, 1]], np.int32), np.zeros(1, np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    st = t.check()
    assert st["became_free"] == 1 and np.isfinite(t.F[8, 16, 1])
    m.SetOccupancyBatchVox(np.array([[8, 7, 1]], np.int32), np.ones(1, np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    st = t.check()
    assert st["became_blocked"] == 1 and t.F[8, 16, 1] == np.inf and st["withdrawn"] == 9
    t.close()


def test_local_map_reset():
    import fiesta_b200
    size = SIZES["gz30"]
    m = fiesta_b200.ESDFMap(ORIGIN, RES, size, mode="fast")
    m.size_m = size
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=6, edge=(0.3, 0.8))
    poses = scenes.pose_walk(6, seed=5, clamp=0.5)
    cast(m, sc, *poses[0], "depth")
    m.UpdateOccupancy(True); m.UpdateESDF()
    gx, gy, gz = m.grid_size
    rng = np.random.default_rng(2)
    box = ((4, 4, 2), (gx - 5, gy - 5, gz - 3))
    t = Tracked(m, box, goal_positions(m, box, 3, rng), RES, True)
    radius = np.array([1.2, 1.2, 0.8])
    changed = 0
    for p, yaw in poses[1:]:
        for _ in range(3):
            sc.step()
        cast(m, sc, p, yaw, "depth")
        m.SetUpdateRange(tuple(p - radius), tuple(p + radius))                       # a new local box: the map outside it resets
        m.UpdateOccupancy(False); m.UpdateESDF()
        st = t.check(paths=True, rng=rng)
        changed += st["became_blocked"] + st["became_free"]
    assert changed > 0
    t.close()


def test_matrix_other_box_and_invalid_calls():
    import fiesta_b200
    from tests.test_gpu_nav import raycast_map
    m, _ = raycast_map("exact", "lidar", SIZES["gz30"], frames=2)
    L = m._L
    gs = m.grid_size
    rng = np.random.default_rng(9)
    # update before any compute: FIESTA_ERR_INVALID, nothing changes
    fresh = m.NavField()
    st = fiesta_b200.NavUpdateStats()
    assert L.fiesta_nav_update(fresh._h, C.byref(st)) == 1 and L.fiesta_nav_update(None, None) == 1
    with pytest.raises(fiesta_b200.FiestaError):
        fresh.update()
    assert L.fiesta_nav_export(fresh._h, np.empty(10).ctypes) == 1
    fresh.close()
    box = ((4, 7, 1), (49, 55, 26))
    goals = goal_positions(m, box, 5, rng)
    t = Tracked(m, box, goals, RES, False)
    D0, O0, S0 = m.export_distance(), m.export_occupancy(), m.stats()
    # a matrix between compute and update changes neither
    src = goal_positions(m, box, 3, rng)
    cost, _, _, _ = t.nav.matrix(box[0], box[1], src, goals, RES)
    assert np.array_equal(t.nav.export(), t.F)
    st = t.check()
    assert st["became_blocked"] == st["became_free"] == 0 and st["generations"] == 0 and np.array_equal(t.F, t.nav.export())
    cost2, _, _, _ = t.nav.matrix(box[0], box[1], src, goals, RES)
    assert np.array_equal(cost, cost2, equal_nan=True)
    # the map is untouched, apart from the launch counter
    S1 = m.stats()
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert {k: v for k, v in S0.items() if k != "kernel_launches"} == {k: v for k, v in S1.items() if k != "kernel_launches"}
    assert S1["kernel_launches"] > S0["kernel_launches"]
    # a compute on a different box, then map changes and an update: the new box, goals, clearance and flags are the ones kept
    box2 = ((0, 0, 0), (gs[0] - 1, 40, gs[2] - 1))
    t.box, t.goals, t.r, t.unk = box2, goal_positions(m, box2, 2, rng), 0.0, True
    t.nav.compute(box2[0], box2[1], t.goals, 0.0, unknown_blocks=True)
    t.F = t.nav.export()
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=4, edge=(0.3, 0.8))
    for _ in range(4):
        sc.step()
    cast(m, sc, np.array([0.4, -0.3, 0.1]), 0.7, "lidar")
    m.UpdateOccupancy(True); m.UpdateESDF()
    st = t.check(paths=True, rng=rng)
    assert st["became_blocked"] + st["became_free"] > 0
    t.close()


def test_stats_struct_matches_header():
    import fiesta_b200
    assert C.sizeof(fiesta_b200.NavUpdateStats) == 12 * 8 + 2 * 4
