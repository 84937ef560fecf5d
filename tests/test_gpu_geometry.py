"""GPU: every kernel on grid shapes at the library's limits -- degenerate and one-voxel-thick grids, gy == 1 (the divisor-1
branch of k_x_relax's index decode), grids smaller than a tile or than the +-2 reach of dirs_, padded z pitch (Pz != Gz),
off-tile shapes and the maximal extents 2046 x 1024 x 1024, where the packed closest-obstacle code has bit 30 set.

EXACT maps are compared with the reference after every update (arrays and expansions), FAST maps with the CPU model
(oracle/fast_model.c) bit for bit and with the reference's occupancy and counters.  Point queries, the host mirror, segment
clearance, the nav field and frontier extraction are compared with their CPU definitions on the same shapes.  The resolution
is dyadic so that ceil(size / res) is exact."""
import numpy as np
import pytest

from tests import frontierref, navref, scenes, segref
from tests.geometry import ORIGIN, RES, SHAPES, logit, random_voxels, shape_id, size_of, special_voxels, trilinear
from tests.parity import compare, invariants

pytestmark = pytest.mark.gpu

LONG = 1000             # an axis at least this long is crossed end to end by one wave
MIRRORED = [(2046, 3, 2), (3, 2, 1024)]                                   # host mirror + EXACT local-map loop


def same_counters(dev, ora):
    (h1, t1), (h2, t2) = dev.export_counters(), ora.export_counters()
    return np.array_equal(h1, h2) and np.array_equal(t1, t2)


class Pair:
    """A device map and the reference driven with the same inputs; FAST maps also drive the CPU model from the device's
    occupancy state (as tests/test_gpu_fast_model.py does) while the update box is the whole grid."""

    def __init__(self, oracle_built, gs, mode, params=scenes.PARAMS_TOGGLE):
        import fiesta_b200
        self.gs, self.mode, self.params = gs, mode, params
        self.dev = fiesta_b200.ESDFMap(ORIGIN, RES, size_of(gs), mode=mode)
        self.ora = oracle_built.OracleMap(ORIGIN, RES, size_of(gs))
        assert self.dev.grid_size == self.ora.grid_size == gs
        for m in (self.dev, self.ora):
            m.SetParameters(*params)
        self.model = oracle_built.FastModel(gs, RES, logit(params[4])) if mode == "fast" else None
        self.full_box = True
        self.updates = 0
        self.mirror = None                     # a Mirror, checked after every update when set

    def both(self, name, *args):
        return [getattr(m, name)(*args) for m in (self.dev, self.ora)]

    def events(self, vox, occ):
        a, b = self.both("SetOccupancyBatchVox", vox, occ)
        assert np.array_equal(a, b)

    def update(self, tag, global_map=True):
        dev, ora = self.dev, self.ora
        assert same_counters(dev, ora), tag
        c = dev.CheckUpdate()
        assert c == ora.CheckUpdate(), tag
        if not c:
            return False
        assert dev.UpdateOccupancy(global_map) == ora.UpdateOccupancy(global_map), tag
        st = None
        if self.model is not None and self.full_box:
            st = self.model.update(dev.export_distance(), dev.export_occupancy())
        dev.UpdateESDF(); ora.UpdateESDF()
        self.updates += 1
        self.check(tag, st)
        if self.mirror:
            self.mirror.check(tag)
        return True

    def check(self, tag, st=None):
        dev, ora = self.dev, self.ora
        r = compare(dev, ora, check_counters=True)
        assert r["occ"] == 0 and r["counters"] == 0, (tag, r)
        if self.mode == "exact":
            assert r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0, (tag, r)
            assert dev.stats()["expansions"] == ora.stats()["expansions"], tag
            return
        inv = invariants(dev, logit(self.params[4]))
        if not self.full_box:                     # the wave stays inside the box: the 24-neighbour check does not apply
            inv.pop("closer_occupied_neighbour")
        assert not any(inv.values()), (tag, inv)
        if st is not None:
            cobs, dist = self.model.export()
            D, C = dev.export_distance(), dev.export_closest_obstacle()
            assert np.array_equal(D, dist), (tag, int((D != dist).sum()))
            assert np.array_equal(C, cobs), (tag, int((C != cobs).any(axis=1).sum()))
            sd = dev.stats()
            assert sd["voxels_changed"] == st["changed"] and sd["generations"] == st["generations"], (tag, st, sd)


def check_point_queries(p, rng):
    """Voxel-form queries at the corners and outside the grid; trilinear queries against the CPU restatement everywhere and
    against the reference strictly inside."""
    dev, ora, gs = p.dev, p.ora, p.gs
    D = dev.export_distance().reshape(gs)
    O = dev.export_occupancy().reshape(gs) > logit(p.params[4])
    corners = [(x, y, z) for x in (0, gs[0] - 1) for y in (0, gs[1] - 1) for z in (0, gs[2] - 1)]
    for v in corners:
        d = dev.GetDistance(v)
        assert d == (10000.0 if D[v] < 0 else D[v]), v
        assert dev.GetOccupancy(v) == int(O[v]), v
        if p.mode == "exact":
            assert d == ora.GetDistance(v) and dev.GetOccupancy(v) == ora.GetOccupancy(v), v
    outside = [(-1, 0, 0), (0, -1, 0), (0, 0, -1), (gs[0], 0, 0), (0, gs[1], 0), (0, 0, gs[2]), (gs[0] - 1, gs[1] - 1, gs[2]),
               (gs[0], gs[1] - 1, gs[2] - 1), (gs[0] - 1, gs[1], gs[2] - 1), (2046, 1024, 1024), (-5, -5, -5)]
    for v in outside:
        assert dev.GetDistance(v) == 10000.0 and dev.GetOccupancy(v) == 0, v
    # trilinear queries everywhere, faces and outside the map included, against the CPU restatement on the exported field
    q = np.asarray(ORIGIN) + rng.uniform(-0.05, 1.05, (512, 3)) * np.asarray(size_of(gs))
    q[:8] = np.asarray(ORIGIN) + np.array(corners) * RES + np.array([0.5, 0.5, 0.5]) * RES
    q[8:16] = np.asarray(ORIGIN) + (np.array(corners) + 1) * RES                          # on the upper faces and corners
    d1, g1 = dev.GetDistWithGradTrilinearBatch(q)
    d2, g2, inside = trilinear(dev.export_distance(), gs, q)
    assert inside.sum() > 16 and np.array_equal(d1, d2), int((d1 != d2).sum())
    assert np.array_equal(g1[inside], g2[inside])
    if p.mode != "exact":
        return
    lo = np.asarray(ORIGIN) + RES
    hi = np.asarray(ORIGIN) + np.asarray(size_of(gs)) - 2 * RES
    q = np.asarray(ORIGIN) + rng.random((256, 3)) * np.asarray(size_of(gs))
    d1, g1 = dev.GetDistWithGradTrilinearBatch(q)
    d2, g2 = ora.GetDistWithGradTrilinearBatch(q)
    ok = np.all((q > lo) & (q < hi), axis=1) | (d2 == -1)
    assert np.array_equal(d1[ok], d2[ok]) and np.array_equal(g1[ok], g2[ok])
    for x in q[:8]:
        a, ga = dev.GetDistWithGradTrilinear(tuple(x))
        b, gb = ora.GetDistWithGradTrilinear(tuple(x))
        if np.all((x > lo) & (x < hi)) or b == -1:
            assert a == b and np.array_equal(ga, gb), x


def voxel_centres(gs):
    return (scenes.all_voxels(gs) + 0.5) * RES + np.asarray(ORIGIN)


class Mirror:
    """Host mirror refreshed after every update; its whole field must equal the device's voxel queries."""

    def __init__(self, dev):
        self.dev, self.mir = dev, dev.HostMirror()
        self.centres = voxel_centres(dev.grid_size)

    def check(self, tag):
        self.mir.refresh()
        D = self.dev.export_distance()
        want = np.where(D < 0, 10000.0, D)
        assert np.array_equal(self.mir.GetDistanceBatch(self.centres), want), tag
        assert np.array_equal(self.dev.GetDistanceBatch(self.centres), want), tag
        gs = self.dev.grid_size
        for v in [(gs[0] - 1, gs[1] - 1, gs[2] - 1), (0, 0, 0), (gs[0] - 1, 0, gs[2] - 1)]:
            assert self.mir.GetDistance(v) == self.dev.GetDistance(v), (tag, v)

    def close(self):
        self.mir.close()


def raycast_frame(p, rng):
    """One LIDAR-like frame from a sensor inside the grid (off the lattice planes); rays are clipped at 30 m, so no ray of
    any shape here reaches the reference's 1500-voxel limit."""
    gs = np.asarray(p.gs)
    sensor = np.asarray(ORIGIN) + (gs // 2 + 0.5) * RES + np.array([0.0137, -0.0211, 0.0093])
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = (d * rng.uniform(0.1, 40.0, (3000, 1))).astype(np.float32)
    T = scenes.body_transform(sensor, 0.0)
    a, b = p.both("RaycastFrame", pts, T, 0.3, 30.0)
    assert a == b
    assert p.dev.stats()["rays_dropped"] == p.ora.hung_rays()


def box_phase(p, rng, tag):
    """SetUpdateRange with a box whose faces are the grid's faces, then one clipped by them."""
    gs = p.gs
    lo, hi = np.asarray(ORIGIN), np.asarray(ORIGIN) + np.asarray(size_of(gs))
    mid = lo + (np.asarray(gs) // 2) * RES
    p.full_box = False
    for k, (a, b) in enumerate([(lo, hi), (lo - 3.0, mid + 0.5 * RES), (mid - 0.25 * RES, hi + 7.0)]):
        p.both("SetUpdateRange", tuple(a), tuple(b))
        vox = np.concatenate([special_voxels(gs), random_voxels(rng, gs, 200)])
        p.events(vox, (rng.random(len(vox)) < 0.5).astype(np.uint8))
        p.update((tag, "box", k))
    p.both("SetOriginalRange")


def local_map_loop(p, rng, tag):
    """The reference's local-map mode: a sliding box and UpdateOccupancy(false) (test_local_map_moving_box_exact)."""
    gs = p.gs
    allv = scenes.all_voxels(gs)
    idx = rng.choice(len(allv), max(1, len(allv) // 40), replace=False)
    p.events(allv, np.zeros(len(allv), np.uint8)); p.update((tag, "observe"))
    p.events(allv[idx], np.ones(len(idx), np.uint8)); p.update((tag, "obstacles"))
    p.both("SetParameters", *scenes.PARAMS_DEFAULT)
    p.params = scenes.PARAMS_DEFAULT
    p.full_box = False
    lo, size = np.asarray(ORIGIN), np.asarray(size_of(gs))
    seen_reset = 0
    for r in range(6):
        c = lo + size * (0.15 + 0.14 * r)
        half = size * 0.3
        p.both("SetUpdateRange", tuple(c - half), tuple(c + half))
        vox = random_voxels(rng, gs, 4000)
        p.events(vox, (rng.random(4000) < 0.4).astype(np.uint8))
        assert p.dev.UpdateOccupancy(False) == p.ora.UpdateOccupancy(False)
        r1 = compare(p.dev, p.ora)
        assert r1["occ"] == 0 and r1["dist"] == 0 and r1["cobs_tie"] == 0 and r1["cobs_nontie"] == 0, (tag, r, r1)
        p.dev.UpdateESDF(); p.ora.UpdateESDF()
        p.check((tag, "local", r))
        p.mirror.check((tag, "local", r))
        D, C = p.ora.export_distance(), p.ora.export_closest_obstacle()
        seen_reset += int(((D == 10000) & (C[:, 0] != -10000)).sum())       # FB_DINF records: infinity, obstacle kept
    assert seen_reset > 0
    p.both("SetOriginalRange")


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("gs", SHAPES, ids=shape_id)
def test_shape_equals_reference(oracle_built, gs, mode):
    si = SHAPES.index(gs)
    rng = np.random.default_rng(1000 + si)
    p = Pair(oracle_built, gs, mode)
    long_axes = [k for k in range(3) if gs[k] >= LONG]
    partial = si % 2 == 1 and not long_axes
    allv = scenes.all_voxels(gs)[rng.permutation(int(np.prod(gs)))]          # observed in a scrambled order
    if partial:
        allv = allv[rng.random(len(allv)) < 0.6]
    p.mirror = Mirror(p.dev) if gs in MIRRORED else None
    p.events(allv, np.zeros(len(allv), np.uint8))
    p.update("observe")
    spec = special_voxels(gs)
    n = min(600, 4 * int(np.prod(gs)))
    for r in range(4):
        vox = np.concatenate([random_voxels(rng, gs, n), spec[rng.random(len(spec)) < 0.5]])
        occ = (rng.random(len(vox)) < (0.7 if r < 2 else 0.4)).astype(np.uint8)
        p.events(vox, occ)
        p.update(("round", r))
    # the largest coordinate on every axis as an obstacle: the decoded code carries x = gx-1, y = gy-1, z = gz-1
    top = tuple(g - 1 for g in gs)
    p.events(np.array([top], np.int32), np.ones(1, np.uint8))
    p.update("top corner")
    C = p.dev.export_closest_obstacle().reshape(gs + (3,))
    assert tuple(C[top]) == top
    for k in long_axes:                     # one obstacle at each end of a long axis, nothing else: the wave crosses all of it
        occupied = np.flatnonzero(p.dev.export_occupancy() > logit(p.params[4]))
        p.events(scenes.all_voxels(gs)[occupied], np.zeros(len(occupied), np.uint8))
        p.update(("clear", k))
        ends = np.zeros((2, 3), np.int32)
        ends[1, k] = gs[k] - 1
        p.events(ends, np.ones(2, np.uint8))
        p.update(("ends", k))
        D = p.dev.export_distance().reshape(gs)
        line = np.zeros((gs[k], 3), int)
        line[:, k] = np.arange(gs[k])
        want = np.minimum(line[:, k], gs[k] - 1 - line[:, k]) * RES
        assert np.array_equal(D[tuple(line.T)], want), k
        p.events(ends, np.zeros(2, np.uint8))
        p.update(("ends deleted", k))
    raycast_frame(p, rng)
    p.update("raycast")
    check_point_queries(p, rng)
    box_phase(p, rng, "box")
    check_point_queries(p, rng)
    if p.mirror:
        if mode == "exact":
            local_map_loop(p, rng, "local map")
        p.mirror.close()
    assert p.updates >= 8


@pytest.mark.parametrize("gs,ok", [((2047, 1, 1), False), ((1, 1025, 1), False), ((1, 1, 1025), False),
                                   ((2046, 1, 1), True), ((1, 1024, 1), True), ((1, 1, 1024), True)], ids=lambda v: str(v))
def test_create_limits(gs, ok):
    import fiesta_b200
    for mode in ("exact", "fast"):
        if ok:
            m = fiesta_b200.ESDFMap(ORIGIN, RES, size_of(gs), mode=mode)
            assert m.grid_size == gs
            m.close()
        else:
            with pytest.raises(fiesta_b200.FiestaError, match="2046 x 1024 x 1024"):
                fiesta_b200.ESDFMap(ORIGIN, RES, size_of(gs), mode=mode)


# ---------------------------------------------------------------- planner kernels on the same shapes

PLANNER_SHAPES = [(1, 1, 1), (5, 1, 1), (37, 1, 29), (9, 1, 4), (2, 2, 2), (3, 3, 3), (2, 17, 3), (13, 11, 1), (13, 11, 3),
                  (13, 11, 5), (13, 11, 30), (17, 3, 28), (2046, 3, 2), (2046, 2, 5), (3, 2, 1024), (2, 1024, 3)]
FRONTIER_SHAPES = [(2046, 3, 2), (3, 2, 1024), (37, 1, 29), (9, 1, 4), (13, 11, 1), (13, 11, 3), (13, 11, 5)]


def planner_map(gs, mode, rng, hole_axis=None):
    """A map with random obstacles and a random 15 % of the voxels never observed; or, with `hole_axis`, a map without
    obstacles whose only unobserved voxels are the plane at index 1 of another axis, so that a frontier cluster spans the
    whole of `hole_axis`."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, size_of(gs), mode=mode)
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(gs)
    keep = rng.random(len(allv)) >= 0.15
    if hole_axis is not None:
        other = [k for k in range(3) if k != hole_axis]
        j = other[0] if gs[other[0]] > 1 else other[1]
        keep = allv[:, j] != min(1, gs[j] - 1)
    m.SetOccupancyBatchVox(allv[keep], np.zeros(int(keep.sum()), np.uint8))
    m.UpdateOccupancy(True); m.UpdateESDF()
    if hole_axis is not None:
        return m
    obs = allv[keep][rng.random(int(keep.sum())) < 0.04]
    m.SetOccupancyBatchVox(obs, np.ones(len(obs), np.uint8))
    m.UpdateOccupancy(True); m.UpdateESDF()
    return m


def segment_set(gs, rng):
    """Random segments, the adversarial set, and segments along every axis with an endpoint exactly on the upper face
    (the largest lattice value, 2046 * 2^20 along x)."""
    lo, hi = np.asarray(ORIGIN), np.asarray(ORIGIN) + np.asarray(size_of(gs))
    a = rng.uniform(lo, hi, (64, 3))
    b = rng.uniform(lo - 0.5, hi + 0.5, (64, 3))
    ab = [np.concatenate([a, b], 1)]
    ab.append(np.array([np.concatenate([lo + u[:3] * RES, lo + u[3:] * RES]) for u in segref.adversarial_voxel_units(gs, rng)]))
    axis = []
    for k in range(3):
        for off in (0.5, 0.0):
            s = lo + (np.asarray(gs) // 2 + off) * RES
            e = s.copy()
            s[k], e[k] = lo[k], hi[k]
            axis += [np.concatenate([s, e]), np.concatenate([e, s])]
            e2 = e.copy(); e2[k] = lo[k] + 0.375 * RES
            axis.append(np.concatenate([e, e2]))
    ab.append(np.array(axis))
    return np.ascontiguousarray(np.concatenate(ab))


def check_segments(m, ab):
    gs = m.grid_size
    lo, hi = np.asarray(ORIGIN), np.asarray(ORIGIN) + np.asarray(size_of(gs))
    D = m.export_distance().reshape(gs)
    walks = [segref.segment_walk(s, ORIGIN, RES, lo, hi) for s in ab]
    mir = m.HostMirror()
    mir.refresh()
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            rows = [segref.apply(w, D, r, unk) for w in walks]
            for got in (m.CheckSegments(ab, r, unknown_blocks=unk), mir.CheckSegments(ab, r, unknown_blocks=unk)):
                for i, want in enumerate(rows):
                    assert segref.same(tuple(x[i] for x in got), want), (r, unk, ab[i], tuple(x[i] for x in got), want)
    mir.close()


def check_nav(m, rng):
    gs = m.grid_size
    D = m.export_distance()
    Dg = D.reshape(gs)
    nav = m.NavField()
    free = np.argwhere(Dg > RES)
    lo = np.asarray(ORIGIN)
    boxes = [((0, 0, 0), tuple(g - 1 for g in gs)),
             (tuple(g // 3 for g in gs), tuple(g - 1 for g in gs)),                     # cut by the upper faces
             ((0, 0, 0), tuple(max(0, (2 * g) // 3 - 1) for g in gs))]                # cut by the lower faces
    for box in boxes:
        gv = free[rng.choice(len(free), min(3, len(free)), replace=False)] if len(free) else np.zeros((1, 3), int)
        goals = lo + (gv + 0.5) * RES                                                # voxel centres: Pos2Vox gives gv back
        for r, unk in ((0.0, False), (RES, True)):
            st = nav.compute(box[0], box[1], goals, r, unknown_blocks=unk)
            got = nav.export()
            want = navref.field(D, gs, box, gv, r, unk, RES)
            assert np.array_equal(got, want), (box, r, unk, int(np.sum(got != want)))
            assert st["box_voxels"] == want.size and st["reached"] == int(np.sum((want >= 0) & (want < np.inf)))
            blo = lo + np.asarray(box[0]) * RES
            bhi = lo + (np.asarray(box[1]) + 1) * RES
            starts = np.concatenate([rng.uniform(blo - 0.2, bhi + 0.2, (64, 3)), goals])
            max_len = int(sum(gs)) + 8
            gp = nav.paths(starts, max_len)
            v, ok = navref.locate(starts, ORIGIN, RES, box, lo, lo + np.asarray(size_of(gs)))
            wp = navref.paths(want, box, RES, v, ok, max_len)
            for name, a, b in zip(("status", "len", "cost", "vox"), gp, wp):
                assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=name == "cost"), (box, r, name)
    nav.close()


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("gs", PLANNER_SHAPES, ids=shape_id)
def test_planner_queries(gs, mode):
    rng = np.random.default_rng(7 + PLANNER_SHAPES.index(gs))
    m = planner_map(gs, mode, rng)
    check_segments(m, segment_set(gs, rng))
    check_nav(m, rng)
    m.close()


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("gs", FRONTIER_SHAPES, ids=shape_id)
def test_frontiers(gs, mode):
    rng = np.random.default_rng(31 + FRONTIER_SHAPES.index(gs))
    long_axis = int(np.argmax(gs))
    for hole in (None, long_axis):
        m = planner_map(gs, mode, rng, hole_axis=hole)
        D, O = m.export_distance(), m.export_occupancy()
        fr = m.Frontiers()
        full = ((0, 0, 0), tuple(g - 1 for g in gs))
        boxes = [full, (tuple(g // 3 for g in gs), full[1]), ((0, 0, 0), tuple(max(0, (2 * g) // 3 - 1) for g in gs))]
        for box in boxes:
            for r, min_size in ((0.0, 1), (RES, 3)):
                fr.compute(box[0], box[1], r, min_size)
                want = frontierref.extract(D, O, gs, box, r, frontierref.l_occ(scenes.PARAMS_TOGGLE[4]), min_size, RES, ORIGIN)
                assert {k: fr.stats[k] for k in want["stats"]} == want["stats"], (box, r, fr.stats, want["stats"])
                assert np.array_equal(fr.export(), want["labels"]), (box, r)
                got = fr.clusters()
                for k in ("size", "rep", "bbox_lo", "bbox_hi", "centroid"):
                    assert np.array_equal(got[k], want[k]), (k, box, r)
                assert np.array_equal(fr.voxels(), want["voxels"]), (box, r)
                if hole is not None and box == full and r == 0.0:
                    span = want["bbox_hi"][:, long_axis] - want["bbox_lo"][:, long_axis]
                    assert span.max() == gs[long_axis] - 1, span.max()           # one cluster spans the whole axis
        fr.close()
        m.close()
