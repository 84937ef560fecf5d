"""GPU: topological skeletons (fiesta_skeleton_*) against tests/skeletonref.py evaluated on export_distance() and
export_closest_obstacle() of the same map -- mask, labels, vertices, edges, edge voxels and stats with np.array_equal -- on ray-cast
maps in both modes over the whole grid, local boxes, boxes on the grid's faces and a 1-voxel box, for three clearances, both flag
settings, two max_cos values and min_branch 1 and 8; on crafted maps (a ring around a pillar, a floating cube, a straight tunnel, a
Y junction, a 2-voxel pocket, an empty and an all-blocked box) with chains across many 8-voxel tiles; under an EXACT local-map reset,
whose FB_DINF records are never anchors.  Also: determinism, isolation from the map, traversability in a cost-to-go field, cap
truncation and every argument error."""
import ctypes as C
import itertools

import numpy as np
import pytest

import fiesta_b200
from tests import scenes, skeletonref
from tests.test_gpu_frontier import crafted_map
from tests.test_gpu_nav import ORIGIN, RES, SIZES, boxes, raycast_map

pytestmark = pytest.mark.gpu


def check(m, sk, box, r, unk, max_cos, min_branch, D=None, O=None):
    """Compute on the device and compare every output with skeletonref; returns the expected dict."""
    D = m.export_distance() if D is None else D
    O = m.export_closest_obstacle() if O is None else O
    st = sk.compute(box[0], box[1], r, unknown_blocks=unk, max_cos=max_cos, min_branch=min_branch)
    want = skeletonref.skeleton(D, O, m.grid_size, box, r, unk, max_cos, min_branch, m.resolution, m.origin)
    ctx = (box, r, unk, max_cos, min_branch)
    assert {k: st[k] for k in want["stats"]} == want["stats"], (ctx, st, want["stats"])
    mask, lab = sk.export()
    assert np.array_equal(mask, want["mask"]), (ctx, int(np.sum(mask != want["mask"])))
    assert np.array_equal(lab, want["labels"]), ctx
    got = sk.vertices()
    for k in ("size", "rep", "centroid", "degree"):
        assert got[k].shape == want["vertices"][k].shape and np.array_equal(got[k], want["vertices"][k]), (k, ctx)
    got = sk.edges()
    for k in ("uv", "n_vox", "length", "min_dist"):
        assert got[k].shape == want["edges"][k].shape and np.array_equal(got[k], want["edges"][k]), (k, ctx)
    assert np.array_equal(sk.edge_voxels(), want["edge_voxels"]), ctx
    return want


def grid_boxes(gs):
    gx, gy, gz = gs
    return boxes(gs) + [((0, 0, gz - 1), (gx - 1, gy - 1, gz - 1)), ((gx - 1, 0, 0), (gx - 1, gy - 1, gz - 1)),
                        ((20, 30, 10), (20, 30, 10))]


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_raycast_maps(kind, mode, size):
    m, _ = raycast_map(mode, kind, SIZES[size])
    sk = m.Skeleton()
    D, O = m.export_distance(), m.export_closest_obstacle()
    gs = m.grid_size
    full = grid_boxes(gs)[0]
    edges = anchors = pruned = 0
    combos = list(itertools.product((0.0, RES, 2.5 * RES), (False, True), (0.5, -0.25), (1, 8)))
    if (kind, mode, size) != ("lidar", "exact", "gz32"):                     # every value on every map, every combination on one
        combos = [c for i, c in enumerate(combos) if i % 5 == 0]
    for r, unk, max_cos, mb in combos:
        w = check(m, sk, full, r, unk, max_cos, mb, D, O)
        edges += w["stats"]["edges"]
        anchors += w["stats"]["anchors"]
        pruned += w["stats"]["pruned_voxels"]
    for box in grid_boxes(gs)[1:]:
        for r, unk, max_cos, mb in ((RES, False, 0.5, 8), (0.0, True, -0.25, 1)):
            check(m, sk, box, r, unk, max_cos, mb, D, O)
    assert edges > 0 and anchors > 0 and pruned > 0
    sk.close()


def test_exact_local_map_reset_records_are_not_anchors():
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
    D, O = m.export_distance(), m.export_closest_obstacle()
    dinf = ((D == 10000) & (O[:, 0] >= 0)).reshape(m.grid_size)
    assert dinf.any(), "no local-map reset voxel"
    sk = m.Skeleton()
    full = grid_boxes(m.grid_size)[0]
    for r in (0.0, RES):
        for mb in (1, 8):
            check(m, sk, full, r, False, 0.5, mb, D, O)
            mask, _ = sk.export()
            assert np.all(mask[dinf] & skeletonref.TRAV) and not np.any(mask[dinf] & skeletonref.ANCHOR)
    m.UpdateESDF()
    check(m, sk, full, RES, False, 0.5, 8)
    sk.close()


def crafted(gs, obst):
    """A map whose voxels are all observed: `obst` (bool, grid-shaped) occupied, the rest free."""
    v = np.argwhere(np.ones(gs, bool))
    return crafted_map(gs, v[~obst.reshape(-1)], v[obst.reshape(-1)])


def crafted_cases():
    gs = (40, 40, 24)
    out = {}
    o = np.zeros(gs, bool)
    o[:, :, :11] = o[:, :, 12:] = True
    o[16:24, 16:24, :] = True
    out["ring"] = o                                                         # a one-voxel-thick slab around a pillar
    o = np.zeros(gs, bool)
    o[15:25, 15:25, 8:16] = True
    out["floating_cube"] = o
    o = np.ones(gs, bool)
    o[:, 18:21, 10:13] = False
    out["tunnel"] = o                                                       # along x through the whole box: 5 tiles
    o = np.ones(gs, bool)
    o[2:21, 19:21, 11:13] = False
    for t in range(19):
        o[20 + t:22 + t, 20 + t:22 + t, 11:13] = False
        o[20 + t:22 + t, 19 - t:21 - t, 11:13] = False
    out["y_junction"] = o
    o = np.zeros(gs, bool)
    o[:, :, 6:18] = True
    o[10, 10, 12:14] = False                                                # a 2-voxel pocket inside the wall
    out["pocket"] = o
    out["all_blocked"] = np.ones(gs, bool)
    return gs, out


@pytest.mark.parametrize("case", ["ring", "floating_cube", "tunnel", "y_junction", "pocket", "all_blocked"])
def test_crafted_maps(case):
    gs, cases = crafted_cases()
    m = crafted(gs, cases[case])
    sk = m.Skeleton()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    for max_cos in (0.5, -0.25):
        for mb in (1, 8):
            w = check(m, sk, full, 0.0, False, max_cos, mb)
    st = w["stats"]
    if case == "ring":
        assert st["vertices"] >= 1 and st["edges"] >= 1
    if case == "tunnel":
        assert st["edges"] >= 1 and max(w["edges"]["n_vox"]) >= 32
    if case == "pocket":
        mask, _ = sk.export()
        assert np.count_nonzero(mask[10, 10, 12:14] & skeletonref.SKEL) == 1    # thinned to one voxel, never removed
    if case == "all_blocked":
        assert st["traversable"] == 0 and st["skeleton_voxels"] == 0
    check(m, sk, ((3, 5, 2), (37, 33, 21)), 0.0, False, 0.5, 8)            # the same map through a box off the tile lattice
    sk.close()


def test_empty_map_and_single_voxel_box():
    gs = (24, 24, 16)
    m = crafted_map(gs, [])                                                 # nothing observed: no obstacle anywhere
    sk = m.Skeleton()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    w = check(m, sk, full, 0.0, False, 0.5, 8)
    assert w["stats"]["anchors"] == 0 and w["stats"]["skeleton_voxels"] == 1
    w = check(m, sk, full, 0.0, True, 0.5, 8)
    assert w["stats"]["traversable"] == 0
    w = check(m, sk, ((5, 6, 7), (5, 6, 7)), 0.0, False, 0.5, 8)
    assert w["stats"]["skeleton_voxels"] == 1 and w["stats"]["vertices"] == 1
    sk.close()


def test_determinism_isolation_nav_and_cap():
    m, _ = raycast_map("fast", "lidar", SIZES["gz32"])
    D, O, occ = m.export_distance(), m.export_closest_obstacle(), m.export_occupancy()
    sk = m.Skeleton()
    full = grid_boxes(m.grid_size)[0]
    r = RES
    w = check(m, sk, full, r, False, 0.5, 8, D, O)
    a = (sk.export(), sk.vertices(), sk.edges(), sk.edge_voxels())
    for _ in range(2):
        sk.compute(full[0], full[1], r, max_cos=0.5, min_branch=8)
        b = (sk.export(), sk.vertices(), sk.edges(), sk.edge_voxels())
        assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))
        for k in a[1]:
            assert np.array_equal(a[1][k], b[1][k])
        for k in a[2]:
            assert np.array_equal(a[2][k], b[2][k])
        assert np.array_equal(a[3], b[3])
    assert np.array_equal(m.export_distance(), D) and np.array_equal(m.export_closest_obstacle(), O)
    assert np.array_equal(m.export_occupancy(), occ)
    # every skeleton voxel is traversable in a cost-to-go field at the same clearance
    nav = m.NavField()
    goal = np.asarray(ORIGIN) + (np.argwhere(w["mask"] & skeletonref.SKEL)[0] + 0.5) * m.resolution
    nav.compute(full[0], full[1], goal[None], r)
    F = nav.export()
    assert np.all(F[(w["mask"] & skeletonref.SKEL) != 0] >= 0)
    nav.close()
    # cap truncation
    V, E, P = w["stats"]["vertices"], w["stats"]["edges"], w["stats"]["edge_voxels"]
    assert V > 3 and E > 3
    for cap in (0, 1, 3):
        v = sk.vertices(cap)
        assert all(np.array_equal(v[k], w["vertices"][k][:cap]) for k in v)
        e = sk.edges(cap)
        assert all(np.array_equal(e[k], w["edges"][k][:cap]) for k in e)
        assert np.array_equal(sk.edge_voxels(cap), w["edge_voxels"][:cap])
    assert np.array_equal(sk.edge_voxels(P + 10), w["edge_voxels"])
    L = m._L
    big = np.full((P + 5) * 3, -7, np.int32)
    assert L.fiesta_skeleton_edge_voxels(sk._h, C.c_int64(P + 5), big.ctypes) == 0
    assert np.array_equal(big[:3 * P].reshape(-1, 3), w["edge_voxels"]) and np.all(big[3 * P:] == -7)
    # export with one pointer null
    mask = np.zeros(w["mask"].shape, np.uint8)
    assert L.fiesta_skeleton_export(sk._h, mask.ctypes, None) == 0 and np.array_equal(mask, w["mask"])
    lab = np.zeros(w["labels"].shape, np.int32)
    assert L.fiesta_skeleton_export(sk._h, None, lab.ctypes) == 0 and np.array_equal(lab, w["labels"])
    sk.close()


def test_invalid_arguments_change_nothing():
    m, _ = raycast_map("exact", "lidar", SIZES["gz32"], frames=2)
    L = m._L
    gs = m.grid_size
    sk = m.Skeleton()
    lo, hi = np.zeros(3, np.int32), np.asarray(gs, np.int32) - 1
    fresh = m.Skeleton()
    buf = np.zeros(64, np.int64)
    for call in (lambda: L.fiesta_skeleton_vertices(fresh._h, C.c_int64(1), *[buf.ctypes] * 4),
                 lambda: L.fiesta_skeleton_edges(fresh._h, C.c_int64(1), *[buf.ctypes] * 4),
                 lambda: L.fiesta_skeleton_edge_voxels(fresh._h, C.c_int64(1), buf.ctypes),
                 lambda: L.fiesta_skeleton_export(fresh._h, buf.ctypes, None)):
        assert call() == 1                                                  # FIESTA_ERR_INVALID
        assert b"no skeleton has been computed" in L.fiesta_last_error()
    fresh.close()
    w = check(m, sk, ((0, 0, 0), tuple(hi)), RES, False, 0.5, 8)
    before = (sk.export(), sk.vertices(), sk.edges(), sk.edge_voxels(), dict(sk.stats))

    def compute(blo=lo, bhi=hi, r=RES, flags=0, max_cos=0.5, mb=8, null=False):
        a, b = np.ascontiguousarray(blo, np.int32), np.ascontiguousarray(bhi, np.int32)
        stats = fiesta_b200.SkeletonStats()
        return L.fiesta_skeleton_compute(None if null else sk._h, a.ctypes, b.ctypes, C.c_double(r), flags, C.c_double(max_cos),
                                         C.c_int64(mb), C.byref(stats))

    bad = [dict(blo=(-1, 0, 0)), dict(bhi=(gs[0], 5, 5)), dict(blo=(5, 5, 5), bhi=(4, 9, 9)), dict(r=float("nan")), dict(r=-0.1),
           dict(r=1e4), dict(flags=4), dict(flags=-1), dict(max_cos=float("nan")), dict(max_cos=1.0), dict(max_cos=-1.0000001),
           dict(max_cos=float("inf")), dict(mb=-1), dict(null=True)]
    for kw in bad:
        assert compute(**kw) == 1, kw                                       # FIESTA_ERR_INVALID
        assert L.fiesta_last_error()
    assert compute(max_cos=-1.0, mb=0) == 0                                 # the edges of the valid ranges
    assert sk.stats is not None
    sk.compute(lo, hi, RES, max_cos=0.5, min_branch=8)
    buf = np.full(16, 123, np.int64)
    for call in (lambda: L.fiesta_skeleton_vertices(sk._h, C.c_int64(-1), *[buf.ctypes] * 4),
                 lambda: L.fiesta_skeleton_vertices(sk._h, C.c_int64(1), None, buf.ctypes, buf.ctypes, buf.ctypes),
                 lambda: L.fiesta_skeleton_edges(sk._h, C.c_int64(1), buf.ctypes, None, buf.ctypes, buf.ctypes),
                 lambda: L.fiesta_skeleton_edges(sk._h, C.c_int64(-2), *[buf.ctypes] * 4),
                 lambda: L.fiesta_skeleton_edge_voxels(sk._h, C.c_int64(1), None),
                 lambda: L.fiesta_skeleton_edge_voxels(sk._h, C.c_int64(-1), buf.ctypes),
                 lambda: L.fiesta_skeleton_export(None, buf.ctypes, None)):
        assert call() == 1
        assert np.all(buf == 123)
    assert L.fiesta_skeleton_vertices(sk._h, C.c_int64(0), None, None, None, None) == 0
    after = (sk.export(), sk.vertices(), sk.edges(), sk.edge_voxels())
    assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0]))
    for i in (1, 2):
        assert all(np.array_equal(before[i][k], after[i][k]) for k in before[i])
    assert np.array_equal(before[3], after[3])
    with pytest.raises(fiesta_b200.FiestaError):
        m.Skeleton().vertices()
    assert w["stats"]["vertices"] > 0
    sk.close()
