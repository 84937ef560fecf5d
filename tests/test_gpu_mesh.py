"""GPU: surface meshes (fiesta_mesh_*) against tests/meshref.py evaluated on export_distance() and export_closest_obstacle() of the same
map -- vertices (bit for bit), triangles and stats with np.array_equal -- on ray-cast maps in both modes over the whole grid, local
boxes, boxes on the grid's faces and a 1-voxel box, at clearances 0, 0.5 res, res (crossings at t = 0) and 2.5 res with both flag
settings; on crafted solids whose surfaces span many 32-voxel bitmap words and 8^3 tiles; under an EXACT local-map reset, whose
records block nowhere and have no distance.  Also: determinism, isolation from the map, cap truncation, save_ply read back and
every argument error."""
import ctypes as C
import itertools

import numpy as np
import pytest

import fiesta_b200
from tests import meshref, scenes
from tests.test_gpu_frontier import crafted_map
from tests.test_gpu_nav import ORIGIN, RES, SIZES, raycast_map
from tests.test_gpu_skeleton import crafted, grid_boxes

pytestmark = pytest.mark.gpu

STATS = ("box_voxels", "blocking", "vertices", "quads", "triangles")


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check(m, me, box, r, unk, D=None, O=None):
    """Compute on the device and compare every output with meshref; returns the expected dict."""
    D = m.export_distance() if D is None else D
    O = m.export_closest_obstacle() if O is None else O
    st = me.compute(box[0], box[1], r, unknown_blocks=unk)
    want = meshref.mesh(D, O, m.grid_size, box, r, unk, m.resolution, m.origin)
    ctx = (box, r, unk)
    assert {k: st[k] for k in STATS} == want["stats"], (ctx, st, want["stats"])
    assert same_bits(me.vertices(), want["vertices"]), ctx
    assert np.array_equal(me.triangles(), want["triangles"]) and me.triangles().dtype == np.int32, ctx
    return want


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_raycast_maps(kind, mode, size):
    m, _ = raycast_map(mode, kind, SIZES[size])
    me = m.Mesh()
    D, O = m.export_distance(), m.export_closest_obstacle()
    tris = 0
    for box in grid_boxes(m.grid_size):
        for r, unk in itertools.product((0.0, 0.5 * RES, RES, 2.5 * RES), (False, True)):
            tris += check(m, me, box, r, unk, D, O)["stats"]["triangles"]
    assert tris > 0
    me.close()


def solids():
    """Crafted obstacle sets on a grid whose z extent spans three bitmap words and whose boxes cross many 8^3 tiles."""
    gs = (44, 40, 70)
    out = {}
    o = np.zeros(gs, bool)
    o[20, 20, 35] = True
    out["one_voxel"] = o
    o = np.zeros(gs, bool)
    o[3:12, 4:30, 2:66] = True
    o[25:40, 20:36, 30:34] = True
    out["two_solids"] = o
    o = np.zeros(gs, bool)
    o[5:39, 5:35, 28:40] = True
    o[12:32, 12:28, 28:40] = False
    out["ring"] = o
    o = np.zeros(gs, bool)
    o[4:40, 4:36, 3:67] = True
    o[10:34, 10:30, 20:50] = False
    out["hollow_shell"] = o
    o = np.zeros(gs, bool)
    o[10, 10, 31] = o[11, 11, 31] = o[12, 12, 32] = True                    # edge and corner contacts across a word boundary
    out["contacts"] = o
    c = np.moveaxis(np.indices(gs), 0, -1) - np.array([22, 20, 33])
    out["ball"] = np.einsum("...i,...i", c, c) <= 15 ** 2
    return gs, out


@pytest.mark.parametrize("case", ["one_voxel", "two_solids", "ring", "hollow_shell", "contacts", "ball"])
def test_crafted_solids(case):
    gs, cases = solids()
    m = crafted(gs, cases[case])
    me = m.Mesh()
    res = m.resolution
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    for r in (0.0, 0.5 * res, res, 2.5 * res):
        w = check(m, me, full, r, False)
    check(m, me, ((3, 5, 2), (41, 33, 68)), 0.5 * res, False)            # off the tile lattice, through the solids
    check(m, me, ((0, 0, 31), (43, 39, 32)), 0.0, True)                   # two z-layers around the first word boundary
    if case == "one_voxel":
        st = check(m, me, full, 0.5 * res, False)["stats"]
        assert st["vertices"] == 8 and st["triangles"] == 12
    me.close()


def test_empty_and_all_blocking():
    gs = (24, 24, 40)
    m = crafted_map(gs, [])                                                 # nothing observed
    me = m.Mesh()
    full = ((0, 0, 0), tuple(g - 1 for g in gs))
    assert check(m, me, full, 0.0, False)["stats"]["triangles"] == 0
    assert me.vertices().shape == (0, 3) and me.triangles().shape == (0, 3)
    w = check(m, me, ((2, 3, 4), (20, 21, 37)), 0.0, True)                 # unknown blocks: the box's boundary
    assert w["stats"]["quads"] == 2 * (19 * 19 + 19 * 34 + 19 * 34)
    w = check(m, me, ((5, 6, 7), (5, 6, 7)), 0.0, True)                    # a 1-voxel box
    assert w["stats"]["vertices"] == 8 and w["stats"]["triangles"] == 12
    me.close()


def test_exact_local_map_reset_records_block_nowhere():
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
    dinf = (D == 10000) & (O[:, 0] >= 0)
    assert dinf.any(), "no local-map reset voxel"
    me = m.Mesh()
    full = grid_boxes(m.grid_size)[0]
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            check(m, me, full, r, unk, D, O)
            blk, has, _ = meshref.from_records(D, O, m.grid_size, full, r, unk)
            assert not np.any(blk.reshape(-1)[dinf]) and not np.any(has.reshape(-1)[dinf])
    m.UpdateESDF()
    check(m, me, full, RES, False)
    me.close()


def test_determinism_isolation_cap_and_ply(tmp_path):
    m, _ = raycast_map("fast", "lidar", SIZES["gz32"])
    D, O, occ = m.export_distance(), m.export_closest_obstacle(), m.export_occupancy()
    me = m.Mesh()
    full = grid_boxes(m.grid_size)[0]
    w = check(m, me, full, RES, False, D, O)
    for _ in range(3):
        me.compute(full[0], full[1], RES)
        assert same_bits(me.vertices(), w["vertices"]) and np.array_equal(me.triangles(), w["triangles"])
    assert np.array_equal(m.export_distance(), D) and np.array_equal(m.export_closest_obstacle(), O)
    assert np.array_equal(m.export_occupancy(), occ)
    V, T = w["stats"]["vertices"], w["stats"]["triangles"]
    assert V > 3 and T > 3
    for cap in (0, 1, 3):
        assert same_bits(me.vertices(cap), w["vertices"][:cap]) and np.array_equal(me.triangles(cap), w["triangles"][:cap])
    L = m._L
    big = np.full((V + 5) * 3, -7.0, np.float32)
    assert L.fiesta_mesh_vertices(me._h, C.c_int64(V + 5), big.ctypes) == 0
    assert same_bits(big[:3 * V].reshape(-1, 3), w["vertices"]) and np.all(big[3 * V:] == -7)
    big = np.full((T + 5) * 3, -7, np.int32)
    assert L.fiesta_mesh_triangles(me._h, C.c_int64(T + 5), big.ctypes) == 0
    assert np.array_equal(big[:3 * T].reshape(-1, 3), w["triangles"]) and np.all(big[3 * T:] == -7)
    # PLY read back
    path = tmp_path / "mesh.ply"
    me.save_ply(str(path))
    data = path.read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    assert "element vertex %d" % V in head and "element face %d" % T in head
    assert "property list uchar int vertex_indices" in head
    body = data[end:]
    v = np.frombuffer(body[:12 * V], "<f4").reshape(-1, 3)
    f = np.frombuffer(body[12 * V:], dtype=[("n", "u1"), ("ijk", "<i4", (3,))])
    assert same_bits(v.copy(), w["vertices"]) and len(f) == T and np.all(f["n"] == 3) and np.array_equal(f["ijk"], w["triangles"])
    me.close()


def test_invalid_arguments_change_nothing():
    m, _ = raycast_map("exact", "lidar", SIZES["gz32"], frames=2)
    L = m._L
    gs = m.grid_size
    fresh = m.Mesh()
    fbuf = np.zeros(64, np.float32)
    ibuf = np.zeros(64, np.int32)
    for call in (lambda: L.fiesta_mesh_vertices(fresh._h, C.c_int64(1), fbuf.ctypes),
                 lambda: L.fiesta_mesh_triangles(fresh._h, C.c_int64(1), ibuf.ctypes)):
        assert call() == 1                                                  # FIESTA_ERR_INVALID
        assert b"no mesh has been computed" in L.fiesta_last_error()
    with pytest.raises(fiesta_b200.FiestaError):
        fresh.vertices()
    fresh.close()
    me = m.Mesh()
    lo, hi = np.zeros(3, np.int32), np.asarray(gs, np.int32) - 1
    w = check(m, me, ((0, 0, 0), tuple(hi)), RES, False)
    before = (me.vertices(), me.triangles(), dict(me.stats))

    def compute(blo=lo, bhi=hi, r=RES, flags=0, null=None):
        a, b = np.ascontiguousarray(blo, np.int32), np.ascontiguousarray(bhi, np.int32)
        st = fiesta_b200.MeshStats()
        args = [me._h, a.ctypes, b.ctypes]
        if null is not None:
            args[null] = None
        return L.fiesta_mesh_compute(*args, C.c_double(r), flags, C.byref(st))

    bad = [dict(blo=(-1, 0, 0)), dict(bhi=(gs[0], 5, 5)), dict(bhi=(5, gs[1], 5)), dict(bhi=(5, 5, gs[2])),
           dict(blo=(5, 5, 5), bhi=(4, 9, 9)), dict(r=float("nan")), dict(r=-0.1), dict(r=1e4), dict(r=float("inf")),
           dict(flags=4), dict(flags=-1), dict(null=0), dict(null=1), dict(null=2)]
    for kw in bad:
        assert compute(**kw) == 1, kw                                       # FIESTA_ERR_INVALID
        assert L.fiesta_last_error()
    for call in (lambda: L.fiesta_mesh_vertices(me._h, C.c_int64(-1), fbuf.ctypes),
                 lambda: L.fiesta_mesh_vertices(me._h, C.c_int64(1), None),
                 lambda: L.fiesta_mesh_vertices(None, C.c_int64(1), fbuf.ctypes),
                 lambda: L.fiesta_mesh_triangles(me._h, C.c_int64(-2), ibuf.ctypes),
                 lambda: L.fiesta_mesh_triangles(me._h, C.c_int64(1), None),
                 lambda: L.fiesta_mesh_triangles(None, C.c_int64(1), ibuf.ctypes)):
        assert call() == 1
    assert np.all(fbuf == 0) and np.all(ibuf == 0)
    assert L.fiesta_mesh_vertices(me._h, C.c_int64(0), None) == 0 and L.fiesta_mesh_triangles(me._h, C.c_int64(0), None) == 0
    assert same_bits(me.vertices(), before[0]) and np.array_equal(me.triangles(), before[1])
    with pytest.raises(fiesta_b200.FiestaError):
        me.compute((0, 0, 0), (gs[0], 0, 0))
    assert me.stats == before[2] and same_bits(me.vertices(), before[0])  # an invalid compute keeps the last result
    assert compute(r=0.0) == 0 and compute(r=np.nextafter(1e4, 0)) == 0     # the edges of the valid range
    assert L.fiesta_mesh_create(None, C.byref(C.c_void_p())) == 1
    assert w["stats"]["triangles"] > 0
    me.close()
