"""GPU: the signed field (fiesta_signed_*) against tests/signedref.py evaluated on export_distance() of the same map -- every export
bit for bit (int64 views, so -0.0 and +0.0 differ), every statistic, every query against the reference's trilinear expression on the
grid's values with the box overwritten by S -- on ray-cast maps in both modes, on the grid shapes at the library's limits with
synthetic obstacle layouts, and on a solid cube whose gradient must lead out.  Also: positions without an interior obstacle in their
stencil get the map query's bits, the device forms give the host forms' bits, and a field refuses to be read after the records
change until it is computed again; argument errors leave a valid field valid."""
import numpy as np
import pytest

from tests import scenes, signedref
from tests.geometry import ORIGIN as G_ORIGIN, RES as G_RES, SHAPES, shape_id, size_of

pytestmark = pytest.mark.gpu

INVALID = 1
ORIGIN, RES = (-3.2, -3.2, -1.6), 0.1
SIZES = {"gz32": (6.4, 6.4, 3.2), "gz30": (6.4, 6.4, 3.0)}     # Gz = 30: padded z pitch Pz = 32 != Gz


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def same_bits(a, b):
    """Bit equality, except that any NaN matches any NaN (0 * -inf on a box with no free voxel; payloads are not specified)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(nan | (bits(a) == bits(b))))


def raycast_map(mode, size, frames=4):
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, size, mode=mode)
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    for f, (p, yaw) in enumerate(scenes.pose_walk(frames, seed=2, clamp=0.5)):
        if f % 2 == 0:
            pts, T = scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=360)
        else:
            pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
        m.RaycastFrame(pts, T, 0.3, 4.0)
        if m.CheckUpdate():
            m.UpdateOccupancy(True)
            m.UpdateESDF()
        for _ in range(3):
            sc.step()
    return m


def check_field(m, sf, box, origin, res):
    """compute + export against signedref; returns (S, q, D)."""
    gs = m.grid_size
    D = m.export_distance()
    st = sf.compute(box[0], box[1])
    got = sf.export()
    S, q = signedref.field(D, gs, box, res)
    assert got.shape == S.shape
    assert np.array_equal(bits(got), bits(S)), (box, int(np.sum(bits(got) != bits(S))))
    want = signedref.stats(q)
    assert {k: st[k] for k in want} == want, (box, st, want)
    return S, q, D


def query_positions(gs, box, rng, origin, res, n=512):
    """Random positions in and around the map, on the box's faces, on voxel centres and on voxel faces inside the box."""
    o = np.asarray(origin)
    lo, hi = o, o + np.asarray(gs) * res
    blo, bhi = o + np.asarray(box[0]) * res, o + (np.asarray(box[1]) + 1) * res
    p = [rng.uniform(lo - 0.3, hi + 0.3, (n, 3)), rng.uniform(blo, bhi, (n, 3))]
    f = rng.uniform(blo, bhi, (n, 3))
    k = rng.integers(0, 3, n)
    f[np.arange(n), k] = np.where(rng.random(n) < 0.5, blo[k], bhi[k])      # on a face of the box
    p.append(f)
    v = np.stack([rng.integers(box[0][i], box[1][i] + 1, n) for i in range(3)], -1)
    p.append(o + (v + 0.5) * res)                                            # voxel centres
    p.append(o + v * res)                                                    # voxel corners
    return np.ascontiguousarray(np.concatenate(p))


def check_queries(m, sf, box, S, q, D, rng, origin, res, device=True):
    gs = m.grid_size
    pos = query_positions(gs, box, rng, origin, res)
    V = signedref.grid_values(D, gs, box, S)
    wd, wg, inside = signedref.trilinear(V, gs, pos, origin, res)
    d, g = sf.GetDistWithGradTrilinearBatch(pos)
    assert same_bits(d, wd), (box, int(np.sum(bits(d) != bits(wd))))
    assert same_bits(g[inside], wg[inside]) and np.all(g[~inside] == 0.0), box
    dd = sf.GetDistanceBatch(pos)
    assert same_bits(dd, signedref.distance(V, gs, pos, origin, res)), box
    # positions whose stencil holds no obstacle with q > 1 read exactly what the map's queries read
    Q = np.zeros(gs, np.int64)
    Q[signedref.box_slices(box)] = q
    idx = np.floor(((pos - 0.5 * res) - np.asarray(origin)) / res).astype(np.int64)
    deep = np.zeros(len(pos), bool)
    for c in [(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)]:
        v = idx + np.array(c)
        ok = np.all((v >= 0) & (v < np.asarray(gs)), axis=1)
        vc = np.where(ok[:, None], v, 0)
        deep |= ok & (Q[vc[:, 0], vc[:, 1], vc[:, 2]] > 1)
    md, mg = m.GetDistWithGradTrilinearBatch(pos)
    assert same_bits(d[~deep], md[~deep]) and same_bits(g[~deep], mg[~deep]), box
    vox = np.floor((pos - np.asarray(origin)) / res).astype(np.int64)
    okv = np.all((vox >= 0) & (vox < np.asarray(gs)), axis=1)
    vc = np.where(okv[:, None], vox, 0)
    shallow = ~(okv & (Q[vc[:, 0], vc[:, 1], vc[:, 2]] > 1))
    assert same_bits(dd[shallow], m.GetDistanceBatch(pos)[shallow]), box
    if device:
        import torch
        tp = torch.from_numpy(pos).cuda()
        td, tg = sf.GetDistWithGradTrilinearBatchDevice(tp)
        tdd = sf.GetDistanceBatchDevice(tp)
        torch.cuda.synchronize()
        assert same_bits(td.cpu().numpy(), d) and same_bits(tg.cpu().numpy(), g) and same_bits(tdd.cpu().numpy(), dd), box
    return int(np.sum(deep))


def raycast_boxes(gs):
    gx, gy, gz = gs
    return [((0, 0, 0), (gx - 1, gy - 1, gz - 1)),                  # the whole grid
            ((10, 12, 3), (50, 47, gz - 5)),                          # off the tile lattice
            ((5, 20, 0), (60, 20, gz - 1)),                           # one voxel thick in y
            ((30, 2, 4), (30, 60, 20)),                               # one voxel thick in x
            ((3, 4, 11), (62, 50, 11)),                               # one voxel thick in z
            ((0, 5, 0), (gx - 1, 40, gz - 1)),                        # touches the x and z faces
            ((3, 0, 1), (37, gy - 1, gz - 2))]                        # touches the y faces


@pytest.mark.parametrize("mode,size", [(m, s) for m in ("exact", "fast") for s in ("gz32", "gz30")])
def test_raycast_maps(mode, size):
    m = raycast_map(mode, SIZES[size])
    sf = m.SignedField()
    rng = np.random.default_rng(3)
    obstacles = 0
    for box in raycast_boxes(m.grid_size):
        S, q, D = check_field(m, sf, box, ORIGIN, RES)
        obstacles += int(np.sum(q > 0))
        check_queries(m, sf, box, S, q, D, rng, ORIGIN, RES)
    assert obstacles > 0
    sf.close()
    m.close()


# ---- grid shapes at the library's limits, synthetic layouts through SetOccupancy
LAYOUT_SHAPES = [s for s in SHAPES if s not in ((2046, 1024, 1), (1, 1024, 1024))] + [(40, 36, 30)]


def layout_map(gs, mode, layout, rng):
    """All voxels observed free (10 % never observed, except for 'all'), then the layout's obstacles: a solid block, the block with a
    one-voxel tunnel along its longest axis, every voxel, or none."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(G_ORIGIN, G_RES, size_of(gs), mode=mode)
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(gs)
    g = np.asarray(gs)
    blo, bhi = g // 5, np.maximum(g // 5, g - 1 - g // 5)
    inblock = np.all((allv >= blo) & (allv <= bhi), axis=1)
    if layout == "tunnel":
        ax = int(np.argmax(bhi - blo))
        mid = (blo + bhi) // 2
        others = [k for k in range(3) if k != ax]
        inblock &= ~np.all(allv[:, others] == mid[others], axis=1)
    obst = {"block": inblock, "tunnel": inblock, "all": np.ones(len(allv), bool), "none": np.zeros(len(allv), bool)}[layout]
    seen = np.ones(len(allv), bool) if layout == "all" else (rng.random(len(allv)) >= 0.1) | obst
    m.SetOccupancyBatchVox(allv[seen & ~obst], np.zeros(int(np.sum(seen & ~obst)), np.uint8))
    m.SetOccupancyBatchVox(allv[obst], np.ones(int(np.sum(obst)), np.uint8))
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    return m


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("gs", LAYOUT_SHAPES, ids=shape_id)
def test_grid_shapes(gs, mode):
    rng = np.random.default_rng(17 + LAYOUT_SHAPES.index(gs))
    for layout in ("block", "tunnel", "all", "none"):
        m = layout_map(gs, mode, layout, rng)
        sf = m.SignedField()
        full = ((0, 0, 0), tuple(g - 1 for g in gs))
        for box in (full, (tuple(g // 3 for g in gs), full[1]), ((0, 0, 0), tuple(max(0, (2 * g) // 3 - 1) for g in gs))):
            S, q, D = check_field(m, sf, box, G_ORIGIN, G_RES)
            if layout == "all" and box == full:
                assert np.all(S == -np.inf)
            if layout == "none":
                assert np.all(q == 0)
            check_queries(m, sf, box, S, q, D, rng, G_ORIGIN, G_RES, device=layout == "tunnel")
        sf.close()
        m.close()


def test_solid_cube_gradient_leads_out():
    """Inside a solid cube the plain field is flat (0, gradient 0); the signed gradient points away from the centre, and following
    it (the descent direction of a collision cost) leaves the cube."""
    gs = (40, 40, 40)
    import fiesta_b200
    m = fiesta_b200.ESDFMap(G_ORIGIN, G_RES, size_of(gs), mode="exact")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(gs)
    cube = np.all((allv >= 10) & (allv <= 29), axis=1)
    m.SetOccupancyBatchVox(allv[~cube], np.zeros(int(np.sum(~cube)), np.uint8))
    m.SetOccupancyBatchVox(allv[cube], np.ones(int(np.sum(cube)), np.uint8))
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    sf = m.SignedField()
    st = sf.compute((4, 4, 4), (35, 35, 35))
    assert st["interior"] > 0 and st["max_depth_sq"] == 100
    o = np.asarray(G_ORIGIN)
    c = o + 20.0 * G_RES
    rng = np.random.default_rng(5)
    p = o + rng.uniform(11.0, 29.0, (256, 3)) * G_RES
    p = p[np.max(np.abs(p - c), axis=1) >= 2 * G_RES]                       # off the centre
    d0, g0 = m.GetDistWithGradTrilinearBatch(p)
    assert np.all(d0 == 0.0) and np.all(g0 == 0.0)                            # the unsigned field gives no direction
    d, g = sf.GetDistWithGradTrilinearBatch(p)
    assert np.all(d < 0)
    assert np.all(np.sum(g * (p - c), axis=1) > 0)
    for _ in range(60):                                                        # half-voxel steps along the gradient
        _, g = sf.GetDistWithGradTrilinearBatch(p)
        n = np.linalg.norm(g, axis=1)
        p = p + np.where(n[:, None] > 0, g / np.maximum(n, 1e-300)[:, None], 0.0) * 0.5 * G_RES
    v = np.floor((p - o) / G_RES).astype(int)
    assert not np.any(np.all((v >= 10) & (v <= 29), axis=1))
    sf.close()
    m.close()


# ---- staleness and argument errors
def rc_calls(m, sf):
    """Return codes of export and the four queries (one position; device forms on the current stream)."""
    import torch
    L, h = m._L, sf._h
    pos = np.zeros(3)
    out, grad = np.empty(1), np.empty(3)
    tp = torch.zeros((1, 3), dtype=torch.float64, device="cuda")
    td, tg = torch.empty(1, dtype=torch.float64, device="cuda"), torch.empty((1, 3), dtype=torch.float64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    ex = np.empty(int(np.prod(sf.shape)))
    return [L.fiesta_signed_export(h, ex.ctypes),
            L.fiesta_signed_get_distance_batch(h, pos.ctypes, 1, out.ctypes),
            L.fiesta_signed_get_dist_grad_trilinear_batch(h, pos.ctypes, 1, out.ctypes, grad.ctypes),
            L.fiesta_signed_get_distance_batch_device(h, tp.data_ptr(), 1, td.data_ptr(), s),
            L.fiesta_signed_get_dist_grad_trilinear_batch_device(h, tp.data_ptr(), 1, td.data_ptr(), tg.data_ptr(), s)]


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_staleness_and_errors(mode):
    import fiesta_b200
    m = layout_map((13, 11, 30), mode, "tunnel", np.random.default_rng(2))
    sf = m.SignedField()
    L, h = m._L, sf._h
    gs = m.grid_size
    lo, hi = np.zeros(3, np.int32), np.array(gs, np.int32) - 1
    sf.shape = tuple(gs)
    assert rc_calls(m, sf) == [INVALID] * 5                                   # before any compute
    assert "no field has been computed" in L.fiesta_last_error().decode()
    sf.compute(lo, hi)
    want = sf.export()
    assert rc_calls(m, sf) == [0] * 5
    for step in ("occupancy", "esdf", "occupancy_no_change", "esdf_no_change"):
        if step == "occupancy":
            m.SetOccupancyBatchVox(np.array([[2, 2, 2]], np.int32), np.ones(1, np.uint8))
        if step.startswith("occupancy"):
            m.UpdateOccupancy(True)
        else:
            m.UpdateESDF()
        assert rc_calls(m, sf) == [INVALID] * 5, step
        assert "compute again" in L.fiesta_last_error().decode()
        with pytest.raises(fiesta_b200.FiestaError):
            sf.export()
        sf.compute(lo, hi)
        assert rc_calls(m, sf) == [0] * 5, step
    want = sf.export()
    # argument errors: the code, and a valid field stays valid and unchanged
    bad_boxes = [(np.array([-1, 0, 0]), hi), (lo, np.array([gs[0], 0, 0])), (np.array([3, 0, 0]), np.array([2, 5, 5]))]
    for blo, bhi in bad_boxes:
        assert L.fiesta_signed_compute(h, np.ascontiguousarray(blo, np.int32).ctypes, np.ascontiguousarray(bhi, np.int32).ctypes, None) == INVALID
        assert "0 <= lo <= hi < grid size" in L.fiesta_last_error().decode()
    assert L.fiesta_signed_compute(h, None, hi.ctypes, None) == INVALID
    assert L.fiesta_signed_export(h, None) == INVALID
    out, pos = np.empty(4), np.zeros(12)
    assert L.fiesta_signed_get_distance_batch(h, None, 4, out.ctypes) == INVALID
    assert L.fiesta_signed_get_distance_batch(h, pos.ctypes, -1, out.ctypes) == INVALID
    assert L.fiesta_signed_get_dist_grad_trilinear_batch(h, pos.ctypes, 4, out.ctypes, None) == INVALID
    assert L.fiesta_signed_get_distance_batch_device(h, None, 4, None, None) == INVALID
    assert L.fiesta_signed_get_dist_grad_trilinear_batch_device(h, None, 4, None, None, None) == INVALID
    assert "negative count or null buffer" in L.fiesta_last_error().decode()
    assert L.fiesta_signed_get_distance_batch(h, None, 0, None) == 0            # no work, no buffers needed
    assert np.array_equal(bits(sf.export()), bits(want))
    # a capturing stream is refused, as for the map's device queries
    import torch
    tp = torch.zeros((1, 3), dtype=torch.float64, device="cuda")
    td, tg = torch.empty(1, dtype=torch.float64, device="cuda"), torch.empty((1, 3), dtype=torch.float64, device="cuda")
    x = torch.zeros(4, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        x.add_(1)
        rc1 = L.fiesta_signed_get_distance_batch_device(h, tp.data_ptr(), 1, td.data_ptr(), s.cuda_stream)
        rc2 = L.fiesta_signed_get_dist_grad_trilinear_batch_device(h, tp.data_ptr(), 1, td.data_ptr(), tg.data_ptr(), s.cuda_stream)
    assert (rc1, rc2) == (INVALID, INVALID)
    assert "capturing" in L.fiesta_last_error().decode()
    torch.cuda.synchronize()
    assert np.array_equal(bits(sf.export()), bits(want))
    sf.close()
    m.close()
