"""GPU: segment clearance (fiesta_check_segments, _device, fiesta_host_mirror_check_segments) against the exact definition in
tests/segref.py evaluated on export_distance(), on ray-cast maps in both modes; and the stream contract of the device-buffer
queries (fiesta_check_segments_device, fiesta_get_distance_batch_device, fiesta_get_dist_grad_trilinear_batch_device)."""
import ctypes as C

import numpy as np
import pytest

from tests import scenes, segref

pytestmark = pytest.mark.gpu

ORIGIN, RES, SIZE = (-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.2)
LO, HI = np.array(ORIGIN), np.array(ORIGIN) + np.array(SIZE)


def raycast_map(mode, kind, frames=4):
    """A ray-cast map with moving boxes (TOGGLE parameters: a box that moves away is deleted at once)."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode=mode)
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


def segments(rng, n, origin=ORIGIN, res=RES, size=SIZE):
    """Short (0.05-1 m) and long (1-8 m) segments, some leaving the map, plus the adversarial set in voxel units."""
    lo, hi = np.asarray(origin), np.asarray(origin) + np.asarray(size)
    a = rng.uniform(lo, hi, (n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    L = np.where(rng.random(n) < 0.6, rng.uniform(0.05, 1.0, n), rng.uniform(1.0, 8.0, n))
    ab = np.concatenate([a, a + d * L[:, None]], 1)
    gs = np.ceil(np.asarray(size) / res)
    adv = np.array([np.concatenate([lo + u[:3] * res, lo + u[3:] * res]) for u in segref.adversarial_voxel_units(gs, rng)])
    return np.ascontiguousarray(np.concatenate([ab, adv]))


def expected(walks, D, r, unknown_blocks):
    rows = [segref.apply(w, D, r, unknown_blocks) for w in walks]
    return (np.array([x[0] for x in rows], np.int32), np.array([x[1] for x in rows], np.int64), np.array([x[2] for x in rows]),
            np.array([x[3] for x in rows]))


def assert_same(got, want, tag):
    st, ix, t, md = (np.asarray(x) for x in got)
    assert np.array_equal(st, want[0]), tag
    assert np.array_equal(ix, want[1]), tag
    assert np.array_equal(t, want[2], equal_nan=True), tag
    assert np.array_equal(md, want[3]), tag


def to_numpy(out):
    return tuple(x.cpu().numpy() for x in out)


def check_map(m, ab, origin=ORIGIN, res=RES, size=SIZE, clearances=(0.0, RES, 2.5), samples=True):
    import torch
    lo, hi = np.asarray(origin), np.asarray(origin) + np.asarray(size)
    D = m.export_distance().reshape(m.grid_size)
    walks = [segref.segment_walk(s, origin, res, lo, hi) for s in ab]
    mir = m.HostMirror()
    ab_t = torch.from_numpy(ab).cuda(m.device)
    statuses, sampled = set(), 0
    for r in clearances:
        for unk in (False, True):
            want = expected(walks, D, r, unk)
            tag = (r, unk)
            got = m.CheckSegments(ab, r, unknown_blocks=unk)
            assert_same(got, want, tag)
            assert_same(mir.CheckSegments(ab, r, unknown_blocks=unk), want, tag)
            dev = m.CheckSegments(ab_t, r, unknown_blocks=unk)
            assert all(x.is_cuda for x in dev)
            torch.cuda.synchronize()
            assert_same(to_numpy(dev), want, tag)
            statuses |= set(int(s) for s in np.unique(want[0]))
            if samples and r > 0:                                          # independent check through the point query
                clear = ab[want[0] == 0]
                t = np.linspace(0, 1, 65)
                p = (clear[:, None, :3] + t[None, :, None] * (clear[:, None, 3:] - clear[:, None, :3])).reshape(-1, 3)
                u = (p - np.asarray(origin)) / res
                away = np.all(np.abs(u - np.round(u)) > 1e-5, axis=1)         # off the faces by more than the 2^-20 voxel lattice step
                d = m.GetDistanceBatch(p[away])
                assert np.all(d > r), tag
                sampled += len(d)
    mir.close()
    assert statuses == {0, 1, 2}, statuses
    assert sampled > 10000 or not samples


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("kind", ["lidar", "depth"])
def test_segments_match_definition(mode, kind):
    m, deletes = raycast_map(mode, kind)
    assert deletes > 0
    ab = segments(np.random.default_rng(7), 2500)
    check_map(m, ab)


def test_segments_long_axis():
    """A 2046-voxel x axis (the grid limit): segments across it take 64 sweeps of 32 slabs in the kernel."""
    import fiesta_b200
    origin, res, size = (0.0, 0.0, 0.0), 0.0625, (127.875, 1.0, 1.0)
    m = fiesta_b200.ESDFMap(origin, res, size, mode="fast")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    gs = m.grid_size
    assert gs == (2046, 16, 16)
    allv = scenes.all_voxels(gs)
    rng = np.random.default_rng(9)
    seen = allv[rng.random(len(allv)) < 0.9]                              # 10 % never observed
    m.SetOccupancyBatchVox(seen, np.zeros(len(seen), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    obst = seen[rng.choice(len(seen), 40, replace=False)]
    m.SetOccupancyBatchVox(obst, np.ones(len(obst), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    a = np.stack([rng.uniform(0, 2, 150), rng.uniform(0, 1, 150), rng.uniform(0, 1, 150)], 1)
    b = np.stack([rng.uniform(125, 127.875, 150), rng.uniform(0, 1, 150), rng.uniform(0, 1, 150)], 1)
    ab = np.concatenate([np.concatenate([a, b], 1), np.concatenate([b, a], 1), segments(rng, 200, origin, res, size)])
    check_map(m, ab, origin, res, size, clearances=(0.0, 0.1, 0.4), samples=False)


def test_segments_sliding_local_map_exact():
    """Local-map mode in EXACT mode: a sliding update box with UpdateOccupancy(false) leaves FB_DINF records (distance +infinity,
    closest obstacle kept); they read +10000 and never block."""
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode="exact")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(m.grid_size)
    rng = np.random.default_rng(7)
    idx = rng.choice(len(allv), 300, replace=False)
    m.SetOccupancyBatchVox(allv, np.zeros(len(allv), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    m.SetOccupancyBatchVox(allv[idx], np.ones(300, np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    m.SetParameters(*scenes.PARAMS_DEFAULT)
    for r in range(6):
        c = np.array([-1.2 + 0.35 * r, -0.9 + 0.3 * r, 0.0])
        m.SetUpdateRange(c - np.array([1.3, 1.2, 0.9]), c + np.array([1.3, 1.2, 0.9]))
        vox = np.stack([rng.integers(0, m.grid_size[i], 6000) for i in range(3)], -1).astype(np.int32)
        m.SetOccupancyBatchVox(vox, (rng.random(6000) < 0.4).astype(np.uint8))
        m.UpdateOccupancy(False)
        m.UpdateESDF()
    D, Cb = m.export_distance(), m.export_closest_obstacle()
    assert int(((D == 10000) & (Cb[:, 0] != -10000)).sum()) > 0           # FB_DINF records are present
    check_map(m, segments(np.random.default_rng(8), 2000))


def frame(sc, f):
    p, yaw = scenes.pose_walk(f + 1, seed=2, clamp=0.5)[f]
    return scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=360)


def test_stream_ordering_after_update():
    """UpdateESDF, then the device queries on a non-default torch stream with no host synchronisation in between: the results equal
    the synchronous host queries taken afterwards, bit for bit."""
    import torch
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode="fast")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    rng = np.random.default_rng(3)
    ab = segments(rng, 4000)
    pos = rng.uniform(LO - 0.2, HI + 0.2, (50000, 3))
    ab_t, pos_t = torch.from_numpy(ab).cuda(), torch.from_numpy(pos).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    outs = []
    with torch.cuda.stream(s):
        for f in range(3):
            pts, T = frame(sc, f)
            m.RaycastFrame(pts, T, 0.3, 4.0)
            m.UpdateOccupancy(True)
            m.UpdateESDF()
            outs.append((m.CheckSegments(ab_t, RES), m.GetDistanceBatchDevice(pos_t), m.GetDistWithGradTrilinearBatchDevice(pos_t)))
            sc.step()
    s.synchronize()
    seg, d, (dt, gt) = outs[-1]
    assert_same(to_numpy(seg), m.CheckSegments(ab, RES), "segments")
    assert np.array_equal(d.cpu().numpy(), m.GetDistanceBatch(pos))
    d2, g2 = m.GetDistWithGradTrilinearBatch(pos)
    assert np.array_equal(dt.cpu().numpy(), d2) and np.array_equal(gt.cpu().numpy(), g2)
    assert not np.array_equal(to_numpy(outs[0][0])[3], to_numpy(seg)[3])   # the map changed between the frames


def test_stream_query_runs_before_later_update():
    """A large device query enqueued right before a frame that rewrites many records answers for the map as it was at the call:
    equal to the host mirror refreshed before the frame."""
    import torch
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode="exact")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    pts, T = frame(sc, 0)
    m.RaycastFrame(pts, T, 0.3, 4.0); m.UpdateOccupancy(True); m.UpdateESDF()
    mir = m.HostMirror()
    rng = np.random.default_rng(5)
    a = rng.uniform(LO, HI, (1 << 20, 3))
    ab = np.concatenate([a, np.clip(a + rng.normal(0, 2.0, a.shape), LO, HI)], 1)
    pos = rng.uniform(LO, HI, (1 << 20, 3))
    ab_t, pos_t = torch.from_numpy(ab).cuda(), torch.from_numpy(pos).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        seg = m.CheckSegments(ab_t, 0.0, unknown_blocks=True)
        d = m.GetDistanceBatchDevice(pos_t)
    for _ in range(3):                                                    # mutate at once: the boxes move far
        sc.step()
    pts, T = frame(sc, 1)
    m.RaycastFrame(pts, T, 0.3, 4.0); m.UpdateOccupancy(True); m.UpdateESDF()
    s.synchronize()
    before = mir.CheckSegments(ab, 0.0, unknown_blocks=True)
    assert_same(to_numpy(seg), before, "query enqueued before the update")
    assert np.array_equal(d.cpu().numpy(), mir.GetDistanceBatch(pos))
    after = m.CheckSegments(ab, 0.0, unknown_blocks=True)
    assert (after[0] != before[0]).sum() > 100 and (after[3] != before[3]).sum() > 100     # the frame did change the answers
    mir.close()


def test_device_queries_reject_capture_and_bad_arguments():
    import torch
    import fiesta_b200
    m, _ = raycast_map("fast", "lidar", frames=1)
    L = m._L
    ab = torch.from_numpy(segments(np.random.default_rng(1), 64)).cuda()
    n = ab.shape[0]
    outs = [torch.empty(n, dtype=dt, device="cuda") for dt in (torch.int32, torch.int64, torch.float64, torch.float64)]
    ptrs = [o.data_ptr() for o in outs]
    pos = torch.zeros((n, 3), dtype=torch.float64, device="cuda")
    x = torch.zeros(4, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        x.add_(1)
        rc1 = L.fiesta_check_segments_device(m._h, ab.data_ptr(), n, C.c_double(0.1), 0, *ptrs, s.cuda_stream)
        rc2 = L.fiesta_get_distance_batch_device(m._h, pos.data_ptr(), n, ptrs[2], s.cuda_stream)
        rc3 = L.fiesta_get_dist_grad_trilinear_batch_device(m._h, pos.data_ptr(), n, ptrs[2], ptrs[3], s.cuda_stream)
    assert (rc1, rc2, rc3) == (1, 1, 1)                                   # FIESTA_ERR_INVALID
    torch.cuda.synchronize()
    abn = ab.cpu().numpy()
    for bad in (-0.1, float("nan"), 1e4, float("inf")):
        with pytest.raises(fiesta_b200.FiestaError):
            m.CheckSegments(abn, bad)
        with pytest.raises(fiesta_b200.FiestaError):
            m.CheckSegments(ab, bad)
    assert L.fiesta_check_segments(m._h, abn.ctypes, n, C.c_double(0.1), 2, *(np.empty(n, dt).ctypes for dt in (np.int32, np.int64, np.float64, np.float64))) == 1
    assert L.fiesta_check_segments_device(m._h, None, n, C.c_double(0.1), 0, *ptrs, None) == 1
    with pytest.raises(ValueError):
        m.CheckSegments(ab.float(), 0.1)
    st = m.CheckSegments(ab, 0.1)                                         # the map is still usable
    torch.cuda.synchronize()
    assert_same(to_numpy(st), m.CheckSegments(abn, 0.1), "after rejections")
