"""GPU: robot-shaped collision checks (fiesta_check_poses, _device, fiesta_host_mirror_check_poses) against the definition in
tests/poseref.py evaluated on export_distance(), on ray-cast maps in both modes and on grid shapes at the library's limits; cross-
checks with safe flight corridors (a box pose over a voxel box) and segment clearance (a point body); the stream contract of the
device form; and the error paths."""
import ctypes as C

import numpy as np
import pytest

from tests import geometry, poseref, scenes
from tests.test_gpu_segments import ORIGIN, RES, SIZE, frame, raycast_map

pytestmark = pytest.mark.gpu

LO, HI = np.array(ORIGIN), np.array(ORIGIN) + np.array(SIZE)
DRONE, CAR = (0.25, 0.25, 0.1), (2.25, 0.9, 0.75)
SETTINGS = [(0.0, False), (0.0, True), (RES, False), (0.3, True)]


def to_numpy(out):
    return tuple(x.cpu().numpy() for x in out)


def assert_same(got, want, tag):
    for g, w, name in zip(got, want, ("status", "n_blocked", "hit_idx")):
        assert np.array_equal(np.asarray(g), w), (tag, name, np.flatnonzero(np.asarray(g) != w)[:5])


def random_poses(rng, n, h, lo=LO, hi=HI, yaw_only=False):
    p = rng.uniform(lo, hi, (n, 3))
    R = poseref.yaw_rotations(rng, n) if yaw_only else poseref.random_rotations(rng, n)
    return poseref.poses(p, R)


def check_forms(m, P, h, origin, res, size, settings=SETTINGS):
    """Host form, device form (torch tensors on a side stream) and mirror form all equal poseref; returns the statuses seen."""
    import torch
    lo, hi = np.asarray(origin), np.asarray(origin) + np.asarray(size)
    D = m.export_distance().reshape(m.grid_size)
    want = poseref.check_all(P, h, origin, res, lo, hi, D, settings)
    mir = m.HostMirror()
    P_t = torch.from_numpy(P).cuda(m.device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    seen = set()
    for r, unk in settings:
        tag = (h, r, unk)
        assert_same(m.CheckPoses(P, h, r, unknown_blocks=unk), want[(r, unk)], tag)
        assert_same(mir.CheckPoses(P, h, r, unknown_blocks=unk), want[(r, unk)], tag)
        with torch.cuda.stream(s):
            dev = m.CheckPoses(P_t, h, r, unknown_blocks=unk)
        assert all(x.is_cuda for x in dev)
        s.synchronize()
        assert_same(to_numpy(dev), want[(r, unk)], tag)
        seen |= set(int(x) for x in want[(r, unk)][0])
    mir.close()
    return seen


@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("kind", ["lidar", "depth"])
def test_poses_match_definition(mode, kind):
    m, _ = raycast_map(mode, kind)
    rng = np.random.default_rng(11)
    seen = set()
    gs = m.grid_size
    for h, n, yaw in ((DRONE, 300, False), (CAR, 40, False), (CAR, 40, True)):
        P = np.concatenate([random_poses(rng, n, h, yaw_only=yaw), poseref.adversarial(rng, ORIGIN, RES, gs, h)])
        seen |= check_forms(m, P, h, ORIGIN, RES, SIZE)
    assert seen == {0, 1, 2, 3}, seen


def test_box_pose_equals_corridor_seed():
    """R = I, the centre of a voxel box and h_k = n_k * res / 2 - res / 4: the pose touches exactly that box, so it is blocked iff
    InflateBoxes rejects the box as a seed (limit box = grid, max_steps 0), and its hit_idx is the box's least blocking index."""
    m, _ = raycast_map("exact", "lidar", frames=2)
    gs = np.asarray(m.grid_size)
    D = m.export_distance().reshape(m.grid_size)
    rng = np.random.default_rng(4)
    counts = np.zeros(2, np.int64)
    for r, unk in SETTINGS:
        for nk in ((1, 1, 1), (3, 2, 5), (8, 1, 2)):
            nk = np.asarray(nk)
            slo = rng.integers(0, gs - nk + 1, (120, 3)).astype(np.int32)
            shi = (slo + nk - 1).astype(np.int32)
            st, _, _, _ = m.InflateBoxes(slo, shi, (0, 0, 0), gs - 1, (0, 0, 0), r, unknown_blocks=unk)
            h = tuple(float(x) for x in nk * RES / 2 - RES / 4)
            cen = (slo + shi + 1) / 2 * RES + np.asarray(ORIGIN)
            P = poseref.poses(cen, np.broadcast_to(np.eye(3), (len(cen), 3, 3)))
            pst, nb, idx = m.CheckPoses(P, h, r, unknown_blocks=unk)
            assert np.array_equal(pst == 1, st == 1) and set(np.unique(pst)) <= {0, 1}, (nk, r, unk)
            counts += np.bincount(pst, minlength=2)
            for i in np.flatnonzero(pst == 1):
                b = D[slo[i, 0]:shi[i, 0] + 1, slo[i, 1]:shi[i, 1] + 1, slo[i, 2]:shi[i, 2] + 1]
                blk = (np.where(b < 0, 1e4, b) <= r) | (unk & (b == -10000))
                assert nb[i] == blk.sum()
                first = np.argwhere(blk)[0] + slo[i]
                assert idx[i] == (first[0] * gs[1] + first[1]) * gs[2] + first[2]
    assert counts.min() > 50, counts


def test_point_body_equals_zero_length_segment():
    """h = 0 at a position strictly inside a voxel touches that voxel only: the status and hit_idx of the segment {p, p}."""
    m, _ = raycast_map("fast", "lidar", frames=2)
    rng = np.random.default_rng(6)
    gs = np.asarray(m.grid_size)
    v = rng.integers(0, gs, (4000, 3))
    p = (v + rng.uniform(0.05, 0.95, (4000, 3))) * RES + np.asarray(ORIGIN)
    P = poseref.poses(p, poseref.random_rotations(rng, len(p)))
    for r, unk in SETTINGS:
        st, nb, idx = m.CheckPoses(P, (0.0, 0.0, 0.0), r, unknown_blocks=unk)
        sst, sidx, _, _ = m.CheckSegments(np.concatenate([p, p], 1), r, unknown_blocks=unk)
        assert np.array_equal(st, sst) and np.array_equal(idx, sidx) and np.array_equal(nb, (sst == 1).astype(np.int32))
        assert 0 < (st == 1).sum() < len(st)


def test_stream_contract():
    """A device query enqueued before an UpdateESDF that rewrites many records answers for the map before it (the host mirror
    refreshed before the frame); one enqueued after it answers for the map after it."""
    import torch
    import fiesta_b200
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, mode="exact")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    sc = scenes.Scene((2.8, 2.8, 1.4), 10, 5, seed=3, edge=(0.3, 0.8))
    pts, T = frame(sc, 0)
    m.RaycastFrame(pts, T, 0.3, 4.0); m.UpdateOccupancy(True); m.UpdateESDF()
    mir = m.HostMirror()
    rng = np.random.default_rng(5)
    P = random_poses(rng, 1 << 18, DRONE)
    P_t = torch.from_numpy(P).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        before_t = m.CheckPoses(P_t, DRONE, 0.0, unknown_blocks=True)
    for _ in range(3):                                                    # the boxes move far
        sc.step()
    pts, T = frame(sc, 1)
    m.RaycastFrame(pts, T, 0.3, 4.0); m.UpdateOccupancy(True); m.UpdateESDF()
    with torch.cuda.stream(s):
        after_t = m.CheckPoses(P_t, DRONE, 0.0, unknown_blocks=True)
    s.synchronize()
    before = mir.CheckPoses(P, DRONE, 0.0, unknown_blocks=True)
    assert_same(to_numpy(before_t), before, "query enqueued before the update")
    after = m.CheckPoses(P, DRONE, 0.0, unknown_blocks=True)
    assert_same(to_numpy(after_t), after, "query enqueued after the update")
    assert (after[1] != before[1]).sum() > 100                            # the frame did change the answers
    mir.close()


SHAPES = [(1, 1, 1), (5, 1, 1), (1, 1, 5), (37, 1, 29), (2, 17, 3), (13, 11, 30), (13, 11, 7), (17, 3, 28), (2046, 3, 2)]


@pytest.mark.parametrize("gs", SHAPES, ids=geometry.shape_id)
def test_poses_on_grid_shapes(gs):
    """Thin, padded (Pz != Gz) and off-tile grids: poses on and near every face, the forms against poseref."""
    import fiesta_b200
    size = geometry.size_of(gs)
    m = fiesta_b200.ESDFMap(geometry.ORIGIN, geometry.RES, size, mode="fast")
    m.SetParameters(*scenes.PARAMS_TOGGLE)
    rng = np.random.default_rng(sum(gs))
    allv = scenes.all_voxels(gs)
    seen_v = allv[rng.random(len(allv)) < 0.85]
    m.SetOccupancyBatchVox(seen_v, np.zeros(len(seen_v), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    obst = seen_v[rng.random(len(seen_v)) < 0.1]
    m.SetOccupancyBatchVox(obst, np.ones(len(obst), np.uint8)); m.UpdateOccupancy(True); m.UpdateESDF()
    lo = np.asarray(geometry.ORIGIN)
    hi = lo + np.asarray(size)
    seen = set()
    for h in ((0.3, 0.2, 0.1), (0.0, 0.0, 0.0), (0.6, 0.05, 0.4)):
        near = np.where(rng.random((80, 3)) < 0.5, rng.choice([0.0, 1.0], (80, 3)), rng.random((80, 3))) * (hi - lo) + lo
        near += rng.choice([0.0, 0.01, -0.01, 0.1], (80, 3))
        P = np.concatenate([poseref.poses(near, poseref.random_rotations(rng, 80)), random_poses(rng, 40, h, lo, hi),
                            poseref.adversarial(rng, geometry.ORIGIN, geometry.RES, gs, h)])
        seen |= check_forms(m, P, h, geometry.ORIGIN, geometry.RES, size, settings=[(0.0, False), (0.25, True)])
    assert {2, 3} <= seen


def test_error_paths():
    import torch
    import fiesta_b200
    m, _ = raycast_map("fast", "lidar", frames=1)
    L = m._L
    rng = np.random.default_rng(1)
    P = random_poses(rng, 64, DRONE)
    n = len(P)

    def host_outs():
        return [np.full(n, 7, np.int32), np.full(n, 7, np.int32), np.full(n, 7, np.int64)]

    def call(h=DRONE, r=0.1, flags=0, nn=n, poses=P, outs=None, fn=L.fiesta_check_poses):
        outs = host_outs() if outs is None else outs
        he = np.asarray(h, np.float64)
        rc = fn(m._h, None if poses is None else poses.ctypes, C.c_int64(nn), he.ctypes, C.c_double(r), flags,
                *(o.ctypes if o is not None else None for o in outs))
        return rc, outs

    mir = m.HostMirror()
    for fn in (L.fiesta_check_poses, lambda h, *a: L.fiesta_host_mirror_check_poses(mir._h, *a)):
        cases = [dict(h=(-0.1, 0.1, 0.1)), dict(h=(np.nan, 0.1, 0.1)), dict(h=(0.1, np.inf, 0.1)), dict(r=-0.1), dict(r=np.nan),
                 dict(r=1e4), dict(flags=2), dict(nn=-1), dict(poses=None)]
        for kw in cases:
            rc, outs = call(fn=fn, **kw)
            assert rc == 1, kw                                            # FIESTA_ERR_INVALID
            assert all((o == 7).all() for o in outs), kw                  # nothing written
        rc, outs = call(fn=fn, outs=[None, np.empty(n, np.int32), np.empty(n, np.int64)])
        assert rc == 1
        for kw in (dict(h=(256 * RES, 0.0, 1e-3)), dict(h=(100 * RES, 100 * RES, 60 * RES)), dict(nn=(1 << 31) - 1)):
            rc, outs = call(fn=fn, **kw)
            assert rc == 4, kw                                            # FIESTA_ERR_LIMIT
            assert all((o == 7).all() for o in outs), kw
        assert call(fn=fn, h=(128 * RES, 128 * RES, 0.0))[0] == 0          # exactly 256 voxels is allowed
        assert call(fn=fn, nn=0, poses=None, outs=[None, None, None])[0] == 0
    mir.close()
    # device form: the same rejections, and a capturing stream
    P_t = torch.from_numpy(P).cuda()
    outs = [torch.full((n,), 7, dtype=dt, device="cuda") for dt in (torch.int32, torch.int32, torch.int64)]
    ptrs = [o.data_ptr() for o in outs]
    he = np.asarray(DRONE, np.float64)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        x.add_(1)
        rc = L.fiesta_check_poses_device(m._h, P_t.data_ptr(), n, he.ctypes, C.c_double(0.1), 0, *ptrs, s.cuda_stream)
    assert rc == 1
    torch.cuda.synchronize()
    bad = [((-1.0, 0.1, 0.1), 0.1, 0, n), (DRONE, np.nan, 0, n), (DRONE, 0.1, 4, n), (DRONE, 0.1, 0, -1), ((300 * RES, 0.0, 0.0), 0.1, 0, n)]
    for h, r, fl, nn in bad:
        hh = np.asarray(h, np.float64)
        rc = L.fiesta_check_poses_device(m._h, P_t.data_ptr(), C.c_int64(nn), hh.ctypes, C.c_double(r), fl, *ptrs, None)
        assert rc in (1, 4), (h, r, fl, nn)
    assert L.fiesta_check_poses_device(m._h, None, n, he.ctypes, C.c_double(0.1), 0, *ptrs, None) == 1
    assert L.fiesta_check_poses_device(m._h, P_t.data_ptr(), n, None, C.c_double(0.1), 0, *ptrs, None) == 1
    torch.cuda.synchronize()
    assert all((o == 7).all().item() for o in outs)                        # nothing written
    # Python: wrong tensor dtype, shape or half extents
    for t in (P_t.float(), P_t[:, :9].contiguous(), P_t.reshape(-1), P_t.t()):
        with pytest.raises(ValueError):
            m.CheckPoses(t, DRONE, 0.1)
    with pytest.raises(ValueError):
        m.CheckPoses(P, (0.1, 0.1), 0.1)
    with pytest.raises(fiesta_b200.FiestaError):
        m.CheckPoses(P, (0.1, -0.1, 0.1), 0.1)
    st = m.CheckPoses(P_t, DRONE, 0.1)                                     # the map is still usable
    torch.cuda.synchronize()
    assert_same(to_numpy(st), m.CheckPoses(P, DRONE, 0.1), "after rejections")
