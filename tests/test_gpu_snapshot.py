"""GPU: map snapshots (fiesta_snapshot_save / fiesta_snapshot_load).  A map loaded from a snapshot must continue, call for call,
exactly like the map it was saved from: after every later call (frames, update boxes, UpdateOccupancy with and without the
local-map reset, UpdateESDF, SetParameters, filtered depth frames) the exports, queries, point cloud, slice marker and statistics
are compared bit for bit.  Covered: both modes, LIDAR and filtered depth frames, grids with Gz % 4 == 0, Gz = 30 and a size that is
not a multiple of 8, snapshots taken right after creation, mid-run and just before SetParameters; once the loaded EXACT map
against the reference oracle; a negative control that drops the dependant-list order (LS, tclock) and must be seen; round trips;
objects attached to the loaded map; and every rejection, each followed by a valid load."""
import ctypes as C

import numpy as np
import pytest

import fiesta_b200
from fiesta_b200 import ESDFMap, FiestaError
from tests import poseref, scenes, snapshot_tool

pytestmark = pytest.mark.gpu

GRIDS = {
    "gz32": ((-3.2, -3.2, -1.6), (6.4, 6.4, 3.2), (2.8, 2.8, 1.4)),
    "gz30": ((-3.2, -3.2, -1.5), (6.4, 6.4, 3.0), (2.8, 2.8, 1.3)),
    "odd": ((-2.5, -2.15, -1.25), (5.0, 4.3, 2.5), (2.2, 1.9, 1.1)),      # 50 x 43 x 25: no axis a multiple of 8
}
RES = 0.1
HALF_BOX = np.array([1.6, 1.6, 0.9])
DROP = {"kernel_launches", "raycast_rounds"}   # raycast_rounds depends on the order concurrent rays claim voxels


@pytest.fixture(scope="module")
def tool(tmp_path_factory):
    return snapshot_tool.build(tmp_path_factory.mktemp("snaptool"))


def state(m, rng_seed=0):
    """Everything the continuation guarantee covers, as bytes per item."""
    gz = m.grid_size[2]
    lo, hi = np.asarray(m.origin), np.asarray(m.origin) + np.asarray(m.grid_size) * m.resolution
    q = np.random.default_rng(rng_seed).uniform(lo - 0.2, hi + 0.2, (512, 3))
    st = {k: v for k, v in m.stats().items() if k not in DROP and not k.startswith("ms_")}
    d, g = m.GetDistWithGradTrilinearBatch(q)
    hit, tot = m.export_counters()
    pc = m.GetPointCloud(0, gz - 1)
    sx, sc = m.GetSliceMarker(gz // 2, 2.0)
    out = dict(dist=m.export_distance(), cobs=m.export_closest_obstacle(), occ=m.export_occupancy(), hit=hit, tot=tot,
               q=m.GetDistanceBatch(q), tri=d, grad=g, occq=np.array([m.GetOccupancy(p) for p in q[:64]]), pc=pc, sx=sx, sc=sc,
               stats=np.array(sorted(st.items()), dtype=object))
    return {k: (v.tobytes() if v.dtype != object else repr(v.tolist())) for k, v in out.items()}


def differences(a, b, seed=0):
    sa, sb = state(a, seed), state(b, seed)
    return [k for k in sa if sa[k] != sb[k]]


class Run:
    """A map A, the maps loaded from its snapshots (followers, which must stay equal to A after every call) and optional
    watchers (maps expected to differ, only recorded)."""

    def __init__(self, grid, mode, kind, seed=1, oracle=False):
        origin, size, room = GRIDS[grid]
        self.kind = kind
        self.A = ESDFMap(origin, RES, size, mode=mode)
        self.followers, self.watchers, self.calls = [], [], 0
        self.ora = None
        if oracle:
            from oracle import pyoracle
            self.ora = pyoracle.OracleMap(origin, RES, size)
        self.sc = scenes.Scene(room, 8, 3, seed=seed, edge=(0.3, 0.8))
        self.poses = scenes.pose_walk(8, seed=seed, clamp=0.6)
        self.dp = fiesta_b200.DepthParams(scenes.FX * 0.125, scenes.FY * 0.125, scenes.CX * 0.125, scenes.CY * 0.125, 1, 2, 10.0, 0.1, 0.1)
        self.last_T = None
        self.seen_diff = set()

    def maps(self):
        return [self.A] + [b for _, b in self.followers] + [w for _, w in self.watchers]

    def check(self):
        self.calls += 1
        for name, b in self.followers:
            diff = differences(self.A, b, self.calls)
            if diff == ["stats"]:
                sa, sb = self.A.stats(), b.stats()
                diff = {k: (sa[k], sb[k]) for k in sa if sa[k] != sb[k] and k not in DROP and not k.startswith("ms_")}
            assert not diff, (name, self.calls, diff)
        for name, w in self.watchers:
            if differences(self.A, w, self.calls):
                self.seen_diff.add(name)

    def save(self, name, watcher=False, edit=None):
        s = self.A.save()
        if edit is not None:
            s = edit(s)
        b = ESDFMap.load(s, device=self.A.device)
        if edit is None:
            assert b.save() == s, name                       # save(load(S)) == S, byte for byte
            assert (b.grid_size, b.resolution, b.origin, b.mode) == (self.A.grid_size, self.A.resolution, self.A.origin, self.A.mode)
        (self.watchers if watcher else self.followers).append((name, b))
        self.check()                                         # exports right after load equal the source's
        return s

    def each(self, fn, ora=True):
        for m in self.maps():
            fn(m)
        if ora and self.ora is not None:
            fn(self.ora)
        self.check()

    def frame(self, f, box):
        p, yaw = self.poses[f]
        if box:                                              # boxes alternate sides of the sensor: UpdateOccupancy(false)
            c = p + (0.6 if f % 2 else -0.6, 0.0, 0.0)       # resets voxels observed before, which keep their obstacle (bit 31)
            self.each(lambda m: m.SetUpdateRange(c - HALF_BOX, c + HALF_BOX, True))
        else:
            self.each(lambda m: m.SetOriginalRange())
        if self.kind == "lidar":
            pts, T = scenes.lidar_frame(self.sc, p, yaw, beams=16, azimuths=360)
            self.each(lambda m: m.RaycastFrame(pts, T, 0.3, 4.0))
        else:
            img, T = scenes.depth_image(self.sc, p, yaw, width=80, height=60, scale=0.125)
            m_rel = np.linalg.inv(self.last_T) @ T if self.last_T is not None else np.eye(4)
            self.last_T = T
            self.each(lambda m: m.DepthFrame(img, self.dp, T, m_rel, 0.3, 4.0), ora=False)
        self.each(lambda m: m.UpdateOccupancy(f != 2))       # frame 2: local-map reset outside the previous box
        self.each(lambda m: m.UpdateESDF())
        self.sc.step()


@pytest.mark.parametrize("grid", sorted(GRIDS))
@pytest.mark.parametrize("kind", ["lidar", "depth"])
@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_continuation(mode, kind, grid, tool, tmp_path):
    oracle = mode == "exact" and kind == "lidar" and grid == "gz32"
    R = Run(grid, mode, kind, oracle=oracle)
    s0 = R.save("created")                                   # right after creation, before SetParameters
    assert snapshot_tool.header(s0)[2] == 0 and len(s0) == 384
    R.each(lambda m: m.SetParameters(*scenes.PARAMS_DEFAULT))
    for f in range(7):
        if f in (2, 3, 5):
            R.save("frame%d" % f)                            # f = 3: just before SetParameters
        if f == 3:
            R.each(lambda m: m.SetParameters(*scenes.PARAMS_TOGGLE))
            if mode == "exact" and kind == "lidar":          # negative control: no dependant-list order
                R.save("no-LS", watcher=True, edit=lambda s: snapshot_tool.edit(tool, s, "zero_ls", tmp_path))
        R.frame(f, box=f in (1, 2, 4, 5))
    if mode == "exact" and kind == "lidar":
        assert "no-LS" in R.seen_diff, "dropping LS and tclock went unnoticed"
    if oracle:
        from tests.parity import compare
        for name, b in R.followers:
            r = compare(b, R.ora, check_counters=True)
            assert r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0 and r["occ"] == 0 and r["counters"] == 0, (name, r)


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_saving_changes_nothing(mode):
    """Two maps fed the same frames, one saved after every call it can be saved at: they stay identical."""
    R = Run("gz30", mode, "lidar")
    twin = Run("gz30", mode, "lidar")
    for r in (R, twin):
        r.each(lambda m: m.SetParameters(*scenes.PARAMS_DEFAULT))
    for f in range(4):
        for r in (R, twin):
            r.frame(f, box=f % 2 == 1)
        s = R.A.save()
        assert not differences(R.A, twin.A)
        assert R.A.save() == s
    untouched = ESDFMap(*GRIDS["odd"][:1], RES, GRIDS["odd"][1], mode=mode)
    assert len(untouched.save()) == 384


def frontier_result(m):
    fr = m.Frontiers()
    st = fr.compute((0, 0, 0), tuple(g - 1 for g in m.grid_size), clearance=0.1, min_cluster_size=2)
    out = [repr(sorted((k, v) for k, v in st.items() if not k.startswith("ms_")))] + [v.tobytes() for v in fr.clusters().values()]
    out.append(fr.export().tobytes())
    fr.close()
    return out


def nav_result(m, rng):
    nav = m.NavField()
    box = ((4, 4, 2), tuple(g - 5 for g in m.grid_size))
    goals = rng.uniform(-1.0, 1.0, (4, 3)) * (1, 1, 0.3)
    st = nav.compute(box[0], box[1], goals, 0.2)
    starts = rng.uniform(-2.0, 2.0, (32, 3)) * (1, 1, 0.3)
    out = [repr(sorted((k, v) for k, v in st.items() if not k.startswith("ms_"))), nav.export().tobytes()]
    out += [a.tobytes() for a in nav.paths(starts, 96)]
    nav.close()
    return out


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_attached_objects(mode):
    R = Run("gz32", mode, "lidar")
    R.each(lambda m: m.SetParameters(*scenes.PARAMS_DEFAULT))
    for f in range(3):
        R.frame(f, box=False)
    B = ESDFMap.load(R.A.save())
    rng = np.random.default_rng(3)
    q = rng.uniform(-3.0, 3.0, (400, 3)) * (1, 1, 0.45)
    mirrors = [m.HostMirror() for m in (R.A, B)]
    for k in range(2):
        got = []
        for mir in mirrors:
            mir.refresh()
            d, g = mir.GetDistWithGradTrilinearBatch(q)
            got.append((mir.GetDistanceBatch(q).tobytes(), d.tobytes(), g.tobytes()))
        assert got[0] == got[1]
        if k == 0:                                            # one more frame on both, then refresh again
            R.followers.append(("loaded", B))
            R.frame(3, box=True)
    for mir in mirrors:
        mir.close()
    assert nav_result(R.A, np.random.default_rng(5)) == nav_result(B, np.random.default_rng(5))
    assert frontier_result(R.A) == frontier_result(B)
    ab = np.concatenate([rng.uniform(-2.5, 2.5, (300, 3)), rng.uniform(-2.5, 2.5, (300, 3))], 1) * (1, 1, 0.4, 1, 1, 0.4)
    seg = [tuple(a.tobytes() for a in m.CheckSegments(ab, 0.15)) for m in (R.A, B)]
    assert seg[0] == seg[1]
    P = poseref.poses(rng.uniform(-2.5, 2.5, (300, 3)) * (1, 1, 0.4), poseref.random_rotations(rng, 300))
    pose = [tuple(a.tobytes() for a in m.CheckPoses(P, (0.3, 0.2, 0.1), 0.05)) for m in (R.A, B)]
    assert pose[0] == pose[1]


def raw_save(m, cap, buf=None):
    size = C.c_int64(-1)
    rc = m._L.fiesta_snapshot_save(m._h, None if buf is None else buf.ctypes.data, C.c_int64(cap), C.byref(size))
    return rc, size.value


def expect_load_error(data, needle):
    with pytest.raises(FiestaError) as e:
        ESDFMap.load(data)
    assert "(1)" in str(e.value) and needle in str(e.value), str(e.value)


def test_rejections(tool, tmp_path):
    Rx = Run("odd", "exact", "lidar")
    Rf = Run("odd", "fast", "lidar")
    for r in (Rx, Rf):
        r.each(lambda m: m.SetParameters(*scenes.PARAMS_DEFAULT))
        for f in range(3):
            r.frame(f, box=f == 1)
    sx, sf = Rx.A.save(), Rf.A.save()
    want = {sx: state(Rx.A), sf: state(Rf.A)}

    def valid_load_still_works():
        for s in (sx, sf):
            b = ESDFMap.load(s)
            assert state(b) == want[s]
            b.close()

    # non-quiescent maps: nothing written, the map still works afterwards
    m = Rx.A
    buf = np.full(1 << 16, 0xAB, np.uint8)
    m.SetOccupancy((0.1, 0.2, 0.3), 1)
    assert raw_save(m, len(buf), buf)[0] == 1 and (buf == 0xAB).all()      # SetOccupancy staged
    assert m.UpdateOccupancy(True) in (0, 1)
    m.UpdateESDF()
    p, yaw = Rx.poses[4]
    pts, T = scenes.lidar_frame(Rx.sc, p, yaw, beams=16, azimuths=360)
    m.RaycastFrame(pts, T, 0.3, 4.0)
    assert m.CheckUpdate()
    assert raw_save(m, len(buf), buf)[0] == 1 and (buf == 0xAB).all()      # occupancy queue not empty
    assert m.UpdateOccupancy(True) == 1
    assert raw_save(m, len(buf), buf)[0] == 1 and (buf == 0xAB).all()      # inserts / deletes pending
    m.UpdateESDF()
    assert raw_save(m, 0)[0] == 0
    sh = ESDFMap(*GRIDS["gz32"][:1], RES, GRIDS["gz32"][1], mode="fast")
    sh.set_shard(0, 2)
    assert raw_save(sh, len(buf), buf)[0] == 1 and (buf == 0xAB).all()     # an x-slab shard
    sh.close()
    # cap too small: FIESTA_ERR_LIMIT, *size set, the buffer untouched
    rc, n = raw_save(Rf.A, 0)
    assert rc == 0 and n == len(sf)
    small = np.full(n - 1, 0xCD, np.uint8)
    assert raw_save(Rf.A, n - 1, small) == (4, n) and (small == 0xCD).all()
    valid_load_still_works()
    # malformed streams
    expect_load_error(sx[:-8], "bytes")                      # truncated
    expect_load_error(sx[:100], "truncated")
    pay = 384 + (4 * snapshot_tool.header(sx)[2] + 7) // 8 * 8
    flipped = bytearray(sx)
    flipped[pay + 13] ^= 0x04
    expect_load_error(bytes(flipped), "checksum mismatch")
    valid_load_still_works()
    for s, op, needle in ((sx, "obstacle_out", "outside the grid"), (sf, "obstacle_out", "outside the grid"), (sf, "bit31", "bit 31"),
                          (sx, "nan_occ", "not finite"), (sf, "nan_occ", "not finite"), (sx, "ls_ge_tclock", "relink clock"),
                          (sx, "tile_past", "past the grid"), (sf, "tile_past", "past the grid")):
        bad = snapshot_tool.edit(tool, s, op, tmp_path)
        assert bad != s
        expect_load_error(bad, needle)
        valid_load_still_works()
    assert snapshot_tool.edit(tool, sx, "refix", tmp_path) == sx       # the editor's checksums are the library's


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_environment_mode_is_ignored(mode, monkeypatch):
    R = Run("gz30", mode, "lidar")
    R.each(lambda m: m.SetParameters(*scenes.PARAMS_DEFAULT))
    R.frame(0, box=False)
    s = R.A.save()
    monkeypatch.setenv("FIESTA_B200_MODE", "fast" if mode == "exact" else "exact")
    b = ESDFMap.load(s)
    assert b.mode == mode
    R.followers.append(("env", b))
    R.check()
    R.frame(1, box=True)
    assert b.save() == R.A.save()
