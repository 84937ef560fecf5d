"""GPU: the exact return code and fiesta_last_error() text of every argument and state check of the planner entry points
(segments, poses, cost-to-go fields and matrices, frontiers and viewpoints, corridors, snapshots) and of the handles and device
queries around them, on small maps in both modes.  Callers match on these messages, so they are part of the C ABI."""
import ctypes as C

import numpy as np
import pytest

import fiesta_b200
from fiesta_b200 import SensorModel
from tests import scenes

pytestmark = pytest.mark.gpu

INVALID, LIMIT = 1, 4
ORIGIN, RES, SIZE = (0.0, 0.0, 0.0), 0.1, (1.6, 1.6, 0.8)
GRID = (16, 16, 8)                                       # two 8-voxel tile columns in x: a 2-rank shard is allowed
SNAP_HDR = 384                                           # bytes of a snapshot header
SENTINEL = "fiesta_nav_create: null argument"            # set before every row, so that a row never passes on a stale message

D = np.zeros(64)
I32 = np.zeros(64, np.int32)
I64 = np.zeros(64, np.int64)
LO = np.zeros(3, np.int32)
HI = np.array(GRID, np.int32) - 1
STEPS = np.full(3, 4, np.int32)
H = np.full(3, 0.1)
ORIENT = np.eye(3).ravel()


def ptr(a):
    return None if a is None else np.ascontiguousarray(a).ctypes


def new_map(mode, params=True):
    m = fiesta_b200.ESDFMap(ORIGIN, RES, SIZE, device=0, mode=mode)
    if params:
        m.SetParameters(*scenes.PARAMS_TOGGLE)
    return m


class Env:
    """A map with its planner handles: a cost-to-go field and a frontier object never computed, a frontier object computed over
    the whole (unobserved) grid, and a host mirror."""

    def __init__(self, mode):
        self.mode = mode
        self.m = new_map(mode)
        self.L, self.h = self.m._L, self.m._h
        self.nav, self.fr, self.frc, self.mirror = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        assert self.L.fiesta_nav_create(self.h, C.byref(self.nav)) == 0
        assert self.L.fiesta_frontiers_create(self.h, C.byref(self.fr)) == 0
        assert self.L.fiesta_frontiers_create(self.h, C.byref(self.frc)) == 0
        assert self.L.fiesta_frontiers_compute(self.frc, LO.ctypes, HI.ctypes, 0.0, 1, None) == 0
        assert self.L.fiesta_host_mirror_create(self.h, C.byref(self.mirror)) == 0

    def close(self):
        self.L.fiesta_nav_destroy(self.nav)
        self.L.fiesta_frontiers_destroy(self.fr)
        self.L.fiesta_frontiers_destroy(self.frc)
        self.m.close()                                   # the mirror goes with its map


@pytest.fixture(scope="module", params=["exact", "fast"])
def env(request):
    e = Env(request.param)
    yield e
    e.close()


def sensor(max_range=2.0, tan_h=1.0, tan_v=0.5):
    s = SensorModel()
    s.max_range = max_range
    s.tan_half_fov[0], s.tan_half_fov[1] = tan_h, tan_v
    return s


# ---- calls: each takes the Env and returns (return code, expected message); most expected messages are fixed strings
def segments(n=1, ab=D, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_check_segments(e.h, ptr(ab), n, clearance, flags, I32.ctypes, I64.ctypes, D.ctypes, D.ctypes)


def segments_device(n=1, ab=D, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_check_segments_device(e.h, ptr(ab), n, clearance, flags, I32.ctypes, I64.ctypes, D.ctypes, D.ctypes, None)


def mirror_segments(n=-1, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_host_mirror_check_segments(e.mirror, D.ctypes, n, clearance, flags, I32.ctypes, I64.ctypes, D.ctypes,
                                                           D.ctypes)


def poses(n=1, h=H, clearance=0.0, flags=0, fn="fiesta_check_poses"):
    def call(e):
        hp = ptr(None if h is None else np.asarray(h, np.float64))
        handle = e.mirror if fn == "fiesta_host_mirror_check_poses" else e.h
        extra = (None,) if fn == "fiesta_check_poses_device" else ()
        return getattr(e.L, fn)(handle, D.ctypes, n, hp, clearance, flags, I32.ctypes, I32.ctypes, I64.ctypes, *extra)
    return call


def nav_compute(lo=LO, hi=HI, goals=D, n=0, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_nav_compute(e.nav, ptr(lo), ptr(hi), ptr(goals), n, clearance, flags, None)


def nav_matrix(lo=LO, hi=HI, n_src=1, n_tgt=1, cost=D, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_nav_matrix(e.nav, ptr(lo), ptr(hi), D.ctypes, n_src, D.ctypes, n_tgt, clearance, flags, I32.ctypes, I32.ctypes,
                                           ptr(cost), None)


def nav_paths(n=1, max_len=4, starts=D):
    return lambda e: e.L.fiesta_nav_paths(e.nav, ptr(starts), n, max_len, I32.ctypes, I32.ctypes, D.ctypes, I32.ctypes)


def fr_compute(lo=LO, hi=HI, clearance=0.0, min_size=1):
    return lambda e: e.L.fiesta_frontiers_compute(e.fr, ptr(lo), ptr(hi), clearance, min_size, None)


def viewpoints(n=1, cluster=I32, orient=ORIENT, n_orient=1, sm="default", clearance=0.0, flags=0, computed=True):
    def call(e):
        s = None if sm is None else C.byref(sensor() if sm == "default" else sm)
        o = ptr(None if orient is None else np.asarray(orient, np.float64))
        cl = ptr(None if cluster is None else np.asarray(cluster, np.int32))
        return e.L.fiesta_frontiers_score_viewpoints(e.frc if computed else e.fr, cl, D.ctypes, n, o, n_orient, s, clearance, flags,
                                                     I32.ctypes, I32.ctypes, None)
    return call


def inflate(lo=LO, hi=HI, n=1, seeds=I32, steps=STEPS, clearance=0.0, flags=0):
    return lambda e: e.L.fiesta_inflate_boxes(e.h, ptr(lo), ptr(hi), ptr(seeds), I32.ctypes, n, ptr(steps), clearance, flags, I32.ctypes, I32.ctypes,
                                              I32.ctypes, None)


def corridors(off, n_paths, vox=I32, steps=STEPS, lo=LO, hi=HI):
    off = np.asarray(off, np.int64)
    return lambda e: e.L.fiesta_corridors(e.h, ptr(lo), ptr(hi), ptr(vox), off.ctypes, n_paths, ptr(steps), 0.0, 0, I32.ctypes, I32.ctypes,
                                          I32.ctypes, I32.ctypes, I32.ctypes, I32.ctypes, None)


def box_rows(tag, make):
    """A box outside the grid (below 0, at the grid size) and an inverted box, on each axis."""
    rows = []
    for k in range(3):
        for what, lo_k, hi_k in (("below", -1, None), ("past", None, GRID[k]), ("inverted", 3, 2)):
            lo, hi = LO.copy(), HI.copy()
            if lo_k is not None:
                lo[k] = lo_k
            if hi_k is not None:
                hi[k] = hi_k
            rows.append(("%s-box-%s-%d" % (tag, what, k), make(lo, hi), INVALID,
                         "%s: the box must satisfy 0 <= lo <= hi < grid size on every axis" % tag))
    return rows


def mixed_rows(fn, make):
    """A bad box and a negative max_steps together: per axis the box is checked before its max_steps, so the earlier axis wins."""
    lo, hi = LO.copy(), HI.copy()
    lo[0], hi[1] = -1, GRID[1]
    return [(fn + "-steps-before-box", make(hi=hi, steps=np.array([-1, 0, 0], np.int32)), INVALID, fn + ": max_steps must be >= 0"),
            (fn + "-box-before-steps", make(lo=lo, steps=np.array([0, -1, 0], np.int32)), INVALID,
             fn + ": the box must satisfy 0 <= lo <= hi < grid size on every axis")]


def arg_rows(fn, call):
    """The count, clearance and flag checks every planner entry point shares."""
    return [
        (fn + "-negative-count", call(n=-1), INVALID, fn + ": negative count or null buffer"),
        (fn + "-clearance-negative", call(clearance=-0.5), INVALID, fn + ": the clearance must be >= 0 and below +10000"),
        (fn + "-clearance-infinity", call(clearance=10000.0), INVALID, fn + ": the clearance must be >= 0 and below +10000"),
        (fn + "-clearance-nan", call(clearance=float("nan")), INVALID, fn + ": the clearance must be >= 0 and below +10000"),
        (fn + "-flags", call(flags=2), INVALID, fn + ": unknown flag bits"),
    ]


ROWS = (
    # segment clearance
    arg_rows("fiesta_check_segments", segments)
    + [("fiesta_check_segments-null-buffer", segments(ab=None), INVALID, "fiesta_check_segments: negative count or null buffer")]
    + arg_rows("fiesta_check_segments_device", segments_device)
    + [("fiesta_host_mirror_check_segments-negative-count", mirror_segments(), INVALID,
        "fiesta_host_mirror_check_segments: negative count or null buffer"),
       ("fiesta_host_mirror_check_segments-flags", mirror_segments(n=1, flags=4), INVALID,
        "fiesta_host_mirror_check_segments: unknown flag bits")]
    # robot-shaped collision checks
    + arg_rows("fiesta_check_poses", poses)
    + [("fiesta_check_poses-null-half-extents", poses(h=None), INVALID, "fiesta_check_poses: null half_extents"),
       ("fiesta_check_poses-half-extent-negative", poses(h=(0.1, -0.1, 0.1)), INVALID,
        "fiesta_check_poses: half extents must be finite and >= 0"),
       ("fiesta_check_poses-half-extent-nan", poses(h=(0.1, 0.1, float("nan"))), INVALID,
        "fiesta_check_poses: half extents must be finite and >= 0"),
       ("fiesta_check_poses-half-extent-inf", poses(h=(float("inf"), 0.1, 0.1)), INVALID,
        "fiesta_check_poses: half extents must be finite and >= 0"),
       ("fiesta_check_poses-span", poses(h=(10.0, 10.0, 10.0)), LIMIT, "fiesta_check_poses: h0 + h1 + h2 = 30 m exceeds 256 voxels"),
       ("fiesta_check_poses-count", poses(n=2 ** 31 - 1), LIMIT, "fiesta_check_poses: n = 2147483647 poses, the limit is 2^31 - 2"),
       ("fiesta_check_poses_device-null-half-extents", poses(h=None, fn="fiesta_check_poses_device"), INVALID,
        "fiesta_check_poses_device: null half_extents"),
       ("fiesta_check_poses_device-negative-count", poses(n=-1, fn="fiesta_check_poses_device"), INVALID,
        "fiesta_check_poses_device: negative count or null buffer"),
       ("fiesta_check_poses_device-span", poses(h=(0.0, 30.0, 0.0), fn="fiesta_check_poses_device"), LIMIT,
        "fiesta_check_poses_device: h0 + h1 + h2 = 30 m exceeds 256 voxels"),
       ("fiesta_host_mirror_check_poses-half-extent-negative", poses(h=(-1.0, 0.0, 0.0), fn="fiesta_host_mirror_check_poses"), INVALID,
        "fiesta_host_mirror_check_poses: half extents must be finite and >= 0"),
       ("fiesta_host_mirror_check_poses-clearance", poses(clearance=-1.0, fn="fiesta_host_mirror_check_poses"), INVALID,
        "fiesta_host_mirror_check_poses: the clearance must be >= 0 and below +10000")]
    # point queries on device buffers
    + [("fiesta_get_distance_batch_device-negative-count", lambda e: e.L.fiesta_get_distance_batch_device(e.h, None, -1, None, None),
        INVALID, "fiesta_get_distance_batch_device: bad argument"),
       ("fiesta_get_dist_grad_trilinear_batch_device-null-buffer",
        lambda e: e.L.fiesta_get_dist_grad_trilinear_batch_device(e.h, None, 1, None, None, None), INVALID,
        "fiesta_get_dist_grad_trilinear_batch_device: bad argument")]
    # cost-to-go fields
    + [("fiesta_nav_create-null", lambda e: e.L.fiesta_nav_create(e.h, None), INVALID, "fiesta_nav_create: null argument"),
       ("fiesta_nav_compute-null", nav_compute(lo=None), INVALID, "fiesta_nav_compute: null argument"),
       ("fiesta_nav_compute-negative-count", nav_compute(n=-1), INVALID, "fiesta_nav_compute: negative count or null buffer"),
       ("fiesta_nav_compute-null-goals", nav_compute(goals=None, n=1), INVALID, "fiesta_nav_compute: negative count or null buffer"),
       ("fiesta_nav_compute-clearance", nav_compute(clearance=-1.0), INVALID,
        "fiesta_nav_compute: the clearance must be >= 0 and below +10000"),
       ("fiesta_nav_compute-flags", nav_compute(flags=8), INVALID, "fiesta_nav_compute: unknown flag bits")]
    + box_rows("fiesta_nav_compute", lambda lo, hi: nav_compute(lo=lo, hi=hi))
    + [("fiesta_nav_update-null", lambda e: e.L.fiesta_nav_update(None, None), INVALID, "fiesta_nav_update: null argument"),
       ("fiesta_nav_update-no-field", lambda e: e.L.fiesta_nav_update(e.nav, None), INVALID,
        "fiesta_nav_update: no field has been computed"),
       ("fiesta_nav_export-null", lambda e: e.L.fiesta_nav_export(e.nav, None), INVALID, "fiesta_nav_export: null argument"),
       ("fiesta_nav_export-no-field", lambda e: e.L.fiesta_nav_export(e.nav, D.ctypes), INVALID,
        "fiesta_nav_export: no field has been computed"),
       ("fiesta_nav_paths-max-len", nav_paths(max_len=0), INVALID, "fiesta_nav_paths: null buffer, negative count or max_len < 1"),
       ("fiesta_nav_paths-negative-count", nav_paths(n=-1), INVALID, "fiesta_nav_paths: null buffer, negative count or max_len < 1"),
       ("fiesta_nav_paths-null-buffer", nav_paths(starts=None), INVALID, "fiesta_nav_paths: null buffer, negative count or max_len < 1"),
       ("fiesta_nav_paths-no-field", nav_paths(), INVALID, "fiesta_nav_paths: no field has been computed"),
       ("fiesta_nav_matrix-null", nav_matrix(hi=None), INVALID, "fiesta_nav_matrix: null argument"),
       ("fiesta_nav_matrix-negative-count", nav_matrix(n_tgt=-1), INVALID, "fiesta_nav_matrix: negative count or null buffer"),
       ("fiesta_nav_matrix-null-cost", nav_matrix(cost=None), INVALID, "fiesta_nav_matrix: negative count or null buffer"),
       ("fiesta_nav_matrix-clearance", nav_matrix(clearance=float("inf")), INVALID,
        "fiesta_nav_matrix: the clearance must be >= 0 and below +10000"),
       ("fiesta_nav_matrix-flags", nav_matrix(flags=-1), INVALID, "fiesta_nav_matrix: unknown flag bits"),
       ("fiesta_nav_matrix-size", nav_matrix(n_src=65536, n_tgt=32768), LIMIT, "fiesta_nav_matrix: n_src * n_tgt must be below 2^31")]
    + box_rows("fiesta_nav_matrix", lambda lo, hi: nav_matrix(lo=lo, hi=hi))
    # frontiers and viewpoints
    + [("fiesta_frontiers_create-null", lambda e: e.L.fiesta_frontiers_create(e.h, None), INVALID,
        "fiesta_frontiers_create: null argument"),
       ("fiesta_frontiers_compute-null", fr_compute(lo=None), INVALID, "fiesta_frontiers_compute: null argument"),
       ("fiesta_frontiers_compute-clearance", fr_compute(clearance=-0.1), INVALID,
        "fiesta_frontiers_compute: the clearance must be >= 0 and below +10000"),
       ("fiesta_frontiers_compute-min-cluster-size", fr_compute(min_size=0), INVALID,
        "fiesta_frontiers_compute: min_cluster_size must be >= 1")]
    + box_rows("fiesta_frontiers_compute", lambda lo, hi: fr_compute(lo=lo, hi=hi))
    + [("fiesta_frontiers_clusters-negative-cap", lambda e: e.L.fiesta_frontiers_clusters(e.frc, -1, *[None] * 5), INVALID,
        "fiesta_frontiers_clusters: null buffer or negative capacity"),
       ("fiesta_frontiers_clusters-null-buffer", lambda e: e.L.fiesta_frontiers_clusters(e.frc, 1, *[None] * 5), INVALID,
        "fiesta_frontiers_clusters: null buffer or negative capacity"),
       ("fiesta_frontiers_clusters-none", lambda e: e.L.fiesta_frontiers_clusters(e.fr, 0, *[None] * 5), INVALID,
        "fiesta_frontiers_clusters: no frontiers have been computed"),
       ("fiesta_frontiers_voxels-null-buffer", lambda e: e.L.fiesta_frontiers_voxels(e.frc, 2, None), INVALID,
        "fiesta_frontiers_voxels: null buffer or negative capacity"),
       ("fiesta_frontiers_voxels-none", lambda e: e.L.fiesta_frontiers_voxels(e.fr, 0, None), INVALID,
        "fiesta_frontiers_voxels: no frontiers have been computed"),
       ("fiesta_frontiers_export-null", lambda e: e.L.fiesta_frontiers_export(e.frc, None), INVALID,
        "fiesta_frontiers_export: null argument"),
       ("fiesta_frontiers_export-none", lambda e: e.L.fiesta_frontiers_export(e.fr, I32.ctypes), INVALID,
        "fiesta_frontiers_export: no frontiers have been computed")]
    + [("fiesta_frontiers_score_viewpoints-null-sensor", viewpoints(sm=None), INVALID, "fiesta_frontiers_score_viewpoints: null argument"),
       ("fiesta_frontiers_score_viewpoints-null-orient", viewpoints(orient=None), INVALID,
        "fiesta_frontiers_score_viewpoints: null argument"),
       ("fiesta_frontiers_score_viewpoints-null-buffer", viewpoints(cluster=None), INVALID,
        "fiesta_frontiers_score_viewpoints: negative count or null buffer")]
    + arg_rows("fiesta_frontiers_score_viewpoints", viewpoints)
    + [("fiesta_frontiers_score_viewpoints-none", viewpoints(computed=False), INVALID,
        "fiesta_frontiers_score_viewpoints: no frontiers have been computed"),
       ("fiesta_frontiers_score_viewpoints-no-orientation", viewpoints(n_orient=0), INVALID,
        "fiesta_frontiers_score_viewpoints: n_orient must be >= 1"),
       ("fiesta_frontiers_score_viewpoints-range", viewpoints(sm=sensor(max_range=0.0)), INVALID,
        "fiesta_frontiers_score_viewpoints: max_range and tan_half_fov must be finite and > 0"),
       ("fiesta_frontiers_score_viewpoints-fov", viewpoints(sm=sensor(tan_v=float("nan"))), INVALID,
        "fiesta_frontiers_score_viewpoints: max_range and tan_half_fov must be finite and > 0"),
       ("fiesta_frontiers_score_viewpoints-orientations", viewpoints(orient=np.tile(ORIENT, 33), n_orient=33), LIMIT,
        "fiesta_frontiers_score_viewpoints: at most 32 orientations per call"),
       ("fiesta_frontiers_score_viewpoints-orientation-nan", viewpoints(orient=np.r_[ORIENT[:4], np.nan, ORIENT[5:]]), INVALID,
        "fiesta_frontiers_score_viewpoints: orientation entry 4 is not finite"),
       ("fiesta_frontiers_score_viewpoints-cluster", viewpoints(cluster=[3]), INVALID,
        "fiesta_frontiers_score_viewpoints: cluster[0] = 3 is not a kept cluster id (there are 0)")]
    # safe flight corridors
    + [("fiesta_inflate_boxes-null", inflate(steps=None), INVALID, "fiesta_inflate_boxes: null argument"),
       ("fiesta_inflate_boxes-null-buffer", inflate(seeds=None), INVALID, "fiesta_inflate_boxes: negative count or null buffer"),
       ("fiesta_inflate_boxes-max-steps", inflate(steps=np.array([0, -1, 0], np.int32)), INVALID,
        "fiesta_inflate_boxes: max_steps must be >= 0"),
       ("fiesta_inflate_boxes-count", inflate(n=2 ** 31 - 1), LIMIT, "fiesta_inflate_boxes: at most 2^31 - 2 seeds per call")]
    + arg_rows("fiesta_inflate_boxes", inflate)
    + box_rows("fiesta_inflate_boxes", lambda lo, hi: inflate(lo=lo, hi=hi))
    + mixed_rows("fiesta_inflate_boxes", inflate)
    + mixed_rows("fiesta_corridors", lambda **kw: corridors([0], 0, **kw))
    + [("fiesta_corridors-negative-count", corridors([0], -1), INVALID, "fiesta_corridors: negative count or null buffer"),
       ("fiesta_corridors-max-steps", corridors([0], 0, steps=np.array([-2, 0, 0], np.int32)), INVALID,
        "fiesta_corridors: max_steps must be >= 0"),
       ("fiesta_corridors-first-offset", corridors([1, 2], 1), INVALID, "fiesta_corridors: path_off[0] must be 0"),
       ("fiesta_corridors-decreasing-offset", corridors([0, 3, 2], 2), INVALID, "fiesta_corridors: path_off decreases at 1"),
       ("fiesta_corridors-null-buffer", corridors([0, 2], 1, vox=None), INVALID, "fiesta_corridors: null buffer"),
       ("fiesta_corridors-count", corridors([0, 2 ** 31 - 1], 1), LIMIT, "fiesta_corridors: at most 2^31 - 2 path voxels per call")]
    # handles
    + [("fiesta_query_plan_create-count", lambda e: e.L.fiesta_query_plan_create(e.h, 0, C.byref(C.c_void_p())), INVALID,
        "fiesta_query_plan_create: bad argument"),
       ("fiesta_host_mirror_create-null", lambda e: e.L.fiesta_host_mirror_create(e.h, None), INVALID,
        "fiesta_host_mirror_create: null argument"),
       ("fiesta_host_mirror_create-twice", lambda e: e.L.fiesta_host_mirror_create(e.h, C.byref(C.c_void_p())), INVALID,
        "fiesta_host_mirror_create: this map already has a host mirror")]
)


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_error_text(env, row):
    _, call, rc, msg = row
    assert env.L.fiesta_nav_create(None, None) == INVALID and env.L.fiesta_last_error().decode() == SENTINEL
    assert (call(env), env.L.fiesta_last_error().decode()) == (rc, msg)


def test_ids_unique():
    assert len({r[0] for r in ROWS}) == len(ROWS)


# ---- states of a whole map: each row builds its own
def save(m, buf=None, cap=0):
    n = C.c_int64(-1)
    rc = m._L.fiesta_snapshot_save(m._h, buf, cap, C.byref(n))
    return rc, n.value


def obstacle(m):
    assert m.SetOccupancy((3, 4, 5), 1) >= 0


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_snapshot_save_errors(mode):
    m = new_map(mode)
    L = m._L
    assert L.fiesta_snapshot_save(m._h, None, -1, None) == INVALID
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: bad argument"
    obstacle(m)
    assert save(m) == (INVALID, 0)
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: SetOccupancy events are staged (UpdateOccupancy has not run)"
    m.export_counters()                                  # the events are applied: the occupancy queue holds their tile
    assert save(m) == (INVALID, 0)
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: the occupancy queue is not empty (UpdateOccupancy has not run)"
    assert m.UpdateOccupancy(True)
    assert save(m) == (INVALID, 0)
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: inserts or deletes are pending (UpdateESDF has not run)"
    m.UpdateESDF()
    rc, size = save(m)
    assert rc == 0 and size > SNAP_HDR
    small = np.zeros(8, np.uint8)
    assert save(m, small.ctypes.data, 8) == (LIMIT, size)
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: the buffer holds 8 bytes, the snapshot needs %d" % size
    if mode == "fast":
        m.set_shard(0, 2)
        assert save(m) == (INVALID, 0)
        assert L.fiesta_last_error().decode() == "fiesta_snapshot_save: an x-slab shard cannot be saved"
    m.close()


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_snapshot_load_errors(mode):
    m = new_map(mode)
    L = m._L
    obstacle(m)
    m.UpdateOccupancy(True)
    m.UpdateESDF()
    buf = np.frombuffer(m.save(), np.uint8).copy()
    m.close()
    out = C.c_void_p()
    assert L.fiesta_snapshot_load(buf.ctypes.data, len(buf), 0, None) == INVALID
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_load: null argument"
    assert L.fiesta_snapshot_load(None, len(buf), 0, C.byref(out)) == INVALID and not out
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_load: bad argument"
    assert L.fiesta_snapshot_load(buf.ctypes.data, 10, 0, C.byref(out)) == INVALID and not out
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_load: truncated: 10 bytes, the header alone is %d" % SNAP_HDR
    assert L.fiesta_snapshot_load(buf.ctypes.data, len(buf) - 8, 0, C.byref(out)) == INVALID and not out
    assert L.fiesta_last_error().decode() == "fiesta_snapshot_load: stream is %d bytes, its header describes %d" % (len(buf) - 8, len(buf))
    assert L.fiesta_snapshot_load(buf.ctypes.data, len(buf), 0, C.byref(out)) == 0 and out
    L.fiesta_destroy(out)


def test_query_plan_needs_parameters():
    m = new_map("fast", params=False)
    assert m._L.fiesta_query_plan_create(m._h, 16, C.byref(C.c_void_p())) == INVALID
    assert m._L.fiesta_last_error().decode() == "fiesta_query_plan_create: call SetParameters first (the occupancy threshold is captured)"
    m.close()
