"""fiesta_b200 -- H100-native (sm_90a) implementation of FIESTA's incremental ESDF hot path.

The product is the C-ABI shared library `fiesta_b200/lib/libfiesta_b200.so` (declared in include/fiesta_b200.h,
built from fiesta_b200/csrc/*.cu by `fiesta_b200.build.build()`); C++ callers use the drop-in facade
include/fiesta_b200/ESDFMap.h.  This module is only the ctypes binding that tests/ and bench.py drive it with:
`ESDFMap` mirrors the reference class's public surface (FIESTA include/ESDFMap.h:111-164) method for method.

There is no CPU fallback: importing works anywhere, but creating a map without the compiled library or without an
sm_90 GPU raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libfiesta_b200.so")

UNDEFINED = -10000
INFINITY = 10000

D3 = C.c_double * 3
I3 = C.c_int * 3


class Config(C.Structure):
    _fields_ = [("origin", C.c_double * 3), ("resolution", C.c_double), ("map_size", C.c_double * 3),
                ("device", C.c_int32), ("mode", C.c_int32), ("reserved", C.c_int32 * 6)]


class RaycastParams(C.Structure):
    _fields_ = [("min_ray_length", C.c_double), ("max_ray_length", C.c_double)]


class DepthParams(C.Structure):
    _fields_ = [("focal_x", C.c_double), ("focal_y", C.c_double), ("center_x", C.c_double), ("center_y", C.c_double), ("use_depth_filter", C.c_int32),
                ("depth_filter_margin", C.c_int32), ("depth_filter_max_dist", C.c_double), ("depth_filter_min_dist", C.c_double),
                ("depth_filter_tolerance", C.c_double)]


class ShardInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("rank", "world", "x_begin", "x_end", "has_lo", "has_hi")] + [("layer_words", C.c_int64)]


class NavStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "blocked", "reached", "goals_placed", "generations", "tile_visits")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class NavUpdateStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "became_blocked", "became_free", "withdrawn", "goals_placed", "goals_new",
                                         "seed_tiles", "withdraw_generations", "generations", "tile_visits", "blocked", "reached")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class NavMatrixStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("sources_placed", "targets_placed", "passes", "generations", "tile_visits",
                                         "sources_retired_early")] + [("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class SignedStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "obstacles", "interior", "max_depth_sq")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class FrontierStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "frontier_voxels", "clusters", "kept_clusters", "kept_voxels")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class SkeletonStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "traversable", "anchors")] + [("iterations", C.c_int64 * 2)] + [
        (n, C.c_int64) for n in ("prune_rounds", "pruned_voxels", "skeleton_voxels", "vertices", "edges", "edge_voxels")] + [
        (n, C.c_float) for n in ("ms_compute", "ms_init", "ms_thin", "ms_graph")]


class MeshStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("box_voxels", "blocking", "vertices", "quads", "triangles")] + [
        (n, C.c_float) for n in ("ms_compute", "ms_classify", "ms_vertices", "ms_faces")]


class SensorModel(C.Structure):
    _fields_ = [("max_range", C.c_double), ("tan_half_fov", C.c_double * 2)]


class ViewpointStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("candidates_scored", "pairs_walked", "pairs_visible")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class CorridorStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("boxes", "layers_tested", "layers_grown", "mask_voxels")] + [
        ("ms_compute", C.c_float), ("reserved_f", C.c_float * 1)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        "occupancy_updates", "inserts", "deletes", "voxels_changed", "expansions", "voxels_reset", "tile_visits", "generations",
        "rays_cast", "rays_dropped", "ray_voxels", "raycast_rounds", "touched_voxels", "kernel_launches")] + [
        (n, C.c_float) for n in ("ms_raycast", "ms_update_occupancy", "ms_update_esdf", "ms_esdf_delete_scan",
                                 "ms_esdf_wavefront")] + [("reserved_f", C.c_float * 1)]

    def asdict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved_f"}


# every symbol include/fiesta_b200.h declares
SYMBOLS = [
    "fiesta_create", "fiesta_destroy", "fiesta_last_error", "fiesta_set_parameters", "fiesta_grid_total_size",
    "fiesta_grid_size", "fiesta_set_occupancy_pos", "fiesta_set_occupancy_vox", "fiesta_set_occupancy_batch_pos",
    "fiesta_set_occupancy_batch_vox", "fiesta_raycast_frame", "fiesta_raycast_frame_device", "fiesta_check_update",
    "fiesta_update_occupancy", "fiesta_update_esdf", "fiesta_set_update_range", "fiesta_set_original_range",
    "fiesta_get_distance_pos", "fiesta_get_distance_vox", "fiesta_get_occupancy_pos", "fiesta_get_occupancy_vox",
    "fiesta_get_dist_grad_trilinear", "fiesta_get_distance_batch_pos", "fiesta_get_dist_grad_trilinear_batch",
    "fiesta_export_distance", "fiesta_export_closest_obstacle", "fiesta_export_occupancy", "fiesta_export_counters",
    "fiesta_get_stats", "fiesta_synchronize", "fiesta_set_shard", "fiesta_shard_pack", "fiesta_shard_ingest", "fiesta_shard_relax", "fiesta_get_point_cloud", "fiesta_get_slice_marker", "fiesta_set_occupancy_batch_vox_device", "fiesta_depth_frame", "fiesta_last_depth_cloud",
    "fiesta_query_plan_create", "fiesta_query_plan_destroy", "fiesta_query_plan_positions", "fiesta_query_plan_distances",
    "fiesta_query_plan_gradients", "fiesta_query_plan_run",
    "fiesta_host_mirror_create", "fiesta_host_mirror_destroy", "fiesta_host_mirror_refresh", "fiesta_host_mirror_get_distance_pos",
    "fiesta_host_mirror_get_distance_vox", "fiesta_host_mirror_get_dist_grad_trilinear", "fiesta_host_mirror_get_distance_batch_pos",
    "fiesta_host_mirror_get_dist_grad_trilinear_batch", "fiesta_host_mirror_records", "fiesta_host_mirror_stats",
    "fiesta_check_segments", "fiesta_check_segments_device", "fiesta_get_distance_batch_device",
    "fiesta_get_dist_grad_trilinear_batch_device", "fiesta_host_mirror_check_segments",
    "fiesta_nav_create", "fiesta_nav_destroy", "fiesta_nav_compute", "fiesta_nav_export", "fiesta_nav_paths",
    "fiesta_nav_matrix", "fiesta_nav_update",
    "fiesta_frontiers_create", "fiesta_frontiers_destroy", "fiesta_frontiers_compute", "fiesta_frontiers_clusters",
    "fiesta_frontiers_voxels", "fiesta_frontiers_export", "fiesta_frontiers_score_viewpoints",
    "fiesta_inflate_boxes", "fiesta_corridors",
    "fiesta_check_poses", "fiesta_check_poses_device", "fiesta_host_mirror_check_poses",
    "fiesta_snapshot_save", "fiesta_snapshot_load", "fiesta_get_config",
    "fiesta_signed_create", "fiesta_signed_destroy", "fiesta_signed_compute", "fiesta_signed_export",
    "fiesta_signed_get_distance_batch", "fiesta_signed_get_dist_grad_trilinear_batch", "fiesta_signed_get_distance_batch_device",
    "fiesta_signed_get_dist_grad_trilinear_batch_device",
    "fiesta_skeleton_create", "fiesta_skeleton_destroy", "fiesta_skeleton_compute", "fiesta_skeleton_vertices",
    "fiesta_skeleton_edges", "fiesta_skeleton_edge_voxels", "fiesta_skeleton_export",
    "fiesta_mesh_create", "fiesta_mesh_destroy", "fiesta_mesh_compute", "fiesta_mesh_vertices", "fiesta_mesh_triangles",
]

SEGMENT_UNKNOWN_BLOCKS = 1     # FIESTA_SEGMENT_UNKNOWN_BLOCKS

_lib = None


class FiestaError(RuntimeError):
    pass


def load_library():
    """dlopen the product library; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FiestaError("%s is missing: run `python -m fiesta_b200.build` (nvcc, sm_90a). There is no CPU "
                              "fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.fiesta_last_error.restype = C.c_char_p
        for n in ("fiesta_get_distance_pos", "fiesta_get_distance_vox", "fiesta_get_dist_grad_trilinear"):
            getattr(L, n).restype = C.c_double
        L.fiesta_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
        L.fiesta_destroy.argtypes = [C.c_void_p]
        L.fiesta_destroy.restype = None
        L.fiesta_query_plan_create.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_void_p)]
        L.fiesta_query_plan_destroy.argtypes = [C.c_void_p]
        L.fiesta_query_plan_destroy.restype = None
        L.fiesta_query_plan_run.argtypes = [C.c_void_p]
        L.fiesta_host_mirror_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_host_mirror_destroy.argtypes = [C.c_void_p]
        L.fiesta_host_mirror_destroy.restype = None
        L.fiesta_host_mirror_refresh.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.fiesta_host_mirror_get_distance_pos.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_host_mirror_get_distance_pos.restype = C.c_double
        L.fiesta_host_mirror_get_distance_vox.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_host_mirror_get_distance_vox.restype = C.c_double
        L.fiesta_host_mirror_get_dist_grad_trilinear.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.fiesta_host_mirror_get_dist_grad_trilinear.restype = C.c_double
        L.fiesta_host_mirror_get_distance_batch_pos.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_host_mirror_get_dist_grad_trilinear_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.fiesta_host_mirror_records.argtypes = [C.c_void_p]
        L.fiesta_host_mirror_records.restype = C.POINTER(C.c_uint32)
        L.fiesta_host_mirror_stats.argtypes = [C.c_void_p, C.c_void_p]
        for n in ("fiesta_query_plan_positions", "fiesta_query_plan_distances", "fiesta_query_plan_gradients"):
            getattr(L, n).argtypes = [C.c_void_p]
            getattr(L, n).restype = C.POINTER(C.c_double)
        seg = [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int] + [C.c_void_p] * 4
        L.fiesta_check_segments.argtypes = seg
        L.fiesta_host_mirror_check_segments.argtypes = seg
        L.fiesta_check_segments_device.argtypes = seg + [C.c_void_p]
        pose = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 3
        L.fiesta_check_poses.argtypes = pose
        L.fiesta_host_mirror_check_poses.argtypes = pose
        L.fiesta_check_poses_device.argtypes = pose + [C.c_void_p]
        L.fiesta_nav_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_nav_destroy.argtypes = [C.c_void_p]
        L.fiesta_nav_destroy.restype = None
        L.fiesta_nav_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int, C.c_void_p]
        L.fiesta_nav_export.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_nav_paths.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32] + [C.c_void_p] * 4
        L.fiesta_nav_update.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_nav_matrix.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_int64, C.c_double, C.c_int] + [C.c_void_p] * 4
        L.fiesta_signed_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_signed_destroy.argtypes = [C.c_void_p]
        L.fiesta_signed_destroy.restype = None
        L.fiesta_signed_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fiesta_signed_export.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_signed_get_distance_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_signed_get_dist_grad_trilinear_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.fiesta_signed_get_distance_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.fiesta_signed_get_dist_grad_trilinear_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                                         C.c_void_p]
        L.fiesta_frontiers_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_frontiers_destroy.argtypes = [C.c_void_p]
        L.fiesta_frontiers_destroy.restype = None
        L.fiesta_frontiers_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int64, C.c_void_p]
        L.fiesta_frontiers_clusters.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5
        L.fiesta_frontiers_voxels.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_frontiers_export.argtypes = [C.c_void_p, C.c_void_p]
        L.fiesta_frontiers_score_viewpoints.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32,
                                                        C.POINTER(SensorModel), C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fiesta_skeleton_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_skeleton_destroy.argtypes = [C.c_void_p]
        L.fiesta_skeleton_destroy.restype = None
        L.fiesta_skeleton_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_double, C.c_int64, C.c_void_p]
        L.fiesta_skeleton_vertices.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 4
        L.fiesta_skeleton_edges.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 4
        L.fiesta_skeleton_edge_voxels.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_skeleton_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.fiesta_mesh_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.fiesta_mesh_destroy.argtypes = [C.c_void_p]
        L.fiesta_mesh_destroy.restype = None
        L.fiesta_mesh_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p]
        L.fiesta_mesh_vertices.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_mesh_triangles.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.fiesta_inflate_boxes.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 4
        L.fiesta_corridors.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 7
        L.fiesta_snapshot_save.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.fiesta_snapshot_load.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.POINTER(C.c_void_p)]
        L.fiesta_get_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.fiesta_get_distance_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.fiesta_get_dist_grad_trilinear_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _is_cuda_tensor(a):
    return getattr(a, "is_cuda", False) is True


def _segment_flags(clearance, unknown_blocks):
    return C.c_double(float(clearance)), SEGMENT_UNKNOWN_BLOCKS if unknown_blocks else 0


def _check_segments_host(fn, h, ab, clearance, unknown_blocks, ck):
    """fiesta_check_segments / fiesta_host_mirror_check_segments on host arrays: (status, hit_idx, hit_t, min_dist)."""
    ab = _f64(ab).reshape(-1, 6)
    n = len(ab)
    out = (np.empty(n, np.int32), np.empty(n, np.int64), np.empty(n), np.empty(n))
    r, flags = _segment_flags(clearance, unknown_blocks)
    ck(fn(h, ab.ctypes, C.c_int64(n), r, flags, *(o.ctypes for o in out)), "CheckSegments")
    return out


def _half_extents(h):
    h = _f64(h)
    if h.shape != (3,):
        raise ValueError("CheckPoses: half_extents must be 3 numbers, got shape %s" % (h.shape,))
    return h


def _check_poses_host(fn, h, poses, half_extents, clearance, unknown_blocks, ck):
    """fiesta_check_poses / fiesta_host_mirror_check_poses on host arrays: (status, n_blocked, hit_idx)."""
    poses = _f64(poses).reshape(-1, 12)
    n = len(poses)
    he = _half_extents(half_extents)
    out = (np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int64))
    r, flags = _segment_flags(clearance, unknown_blocks)
    ck(fn(h, poses.ctypes, C.c_int64(n), he.ctypes, r, flags, *(o.ctypes for o in out)), "CheckPoses")
    return out


class QueryPlan:
    """fiesta_query_plan: positions in, distances + gradients out, one graph launch per run()."""

    def __init__(self, m, n):
        self._m, self.n = m, int(n)
        h = C.c_void_p()
        m._ck(m._L.fiesta_query_plan_create(m._h, self.n, C.byref(h)), "fiesta_query_plan_create")
        self._h = h
        self.positions = np.ctypeslib.as_array(m._L.fiesta_query_plan_positions(h), shape=(self.n, 3))
        self.distances = np.ctypeslib.as_array(m._L.fiesta_query_plan_distances(h), shape=(self.n,))
        self.gradients = np.ctypeslib.as_array(m._L.fiesta_query_plan_gradients(h), shape=(self.n, 3))

    def run(self, pos=None):
        if pos is not None:
            self.positions[:] = pos
        self._m._ck(self._m._L.fiesta_query_plan_run(self._h), "fiesta_query_plan_run")
        return self.distances, self.gradients

    def close(self):
        if self._h:
            self._m._L.fiesta_query_plan_destroy(self._h)
            self._h = None


class HostMirror:
    """fiesta_host_mirror: the distance records in pinned host memory, patched from the device by refresh(); the getters are
    pure host code (no CUDA call) and return the bits of the device queries as of the last refresh."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_host_mirror_create(m._h, C.byref(h)), "fiesta_host_mirror_create")
        self._h = h

    def refresh(self):
        n = C.c_int64(0)
        self._m._ck(self._m._L.fiesta_host_mirror_refresh(self._h, C.byref(n)), "fiesta_host_mirror_refresh")
        return n.value

    def stats(self):
        a = np.zeros(4, np.int64)
        self._m._ck(self._m._L.fiesta_host_mirror_stats(self._h, a.ctypes), "fiesta_host_mirror_stats")
        return dict(zip(("changed", "scanned", "refreshes", "full_copies"), (int(x) for x in a)))

    def GetDistance(self, p):
        if all(isinstance(x, (int, np.integer)) for x in p):
            v = np.ascontiguousarray(p, dtype=np.int32)
            return float(self._m._L.fiesta_host_mirror_get_distance_vox(self._h, v.ctypes))
        return float(self._m._L.fiesta_host_mirror_get_distance_pos(self._h, _f64(p).ctypes))

    def GetDistWithGradTrilinear(self, pos):
        g = np.zeros(3)
        d = float(self._m._L.fiesta_host_mirror_get_dist_grad_trilinear(self._h, _f64(pos).ctypes, g.ctypes))
        return d, g

    def GetDistanceBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        d = np.empty(len(pos))
        self._m._ck(self._m._L.fiesta_host_mirror_get_distance_batch_pos(self._h, pos.ctypes, C.c_int64(len(pos)), d.ctypes), "mirror batch")
        return d

    def GetDistWithGradTrilinearBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        d = np.empty(len(pos))
        g = np.empty((len(pos), 3))
        self._m._ck(self._m._L.fiesta_host_mirror_get_dist_grad_trilinear_batch(self._h, pos.ctypes, C.c_int64(len(pos)), d.ctypes, g.ctypes),
                    "mirror trilinear batch")
        return d, g

    def CheckSegments(self, ab, clearance, unknown_blocks=False):
        """Segment clearance from the pinned records (fiesta_host_mirror_check_segments): ab (n,6) -> (status, hit_idx, hit_t, min_dist)."""
        return _check_segments_host(self._m._L.fiesta_host_mirror_check_segments, self._h, ab, clearance, unknown_blocks, self._m._ck)

    def CheckPoses(self, poses, half_extents, clearance, unknown_blocks=False):
        """Robot-shaped collision checks from the pinned records (fiesta_host_mirror_check_poses): poses (n, 12) ->
        (status, n_blocked, hit_idx)."""
        return _check_poses_host(self._m._L.fiesta_host_mirror_check_poses, self._h, poses, half_extents, clearance, unknown_blocks,
                                 self._m._ck)

    def close(self):
        if self._h:
            self._m._L.fiesta_host_mirror_destroy(self._h)
            self._h = None


class NavField:
    """fiesta_nav_field: cost-to-go field of a voxel box -- geodesic distance to a goal set through free space at a clearance --
    and path extraction down it.  The buffers grow to the largest box computed; close() it before the map."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_nav_create(m._h, C.byref(h)), "fiesta_nav_create")
        self._h = h
        self.shape = None

    def compute(self, box_lo, box_hi, goals, clearance, unknown_blocks=False):
        """Field over the inclusive voxel box [box_lo, box_hi] for goals (n, 3) in metres -> stats dict."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("NavField.compute: box_lo and box_hi must be 3 voxel coordinates each")
        goals = _f64(goals).reshape(-1, 3)
        st = NavStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._m._ck(self._m._L.fiesta_nav_compute(self._h, lo.ctypes, hi.ctypes, goals.ctypes, C.c_int64(len(goals)), r, flags, C.byref(st)),
                    "NavField.compute")
        self.shape = tuple(int(b - a + 1) for a, b in zip(lo, hi))
        return {n: getattr(st, n) for n, _ in st._fields_ if n != "reserved_f"}

    def update(self):
        """Repair the field after map updates (fiesta_nav_update): afterwards it is bit for bit what compute() with the last box,
        goals, clearance and flags would give on the current records -> stats dict."""
        st = NavUpdateStats()
        self._m._ck(self._m._L.fiesta_nav_update(self._h, C.byref(st)), "NavField.update")
        return {n: getattr(st, n) for n, _ in st._fields_ if n != "reserved_f"}

    def export(self):
        """The last computed field as a (Bx, By, Bz) float64 array: -1 blocked, +inf unreachable."""
        if self.shape is None:
            raise FiestaError("NavField.export: no field has been computed")
        out = np.empty(self.shape)
        self._m._ck(self._m._L.fiesta_nav_export(self._h, out.ctypes), "NavField.export")
        return out

    def paths(self, starts, max_len):
        """Paths from starts (n, 3) in metres -> (status (n,), len (n,), cost (n,), vox (n, max_len, 3) grid voxels, -1 past len)."""
        starts = _f64(starts).reshape(-1, 3)
        n = len(starts)
        st, ln, cost = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n)
        vox = np.empty((n, int(max_len), 3), np.int32)
        self._m._ck(self._m._L.fiesta_nav_paths(self._h, starts.ctypes, C.c_int64(n), C.c_int32(int(max_len)), st.ctypes, ln.ctypes,
                                                cost.ctypes, vox.ctypes), "NavField.paths")
        return st, ln, cost, vox

    def matrix(self, box_lo, box_hi, sources, targets, clearance, unknown_blocks=False):
        """Geodesic costs from every source to every target (positions (n, 3) in metres) through the free space of the inclusive voxel
        box [box_lo, box_hi] -> (cost (n_src, n_tgt), src_status (n_src,), tgt_status (n_tgt,), stats dict).  Row i is the field
        of compute(goals=[source i]) read at the targets; NaN where a point's status is not 0.  The last computed field, its
        export() and paths() are left as they were."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("NavField.matrix: box_lo and box_hi must be 3 voxel coordinates each")
        src, tgt = _f64(sources).reshape(-1, 3), _f64(targets).reshape(-1, 3)
        ns, nt = len(src), len(tgt)
        cost = np.empty((ns, nt))
        ss, ts = np.empty(ns, np.int32), np.empty(nt, np.int32)
        st = NavMatrixStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._m._ck(self._m._L.fiesta_nav_matrix(self._h, lo.ctypes, hi.ctypes, src.ctypes, C.c_int64(ns), tgt.ctypes, C.c_int64(nt), r,
                                                 flags, ss.ctypes, ts.ctypes, cost.ctypes, C.byref(st)), "NavField.matrix")
        return cost, ss, ts, {n: getattr(st, n) for n, _ in st._fields_ if n != "reserved_f"}

    def close(self):
        if self._h:
            self._m._L.fiesta_nav_destroy(self._h)
            self._h = None


class SignedField:
    """fiesta_signed_field: signed distance over a voxel box -- FIESTA's distance outside obstacles, minus the exact Euclidean depth
    inside them -- with GetDistance / GetDistWithGradTrilinear queries that read it inside the box and the map elsewhere.  A field
    refuses export and queries after UpdateOccupancy / UpdateESDF until it is computed again.  The buffers grow to the largest box
    computed; close() it before the map."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_signed_create(m._h, C.byref(h)), "fiesta_signed_create")
        self._h = h
        self.shape = None

    def compute(self, box_lo, box_hi):
        """Field over the inclusive voxel box [box_lo, box_hi] -> stats dict."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("SignedField.compute: box_lo and box_hi must be 3 voxel coordinates each")
        st = SignedStats()
        self._m._ck(self._m._L.fiesta_signed_compute(self._h, lo.ctypes, hi.ctypes, C.byref(st)), "SignedField.compute")
        self.shape = tuple(int(b - a + 1) for a, b in zip(lo, hi))
        return {n: getattr(st, n) for n, _ in st._fields_ if n != "reserved_f"}

    def export(self):
        """S of the last computed box as a (Bx, By, Bz) float64 array."""
        if self.shape is None:
            raise FiestaError("SignedField.export: no field has been computed")
        out = np.empty(self.shape)
        self._m._ck(self._m._L.fiesta_signed_export(self._h, out.ctypes), "SignedField.export")
        return out

    def GetDistanceBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        out = np.empty(len(pos))
        self._m._ck(self._m._L.fiesta_signed_get_distance_batch(self._h, pos.ctypes, C.c_int64(len(pos)), out.ctypes),
                    "SignedField.GetDistanceBatch")
        return out

    def GetDistWithGradTrilinearBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        d = np.empty(len(pos))
        g = np.empty((len(pos), 3))
        self._m._ck(self._m._L.fiesta_signed_get_dist_grad_trilinear_batch(self._h, pos.ctypes, C.c_int64(len(pos)), d.ctypes, g.ctypes),
                    "SignedField.GetDistWithGradTrilinearBatch")
        return d, g

    def GetDistanceBatchDevice(self, pos):
        """GetDistance for a CUDA float64 (n, 3) tensor, on the current torch stream (fiesta_signed_get_distance_batch_device)."""
        torch, stream = self._m._device_tensor(pos, 3, "SignedField.GetDistanceBatchDevice")
        d = torch.empty(pos.shape[0], dtype=torch.float64, device=pos.device)
        self._m._ck(self._m._L.fiesta_signed_get_distance_batch_device(self._h, pos.data_ptr(), pos.shape[0], d.data_ptr(), stream),
                    "SignedField.GetDistanceBatchDevice")
        return d

    def GetDistWithGradTrilinearBatchDevice(self, pos):
        """GetDistWithGradTrilinear for a CUDA float64 (n, 3) tensor, on the current torch stream -> (dist (n,), grad (n, 3))."""
        torch, stream = self._m._device_tensor(pos, 3, "SignedField.GetDistWithGradTrilinearBatchDevice")
        d = torch.empty(pos.shape[0], dtype=torch.float64, device=pos.device)
        g = torch.empty((pos.shape[0], 3), dtype=torch.float64, device=pos.device)
        self._m._ck(self._m._L.fiesta_signed_get_dist_grad_trilinear_batch_device(self._h, pos.data_ptr(), pos.shape[0], d.data_ptr(),
                                                                                  g.data_ptr(), stream),
                    "SignedField.GetDistWithGradTrilinearBatchDevice")
        return d, g

    def close(self):
        if self._h:
            self._m._L.fiesta_signed_destroy(self._h)
            self._h = None


class Frontiers:
    """fiesta_frontiers: the free voxels of a voxel box that border never-observed space, in 26-connected clusters, with cluster
    statistics and member lists.  The buffers grow to the largest box computed; close() it before the map."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_frontiers_create(m._h, C.byref(h)), "fiesta_frontiers_create")
        self._h = h
        self.shape = None
        self.stats = None

    def compute(self, box_lo, box_hi, clearance=0.0, min_cluster_size=1):
        """Frontiers of the inclusive voxel box [box_lo, box_hi] at the clearance (metres) -> stats dict."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("Frontiers.compute: box_lo and box_hi must be 3 voxel coordinates each")
        st = FrontierStats()
        self._m._ck(self._m._L.fiesta_frontiers_compute(self._h, lo.ctypes, hi.ctypes, C.c_double(float(clearance)),
                                                         C.c_int64(int(min_cluster_size)), C.byref(st)), "Frontiers.compute")
        self.shape = tuple(int(b - a + 1) for a, b in zip(lo, hi))
        self.stats = {n: getattr(st, n) for n, _ in st._fields_ if n != "reserved_f"}
        return dict(self.stats)

    def _need(self, what):
        if self.stats is None:
            raise FiestaError("Frontiers.%s: no frontiers have been computed" % what)

    def clusters(self, cap=None):
        """The kept clusters (the first `cap`): dict of size (K,) int64, rep / bbox_lo / bbox_hi (K, 3) int32 grid voxels and
        centroid (K, 3) float64 metres."""
        self._need("clusters")
        k = self.stats["kept_clusters"] if cap is None else min(int(cap), self.stats["kept_clusters"])
        out = dict(size=np.empty(k, np.int64), rep=np.empty((k, 3), np.int32), bbox_lo=np.empty((k, 3), np.int32),
                   bbox_hi=np.empty((k, 3), np.int32), centroid=np.empty((k, 3)))
        self._m._ck(self._m._L.fiesta_frontiers_clusters(self._h, C.c_int64(k), *(out[n].ctypes for n in out)), "Frontiers.clusters")
        return out

    def voxels(self, cap=None):
        """Members of the kept clusters (the first `cap`) as (n, 3) int32 grid voxels, cluster by cluster."""
        self._need("voxels")
        n = self.stats["kept_voxels"] if cap is None else min(int(cap), self.stats["kept_voxels"])
        out = np.empty((n, 3), np.int32)
        self._m._ck(self._m._L.fiesta_frontiers_voxels(self._h, C.c_int64(n), out.ctypes), "Frontiers.voxels")
        return out

    def export(self):
        """Cluster labels as a (Bx, By, Bz) int32 array: the cluster id, -1 elsewhere."""
        self._need("export")
        out = np.empty(self.shape, np.int32)
        self._m._ck(self._m._L.fiesta_frontiers_export(self._h, out.ctypes), "Frontiers.export")
        return out

    def score_viewpoints(self, cluster, positions, orientations, max_range, tan_half_fov, clearance=0.0, unknown_blocks=False):
        """How many members of its kept cluster a sensor at each candidate would see (fiesta_frontiers_score_viewpoints).
        cluster (n,) kept cluster ids, positions (n, 3) metres, orientations (n_orient, 3, 3) world-to-sensor rows (optical axis,
        horizontal, vertical), tan_half_fov (horizontal, vertical) -> (status (n,) int32, score (n, n_orient) int32, stats dict)."""
        self._need("score_viewpoints")
        cl = np.ascontiguousarray(cluster, dtype=np.int32).reshape(-1)
        pos = _f64(positions).reshape(-1, 3)
        R = _f64(orientations).reshape(-1, 9)
        if len(cl) != len(pos):
            raise ValueError("Frontiers.score_viewpoints: %d cluster ids for %d positions" % (len(cl), len(pos)))
        n, k = len(pos), len(R)
        status, score = np.empty(n, np.int32), np.empty((n, k), np.int32)
        sm = SensorModel(float(max_range), (C.c_double * 2)(*[float(x) for x in tan_half_fov]))
        st = ViewpointStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._m._ck(self._m._L.fiesta_frontiers_score_viewpoints(self._h, cl.ctypes, pos.ctypes, C.c_int64(n), R.ctypes, C.c_int32(k),
                                                                  C.byref(sm), r, flags, status.ctypes, score.ctypes, C.byref(st)),
                    "Frontiers.score_viewpoints")
        return status, score, {n_: getattr(st, n_) for n_, _ in st._fields_ if n_ != "reserved_f"}

    def close(self):
        if self._h:
            self._m._L.fiesta_frontiers_destroy(self._h)
            self._h = None


class Skeleton:
    """fiesta_skeleton: the topological skeleton of a voxel box's free space -- voxels on the generalized Voronoi diagram of the
    obstacles, thinned to curves -- as a graph of vertices (junctions, ends) and edges (voxel paths).  The buffers grow to the
    largest box computed; close() it before the map."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_skeleton_create(m._h, C.byref(h)), "fiesta_skeleton_create")
        self._h = h
        self.shape = None
        self.stats = None

    def compute(self, box_lo, box_hi, clearance=0.0, unknown_blocks=False, max_cos=0.5, min_branch=1):
        """Skeleton of the inclusive voxel box [box_lo, box_hi] at the clearance (metres) -> stats dict (iterations: a list of the
        two phases' counts)."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("Skeleton.compute: box_lo and box_hi must be 3 voxel coordinates each")
        st = SkeletonStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._m._ck(self._m._L.fiesta_skeleton_compute(self._h, lo.ctypes, hi.ctypes, r, flags, C.c_double(float(max_cos)),
                                                        C.c_int64(int(min_branch)), C.byref(st)), "Skeleton.compute")
        self.shape = tuple(int(b - a + 1) for a, b in zip(lo, hi))
        self.stats = {n: (list(getattr(st, n)) if n == "iterations" else getattr(st, n)) for n, _ in st._fields_}
        return dict(self.stats)

    def _need(self, what):
        if self.stats is None:
            raise FiestaError("Skeleton.%s: no skeleton has been computed" % what)

    def vertices(self, cap=None):
        """The vertices (the first `cap`): dict of size (V,) int64, rep (V, 3) int32 grid voxels, centroid (V, 3) float64 metres
        and degree (V,) int32."""
        self._need("vertices")
        k = self.stats["vertices"] if cap is None else min(int(cap), self.stats["vertices"])
        out = dict(size=np.empty(k, np.int64), rep=np.empty((k, 3), np.int32), centroid=np.empty((k, 3)), degree=np.empty(k, np.int32))
        self._m._ck(self._m._L.fiesta_skeleton_vertices(self._h, C.c_int64(k), *(out[n].ctypes for n in out)), "Skeleton.vertices")
        return out

    def edges(self, cap=None):
        """The edges (the first `cap`): dict of uv (E, 2) int32 vertex ids, n_vox (E,) int64, length and min_dist (E,) float64."""
        self._need("edges")
        k = self.stats["edges"] if cap is None else min(int(cap), self.stats["edges"])
        out = dict(uv=np.empty((k, 2), np.int32), n_vox=np.empty(k, np.int64), length=np.empty(k), min_dist=np.empty(k))
        self._m._ck(self._m._L.fiesta_skeleton_edges(self._h, C.c_int64(k), *(out[n].ctypes for n in out)), "Skeleton.edges")
        return out

    def edge_voxels(self, cap=None):
        """The edge paths concatenated in edge order (the first `cap` voxels) as (n, 3) int32 grid voxels."""
        self._need("edge_voxels")
        n = self.stats["edge_voxels"] if cap is None else min(int(cap), self.stats["edge_voxels"])
        out = np.empty((n, 3), np.int32)
        self._m._ck(self._m._L.fiesta_skeleton_edge_voxels(self._h, C.c_int64(n), out.ctypes), "Skeleton.edge_voxels")
        return out

    def export(self):
        """(mask, labels) as (Bx, By, Bz) arrays: uint8 bits 1 traversable, 2 anchor, 4 skeleton; int32 vertex id, -2 - edge id on
        chain voxels, -1 elsewhere."""
        self._need("export")
        mask, lab = np.empty(self.shape, np.uint8), np.empty(self.shape, np.int32)
        self._m._ck(self._m._L.fiesta_skeleton_export(self._h, mask.ctypes, lab.ctypes), "Skeleton.export")
        return mask, lab

    def close(self):
        if self._h:
            self._m._L.fiesta_skeleton_destroy(self._h)
            self._h = None


class Mesh:
    """fiesta_mesh: the triangle mesh of the boundary of what blocks at a clearance in a voxel box -- float32 vertices in metres
    placed on the records' exact distances, int32 triangles with normals from blocking to free space, closed at the box faces.
    The buffers grow to the largest box computed; close() it before the map."""

    def __init__(self, m):
        self._m = m
        h = C.c_void_p()
        m._ck(m._L.fiesta_mesh_create(m._h, C.byref(h)), "fiesta_mesh_create")
        self._h = h
        self.stats = None

    def compute(self, box_lo, box_hi, clearance=0.0, unknown_blocks=False):
        """Mesh of the inclusive voxel box [box_lo, box_hi] at the clearance (metres) -> stats dict."""
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,):
            raise ValueError("Mesh.compute: box_lo and box_hi must be 3 voxel coordinates each")
        st = MeshStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        rc = self._m._L.fiesta_mesh_compute(self._h, lo.ctypes, hi.ctypes, r, flags, C.byref(st))
        if rc not in (0, 1):                                                # only FIESTA_ERR_INVALID keeps the last result
            self.stats = None
        self._m._ck(rc, "Mesh.compute")
        self.stats = {n: getattr(st, n) for n, _ in st._fields_}
        return dict(self.stats)

    def _need(self, what):
        if self.stats is None:
            raise FiestaError("Mesh.%s: no mesh has been computed" % what)

    def vertices(self, cap=None):
        """The vertex positions (the first `cap`) as (V, 3) float32 metres."""
        self._need("vertices")
        n = self.stats["vertices"] if cap is None else min(int(cap), self.stats["vertices"])
        out = np.empty((n, 3), np.float32)
        self._m._ck(self._m._L.fiesta_mesh_vertices(self._h, C.c_int64(n), out.ctypes), "Mesh.vertices")
        return out

    def triangles(self, cap=None):
        """The triangles (the first `cap`) as (T, 3) int32 vertex ids, counter-clockwise seen from free space."""
        self._need("triangles")
        n = self.stats["triangles"] if cap is None else min(int(cap), self.stats["triangles"])
        out = np.empty((n, 3), np.int32)
        self._m._ck(self._m._L.fiesta_mesh_triangles(self._h, C.c_int64(n), out.ctypes), "Mesh.triangles")
        return out

    def save_ply(self, path):
        """Write the mesh as binary little-endian PLY (float x y z; list uchar int vertex_indices)."""
        v, t = self.vertices(), self.triangles()
        face = np.empty(len(t), dtype=[("n", "u1"), ("ijk", "<i4", (3,))])
        face["n"] = 3
        face["ijk"] = t
        head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), len(t)))
        with open(path, "wb") as f:
            f.write(head.encode("ascii"))
            f.write(v.astype("<f4").tobytes())
            f.write(face.tobytes())

    def close(self):
        if self._h:
            self._m._L.fiesta_mesh_destroy(self._h)
            self._h = None


class ESDFMap:
    """Mirror of fiesta::ESDFMap (ESDFMap.h:111-164); every method forwards 1:1 to the C ABI."""

    def __init__(self, origin, resolution, map_size, device=0, mode="exact"):
        self._L = load_library()
        cfg = Config()
        cfg.origin = D3(*origin)
        cfg.resolution = float(resolution)
        cfg.map_size = D3(*map_size)
        cfg.device = int(device)
        cfg.mode = {"exact": 0, "fast": 1}[mode]             # FIESTA_MODE_EXACT / FIESTA_MODE_FAST
        self.mode = mode
        h = C.c_void_p()
        rc = self._L.fiesta_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise FiestaError("fiesta_create failed (%d): %s" % (rc, self._L.fiesta_last_error().decode()))
        self._h = h
        self._describe()
        self.mode = mode                                     # as requested (FIESTA_B200_MODE may override the map's own)

    def _describe(self):
        """grid_size, resolution, origin, mode and device of the map behind the handle (fiesta_get_config)."""
        cfg = Config()
        self._ck(self._L.fiesta_get_config(self._h, C.byref(cfg)), "fiesta_get_config")
        self.grid_total_size_ = int(self._L.fiesta_grid_total_size(self._h))
        g = I3()
        self._L.fiesta_grid_size(self._h, g)
        self.grid_size = tuple(int(x) for x in g)
        self.resolution = float(cfg.resolution)
        self.origin = tuple(float(x) for x in cfg.origin)
        self.mode = ("exact", "fast")[cfg.mode]
        self.device = int(cfg.device)

    # --- map snapshots (fiesta_snapshot_save / fiesta_snapshot_load) ---
    def save(self, path=None):
        """Snapshot of the map (it must be quiescent: after UpdateESDF) as bytes, or written to the file `path`."""
        n = C.c_int64(0)
        self._ck(self._L.fiesta_snapshot_save(self._h, None, C.c_int64(0), C.byref(n)), "save")
        buf = np.empty(n.value, np.uint8)
        self._ck(self._L.fiesta_snapshot_save(self._h, buf.ctypes.data, C.c_int64(n.value), C.byref(n)), "save")
        if path is None:
            return buf.tobytes()
        with open(path, "wb") as f:
            f.write(buf.data)
        return None

    @classmethod
    def load(cls, src, device=0):
        """A new map from a snapshot: bytes-like data, or the path of a file holding one.  It continues bit for bit like the
        saved map, in the snapshot's mode."""
        if isinstance(src, (str, os.PathLike)):
            with open(src, "rb") as f:
                src = f.read()
        buf = np.frombuffer(src, np.uint8)
        self = cls.__new__(cls)
        self._L = load_library()
        h = C.c_void_p()
        rc = self._L.fiesta_snapshot_load(buf.ctypes.data if len(buf) else None, C.c_int64(len(buf)), C.c_int32(int(device)), C.byref(h))
        if rc != 0:
            self._h = None
            raise FiestaError("fiesta_snapshot_load failed (%d): %s" % (rc, self._L.fiesta_last_error().decode()))
        self._h = h
        self._describe()
        return self

    def _ck(self, rc, what):
        if rc != 0:
            raise FiestaError("%s failed (%d): %s" % (what, rc, self._L.fiesta_last_error().decode()))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._L.fiesta_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- ESDFMap public surface ---
    def SetParameters(self, p_hit, p_miss, p_min, p_max, p_occ):
        self._ck(self._L.fiesta_set_parameters(self._h, *(C.c_double(x) for x in (p_hit, p_miss, p_min, p_max, p_occ))),
                 "SetParameters")

    def SetOccupancy(self, p, occ):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return int(self._L.fiesta_set_occupancy_vox(self._h, I3(*[int(x) for x in p]), int(occ)))
        return int(self._L.fiesta_set_occupancy_pos(self._h, D3(*[float(x) for x in p]), int(occ)))

    def SetOccupancyBatchVox(self, vox, occ):
        vox = np.ascontiguousarray(vox, dtype=np.int32).reshape(-1, 3)
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        out = np.empty(len(vox), np.int32)
        self._ck(self._L.fiesta_set_occupancy_batch_vox(self._h, vox.ctypes, occ.ctypes, C.c_int64(len(vox)), out.ctypes),
                 "SetOccupancy batch")
        return out

    def SetOccupancyBatchPos(self, pos, occ):
        pos = _f64(pos).reshape(-1, 3)
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        out = np.empty(len(pos), np.int32)
        self._ck(self._L.fiesta_set_occupancy_batch_pos(self._h, pos.ctypes, occ.ctypes, C.c_int64(len(pos)), out.ctypes),
                 "SetOccupancy batch")
        return out

    def SetOccupancyBatchVoxDevice(self, d_vox_ptr, d_occ_ptr, n):
        self._ck(self._L.fiesta_set_occupancy_batch_vox_device(self._h, C.c_void_p(int(d_vox_ptr)), C.c_void_p(int(d_occ_ptr)), C.c_int64(int(n))),
                 "SetOccupancy batch (device)")

    def CheckUpdate(self):
        return bool(self._L.fiesta_check_update(self._h))

    def UpdateOccupancy(self, global_map=True):
        rc = self._L.fiesta_update_occupancy(self._h, int(bool(global_map)))
        if rc < 0:
            raise FiestaError("UpdateOccupancy failed (%d): %s" % (rc, self._L.fiesta_last_error().decode()))
        return bool(rc)

    def UpdateESDF(self):
        self._ck(self._L.fiesta_update_esdf(self._h), "UpdateESDF")

    def SetUpdateRange(self, min_pos, max_pos, new_vec=True):
        self._ck(self._L.fiesta_set_update_range(self._h, D3(*min_pos), D3(*max_pos), int(bool(new_vec))), "SetUpdateRange")

    def SetOriginalRange(self):
        self._ck(self._L.fiesta_set_original_range(self._h), "SetOriginalRange")

    def GetDistance(self, p):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return float(self._L.fiesta_get_distance_vox(self._h, I3(*[int(x) for x in p])))
        return float(self._L.fiesta_get_distance_pos(self._h, D3(*[float(x) for x in p])))

    def GetOccupancy(self, p):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return int(self._L.fiesta_get_occupancy_vox(self._h, I3(*[int(x) for x in p])))
        return int(self._L.fiesta_get_occupancy_pos(self._h, D3(*[float(x) for x in p])))

    def GetDistWithGradTrilinear(self, pos):
        g = D3()
        d = float(self._L.fiesta_get_dist_grad_trilinear(self._h, D3(*[float(x) for x in pos]), g))
        return d, np.array(list(g))

    def GetDistanceBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        out = np.empty(len(pos))
        self._ck(self._L.fiesta_get_distance_batch_pos(self._h, pos.ctypes, C.c_int64(len(pos)), out.ctypes), "GetDistance batch")
        return out

    def GetDistWithGradTrilinearBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        d = np.empty(len(pos))
        g = np.empty((len(pos), 3))
        self._ck(self._L.fiesta_get_dist_grad_trilinear_batch(self._h, pos.ctypes, C.c_int64(len(pos)), d.ctypes, g.ctypes),
                 "GetDistWithGradTrilinear batch")
        return d, g

    # --- planner queries: segment clearance, and stream-ordered queries on CUDA tensors (torch is imported on these paths only) ---
    def _device_tensor(self, t, cols, what):
        import torch
        if not (t.is_cuda and t.device.index == self.device and t.dtype == torch.float64 and t.is_contiguous()
                and t.dim() == 2 and t.shape[1] == cols):
            raise ValueError("%s: expected a contiguous float64 (n, %d) tensor on cuda:%d, got %s %s on %s"
                             % (what, cols, self.device, t.dtype, tuple(t.shape), t.device))
        return torch, torch.cuda.current_stream(t.device).cuda_stream

    def CheckSegments(self, ab, clearance, unknown_blocks=False):
        """Segment clearance (fiesta_check_segments): ab holds n segments {ax, ay, az, bx, by, bz} -> (status, hit_idx, hit_t,
        min_dist).  numpy in, numpy out; a CUDA float64 (n, 6) tensor on the map's device runs fiesta_check_segments_device on the
        current torch stream and returns tensors on that device without synchronising."""
        if not _is_cuda_tensor(ab):
            return _check_segments_host(self._L.fiesta_check_segments, self._h, ab, clearance, unknown_blocks, self._ck)
        torch, stream = self._device_tensor(ab, 6, "CheckSegments")
        n = ab.shape[0]
        out = (torch.empty(n, dtype=torch.int32, device=ab.device), torch.empty(n, dtype=torch.int64, device=ab.device),
               torch.empty(n, dtype=torch.float64, device=ab.device), torch.empty(n, dtype=torch.float64, device=ab.device))
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._ck(self._L.fiesta_check_segments_device(self._h, ab.data_ptr(), n, r, flags, *(o.data_ptr() for o in out), stream),
                 "CheckSegments(device)")
        return out

    def CheckPoses(self, poses, half_extents, clearance, unknown_blocks=False):
        """Robot-shaped collision checks (fiesta_check_poses): an oriented box of half extents (h0, h1, h2) metres at n poses
        {px, py, pz, R00 .. R22} (R world-to-body, row-major: its rows are the box axes) -> (status, n_blocked, hit_idx), status
        0 clear / 1 blocked / 2 invalid pose / 3 the box leaves the map.  numpy in, numpy out; a CUDA float64 (n, 12) tensor on the
        map's device runs fiesta_check_poses_device on the current torch stream and returns tensors without synchronising."""
        if not _is_cuda_tensor(poses):
            return _check_poses_host(self._L.fiesta_check_poses, self._h, poses, half_extents, clearance, unknown_blocks, self._ck)
        torch, stream = self._device_tensor(poses, 12, "CheckPoses")
        he = _half_extents(half_extents)
        n = poses.shape[0]
        out = (torch.empty(n, dtype=torch.int32, device=poses.device), torch.empty(n, dtype=torch.int32, device=poses.device),
               torch.empty(n, dtype=torch.int64, device=poses.device))
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._ck(self._L.fiesta_check_poses_device(self._h, poses.data_ptr(), n, he.ctypes, r, flags, *(o.data_ptr() for o in out), stream),
                 "CheckPoses(device)")
        return out

    def GetDistanceBatchDevice(self, pos):
        """GetDistance for a CUDA float64 (n, 3) tensor, on the current torch stream (fiesta_get_distance_batch_device)."""
        torch, stream = self._device_tensor(pos, 3, "GetDistanceBatchDevice")
        d = torch.empty(pos.shape[0], dtype=torch.float64, device=pos.device)
        self._ck(self._L.fiesta_get_distance_batch_device(self._h, pos.data_ptr(), pos.shape[0], d.data_ptr(), stream),
                 "GetDistanceBatchDevice")
        return d

    def GetDistWithGradTrilinearBatchDevice(self, pos):
        """GetDistWithGradTrilinear for a CUDA float64 (n, 3) tensor, on the current torch stream -> (dist (n,), grad (n, 3))."""
        torch, stream = self._device_tensor(pos, 3, "GetDistWithGradTrilinearBatchDevice")
        d = torch.empty(pos.shape[0], dtype=torch.float64, device=pos.device)
        g = torch.empty((pos.shape[0], 3), dtype=torch.float64, device=pos.device)
        self._ck(self._L.fiesta_get_dist_grad_trilinear_batch_device(self._h, pos.data_ptr(), pos.shape[0], d.data_ptr(), g.data_ptr(), stream),
                 "GetDistWithGradTrilinearBatchDevice")
        return d, g

    # --- safe flight corridors: free axis-aligned voxel boxes in a limit box (fiesta_inflate_boxes, fiesta_corridors) ---
    def _corridor_args(self, box_lo, box_hi, max_steps, what):
        lo, hi = np.ascontiguousarray(box_lo, dtype=np.int32), np.ascontiguousarray(box_hi, dtype=np.int32)
        ms = np.ascontiguousarray(max_steps, dtype=np.int32)
        if lo.shape != (3,) or hi.shape != (3,) or ms.shape != (3,):
            raise ValueError("%s: box_lo, box_hi and max_steps must be 3 integers each" % what)
        return lo, hi, ms

    def InflateBoxes(self, seed_lo, seed_hi, box_lo, box_hi, max_steps, clearance, unknown_blocks=False):
        """Inflate n independent seed boxes (n, 3) inclusive grid voxels inside the limit box [box_lo, box_hi] ->
        (status (n,) int32, lo (n, 3), hi (n, 3) int32 (-1 unless status 0), stats dict)."""
        lo, hi, ms = self._corridor_args(box_lo, box_hi, max_steps, "InflateBoxes")
        slo = np.ascontiguousarray(seed_lo, dtype=np.int32).reshape(-1, 3)
        shi = np.ascontiguousarray(seed_hi, dtype=np.int32).reshape(-1, 3)
        if len(slo) != len(shi):
            raise ValueError("InflateBoxes: %d lower and %d upper seed corners" % (len(slo), len(shi)))
        n = len(slo)
        status, olo, ohi = np.empty(n, np.int32), np.empty((n, 3), np.int32), np.empty((n, 3), np.int32)
        st = CorridorStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._ck(self._L.fiesta_inflate_boxes(self._h, lo.ctypes, hi.ctypes, slo.ctypes, shi.ctypes, C.c_int64(n), ms.ctypes, r, flags,
                                              status.ctypes, olo.ctypes, ohi.ctypes, C.byref(st)), "InflateBoxes")
        return status, olo, ohi, {k: getattr(st, k) for k, _ in st._fields_ if k != "reserved_f"}

    def Corridors(self, paths, box_lo, box_hi, max_steps, clearance, unknown_blocks=False):
        """Chains of overlapping free boxes along paths inside the limit box [box_lo, box_hi].  paths: a list of (L_i, 3) grid-voxel
        arrays, or the (status, len, cost, vox) tuple of NavField.paths (path i is vox[i, :len[i]]) -> (status (n,), n_boxes (n,),
        blocked_at (n,) int32, [(lo (k, 3), hi (k, 3), first (k,)) per path], stats dict)."""
        lo, hi, ms = self._corridor_args(box_lo, box_hi, max_steps, "Corridors")
        if isinstance(paths, tuple) and len(paths) == 4:
            _, ln, _, vox = paths
            paths = [vox[i, :int(ln[i])] for i in range(len(ln))]
        P = [np.ascontiguousarray(p, dtype=np.int32).reshape(-1, 3) for p in paths]
        n = len(P)
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum([len(p) for p in P])
        vox = np.ascontiguousarray(np.concatenate(P) if n else np.zeros((0, 3), np.int32))
        T = int(off[-1])
        status, nb, bl = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32)
        blo, bhi, first = np.empty((T, 3), np.int32), np.empty((T, 3), np.int32), np.empty(T, np.int32)
        st = CorridorStats()
        r, flags = _segment_flags(clearance, unknown_blocks)
        self._ck(self._L.fiesta_corridors(self._h, lo.ctypes, hi.ctypes, vox.ctypes, off.ctypes, C.c_int64(n), ms.ctypes, r, flags,
                                          status.ctypes, nb.ctypes, bl.ctypes, blo.ctypes, bhi.ctypes, first.ctypes, C.byref(st)),
                 "Corridors")
        boxes = [(blo[off[i]:off[i] + nb[i]], bhi[off[i]:off[i] + nb[i]], first[off[i]:off[i] + nb[i]]) for i in range(n)]
        return status, nb, bl, boxes, {k: getattr(st, k) for k, _ in st._fields_ if k != "reserved_f"}

    def box_corners(self, lo, hi):
        """Metric corners of inclusive voxel boxes: (lo * resolution + origin, (hi + 1) * resolution + origin)."""
        o = np.asarray(self.origin)
        return np.asarray(lo) * self.resolution + o, (np.asarray(hi) + 1) * self.resolution + o

    # --- Fiesta::RaycastMultithread (Fiesta.h:281-303), serial semantics ---
    def QueryPlan(self, n):
        """Fixed-size GetDistWithGradTrilinear batch as a CUDA graph over pinned buffers (fiesta_query_plan_*)."""
        return QueryPlan(self, n)

    def HostMirror(self):
        """Pinned host copy of the distance records, patched by refresh() with the records UpdateESDF changed (fiesta_host_mirror_*)."""
        return HostMirror(self)

    def NavField(self):
        """Cost-to-go field of a voxel box through free space at a clearance, with path extraction (fiesta_nav_*)."""
        return NavField(self)

    def SignedField(self):
        """Signed distance of a voxel box: negative inside obstacles by the exact depth to free space (fiesta_signed_*)."""
        return SignedField(self)

    def Frontiers(self):
        """Frontier voxels of a box (free voxels bordering unknown space) in clusters, with statistics (fiesta_frontiers_*)."""
        return Frontiers(self)

    def Skeleton(self):
        """Topological skeleton of a box's free space as a graph of junctions and edges (fiesta_skeleton_*)."""
        return Skeleton(self)

    def Mesh(self):
        """Triangle mesh of the surface of what blocks at a clearance in a box (fiesta_mesh_*)."""
        return Mesh(self)

    def RaycastFrame(self, xyz, T, min_ray_length, max_ray_length):
        """xyz: (n,3) float32 host array, or an integer device pointer paired with `n` as a tuple (ptr, n)."""
        p = RaycastParams(float(min_ray_length), float(max_ray_length))
        T = _f64(T).reshape(16)
        if isinstance(xyz, tuple):
            ptr, n = xyz
            self._ck(self._L.fiesta_raycast_frame_device(self._h, C.c_void_p(int(ptr)), C.c_int64(int(n)), T.ctypes, C.byref(p)),
                     "RaycastFrame(device)")
        else:
            xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
            self._ck(self._L.fiesta_raycast_frame(self._h, xyz.ctypes, C.c_int64(len(xyz)), T.ctypes, C.byref(p)), "RaycastFrame")
        return self.stats()["rays_cast"]

    def RaycastFramePtr(self, host_ptr, n, T, min_ray_length, max_ray_length):
        """Same, from a raw HOST pointer (e.g. a pinned torch tensor's data_ptr())."""
        p = RaycastParams(float(min_ray_length), float(max_ray_length))
        T = _f64(T).reshape(16)
        self._ck(self._L.fiesta_raycast_frame(self._h, C.c_void_p(int(host_ptr)), C.c_int64(int(n)), T.ctypes, C.byref(p)),
                 "RaycastFrame")

    # --- Fiesta::DepthConversion + RaycastMultithread (Fiesta.h:319-382, 281-303) ---
    def DepthFrame(self, depth_u16, dparams, T, m_rel, min_ray_length, max_ray_length):
        img = np.ascontiguousarray(depth_u16, dtype=np.uint16)
        rp = RaycastParams(float(min_ray_length), float(max_ray_length))
        T = _f64(T).reshape(16)
        mr = _f64(m_rel if m_rel is not None else np.eye(4)).reshape(16)
        n = C.c_int64(0)
        self._ck(self._L.fiesta_depth_frame(self._h, img.ctypes, int(img.shape[0]), int(img.shape[1]), C.byref(dparams), T.ctypes, mr.ctypes, C.byref(rp), C.byref(n)),
                 "DepthFrame")
        return int(n.value)

    def last_depth_cloud(self):
        n = C.c_int64(0)
        self._ck(self._L.fiesta_last_depth_cloud(self._h, None, C.c_int64(0), C.byref(n)), "last_depth_cloud")
        out = np.empty((n.value, 3), np.float32)
        if n.value:
            self._ck(self._L.fiesta_last_depth_cloud(self._h, out.ctypes, n, C.byref(n)), "last_depth_cloud")
        return out

    # --- state dumps / stats ---
    def export_distance(self):
        out = np.empty(self.grid_total_size_)
        self._ck(self._L.fiesta_export_distance(self._h, out.ctypes), "export_distance")
        return out

    def export_occupancy(self):
        out = np.empty(self.grid_total_size_)
        self._ck(self._L.fiesta_export_occupancy(self._h, out.ctypes), "export_occupancy")
        return out

    def export_closest_obstacle(self):
        out = np.empty((self.grid_total_size_, 3), np.int32)
        self._ck(self._L.fiesta_export_closest_obstacle(self._h, out.ctypes), "export_closest_obstacle")
        return out

    def export_counters(self):
        hit = np.empty(self.grid_total_size_, np.int32)
        tot = np.empty(self.grid_total_size_, np.int32)
        self._ck(self._L.fiesta_export_counters(self._h, hit.ctypes, tot.ctypes), "export_counters")
        return hit, tot

    def stats(self):
        s = Stats()
        self._ck(self._L.fiesta_get_stats(self._h, C.byref(s)), "get_stats")
        return s.asdict()

    # --- multi-GPU x-slab sharding (see fiesta_b200/shard.py for the exchange loop) ---
    def set_shard(self, rank, world):
        info = ShardInfo()
        self._ck(self._L.fiesta_set_shard(self._h, int(rank), int(world), C.byref(info)), "set_shard")
        return info

    def shard_pack(self, d_lo_ptr, d_hi_ptr):
        self._ck(self._L.fiesta_shard_pack(self._h, C.c_void_p(d_lo_ptr or 0), C.c_void_p(d_hi_ptr or 0)), "shard_pack")

    def shard_ingest(self, d_from_lo_ptr, d_from_hi_ptr):
        ch = C.c_int64(0)
        self._ck(self._L.fiesta_shard_ingest(self._h, C.c_void_p(d_from_lo_ptr or 0), C.c_void_p(d_from_hi_ptr or 0), C.byref(ch)), "shard_ingest")
        return int(ch.value)

    def shard_relax(self):
        ch = C.c_int64(0)
        self._ck(self._L.fiesta_shard_relax(self._h, C.byref(ch)), "shard_relax")
        return int(ch.value)

    # --- visualisation extraction (ESDFMap.h:144-145) ---
    def GetPointCloud(self, vis_lower_bound, vis_upper_bound):
        n = C.c_int64(0)
        self._ck(self._L.fiesta_get_point_cloud(self._h, int(vis_lower_bound), int(vis_upper_bound), None, C.c_int64(0), C.byref(n)), "GetPointCloud")
        out = np.empty((n.value, 3), np.float32)
        if n.value:
            self._ck(self._L.fiesta_get_point_cloud(self._h, int(vis_lower_bound), int(vis_upper_bound), out.ctypes, n, C.byref(n)), "GetPointCloud")
        return out

    def GetSliceMarker(self, slice_, max_dist):
        n = C.c_int64(0)
        self._ck(self._L.fiesta_get_slice_marker(self._h, int(slice_), C.c_double(max_dist), None, None, C.c_int64(0), C.byref(n)), "GetSliceMarker")
        xyz, rgba = np.empty((n.value, 3), np.float64), np.empty((n.value, 4), np.float32)
        if n.value:
            self._ck(self._L.fiesta_get_slice_marker(self._h, int(slice_), C.c_double(max_dist), xyz.ctypes, rgba.ctypes, n, C.byref(n)), "GetSliceMarker")
        return xyz, rgba

    def synchronize(self):
        self._ck(self._L.fiesta_synchronize(self._h), "synchronize")
