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
]

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
        _lib = L
    return _lib


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


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

    def close(self):
        if self._h:
            self._m._L.fiesta_host_mirror_destroy(self._h)
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
        self.grid_total_size_ = int(self._L.fiesta_grid_total_size(self._h))
        g = I3()
        self._L.fiesta_grid_size(self._h, g)
        self.grid_size = tuple(int(x) for x in g)
        self.resolution = float(resolution)
        self.device = int(device)

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

    # --- Fiesta::RaycastMultithread (Fiesta.h:281-303), serial semantics ---
    def QueryPlan(self, n):
        """Fixed-size GetDistWithGradTrilinear batch as a CUDA graph over pinned buffers (fiesta_query_plan_*)."""
        return QueryPlan(self, n)

    def HostMirror(self):
        """Pinned host copy of the distance records, patched by refresh() with the records UpdateESDF changed (fiesta_host_mirror_*)."""
        return HostMirror(self)

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
