"""TEST INFRASTRUCTURE ONLY -- ctypes drivers for the two CPU oracles.

  kind="ref"  : oracle/_ref/libfiesta_ref.so   -- the UNMODIFIED reference (ESDFMap.cpp + raycast.cpp compiled in
                place, see oracle/Makefile) + the restated serial RaycastProcess (oracle/ref_capi.cpp).
  kind="port" : oracle/_build/libfiesta_oracle.so -- oracle/esdf_oracle.c, the plain-C restatement.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
The product package (fiesta_b200/) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATHS = {"ref": os.path.join(_HERE, "_ref", "libfiesta_ref.so"),
          "port": os.path.join(_HERE, "_build", "libfiesta_oracle.so")}
_PREFIX = {"ref": "fiesta_ref_", "port": "fiesta_oracle_"}
_LIBS = {}

D3 = C.c_double * 3
I3 = C.c_int * 3


# Checkout of the upstream FIESTA sources that oracle/_ref is compiled from.  Optional: tests/golden holds what the
# tests compare against, so the suite runs without it.
REFERENCE = os.environ.get("FIESTA_REFERENCE", "")


def reference_present(reference=REFERENCE):
    return bool(reference) and os.path.exists(os.path.join(reference, "src", "ESDFMap.cpp"))


def build(reference=REFERENCE):
    """Compile the C restatement and, when the reference sources are present, oracle/_ref."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "all", "REFERENCE=" + reference])


def available(kind):
    return os.path.exists(_PATHS[kind])


def best_kind():
    """'ref' (the real reference) when it was built here, else the C restatement."""
    return "ref" if available("ref") else "port"


def _lib(kind):
    if kind not in _LIBS:
        if not available(kind):
            raise RuntimeError("oracle library missing: %s (run `make -C oracle`)" % _PATHS[kind])
        L = C.CDLL(_PATHS[kind])
        p = _PREFIX[kind]
        getattr(L, p + "create").restype = C.c_void_p
        for name in ("get_distance_pos", "get_distance_vox", "get_dist_grad_trilinear"):
            getattr(L, p + name).restype = C.c_double
        for name in ("pending_occupancy", "raycast_frame", "raycast", "hung_rays"):
            getattr(L, p + name).restype = C.c_long
        _LIBS[kind] = L
    return _LIBS[kind]


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class OracleMap:
    """Mirror of fiesta::ESDFMap's public surface (ESDFMap.h:111-164) over a CPU oracle library."""

    def __init__(self, origin, resolution, map_size, kind=None):
        self.kind = kind or best_kind()
        self._L = _lib(self.kind)
        self._p = _PREFIX[self.kind]
        self._h = C.c_void_p(self._f("create")(D3(*origin), C.c_double(resolution), D3(*map_size)))
        self.grid_total_size_ = int(self._f("grid_total_size")(self._h))
        g = I3()
        self._f("grid_size")(self._h, g)
        self.grid_size = tuple(int(x) for x in g)
        self.resolution = float(resolution)

    def _f(self, name):
        return getattr(self._L, self._p + name)

    def close(self):
        if self._h is not None:
            self._f("destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- ESDFMap public surface ---
    def SetParameters(self, p_hit, p_miss, p_min, p_max, p_occ):
        self._f("set_parameters")(self._h, *(C.c_double(x) for x in (p_hit, p_miss, p_min, p_max, p_occ)))

    def SetOccupancy(self, p, occ):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return int(self._f("set_occupancy_vox")(self._h, I3(*[int(x) for x in p]), int(occ)))
        return int(self._f("set_occupancy_pos")(self._h, D3(*[float(x) for x in p]), int(occ)))

    def SetOccupancyBatchVox(self, vox, occ):
        vox = np.ascontiguousarray(vox, dtype=np.int32).reshape(-1, 3)
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        out = np.empty(len(vox), np.int32)
        self._f("set_occupancy_batch_vox")(self._h, vox.ctypes, occ.ctypes, C.c_long(len(vox)), out.ctypes)
        return out

    def SetOccupancyBatchPos(self, pos, occ):
        pos = _f64(pos).reshape(-1, 3)
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        out = np.empty(len(pos), np.int32)
        self._f("set_occupancy_batch_pos")(self._h, pos.ctypes, occ.ctypes, C.c_long(len(pos)), out.ctypes)
        return out

    def CheckUpdate(self):
        return bool(self._f("check_update")(self._h))

    def UpdateOccupancy(self, global_map=True):
        return bool(self._f("update_occupancy")(self._h, int(bool(global_map))))

    def UpdateESDF(self):
        self._f("update_esdf")(self._h)

    def SetUpdateRange(self, min_pos, max_pos, new_vec=True):
        self._f("set_update_range")(self._h, D3(*min_pos), D3(*max_pos), int(bool(new_vec)))

    def SetOriginalRange(self):
        self._f("set_original_range")(self._h)

    def GetDistance(self, p):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return float(self._f("get_distance_vox")(self._h, I3(*[int(x) for x in p])))
        return float(self._f("get_distance_pos")(self._h, D3(*[float(x) for x in p])))

    def GetOccupancy(self, p):
        if all(isinstance(x, (int, np.integer)) for x in p):
            return int(self._f("get_occupancy_vox")(self._h, I3(*[int(x) for x in p])))
        return int(self._f("get_occupancy_pos")(self._h, D3(*[float(x) for x in p])))

    def GetDistWithGradTrilinear(self, pos):
        g = D3()
        d = float(self._f("get_dist_grad_trilinear")(self._h, D3(*[float(x) for x in pos]), g))
        return d, np.array(list(g))

    def GetDistanceBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        out = np.empty(len(pos))
        self._f("get_distance_batch_pos")(self._h, pos.ctypes, C.c_long(len(pos)), out.ctypes)
        return out

    def GetDistWithGradTrilinearBatch(self, pos):
        pos = _f64(pos).reshape(-1, 3)
        d = np.empty(len(pos))
        g = np.empty((len(pos), 3))
        self._f("get_dist_grad_trilinear_batch")(self._h, pos.ctypes, C.c_long(len(pos)), d.ctypes, g.ctypes)
        return d, g

    # --- Fiesta::RaycastMultithread (serial mode) ---
    def RaycastFrame(self, xyz, T, min_ray_length, max_ray_length):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        T = _f64(T).reshape(16)
        r = int(self._f("raycast_frame")(self._h, xyz.ctypes, C.c_long(len(xyz)), T.ctypes,
                                        C.c_double(min_ray_length), C.c_double(max_ray_length)))
        if r < 0:
            raise RuntimeError("reference Raycast() threw: more than 1500 voxels on one ray")
        return r

    # --- state dumps / stats ---
    def export_distance(self):
        out = np.empty(self.grid_total_size_)
        self._f("export_distance")(self._h, out.ctypes)
        return out

    def export_occupancy(self):
        out = np.empty(self.grid_total_size_)
        self._f("export_occupancy")(self._h, out.ctypes)
        return out

    def export_closest_obstacle(self):
        out = np.empty((self.grid_total_size_, 3), np.int32)
        self._f("export_closest_obstacle")(self._h, out.ctypes)
        return out

    def export_counters(self):
        hit = np.empty(self.grid_total_size_, np.int32)
        tot = np.empty(self.grid_total_size_, np.int32)
        self._f("export_counters")(self._h, hit.ctypes, tot.ctypes)
        return hit, tot

    def hung_rays(self):
        """Rays dropped because the reference Raycast() loop would never return (see the hang guard)."""
        return int(self._f("hung_rays")(self._h))

    def pending_occupancy(self):
        return int(self._f("pending_occupancy")(self._h))

    def stats(self):
        s = (C.c_long * 6)()
        self._f("get_stats")(self._h, s)
        return dict(occupancy_updates=s[0], inserts=s[1], deletes=s[2], expansions=s[3], change_num=s[4],
                    accumulator=s[5])

    def GetPointCloud(self, lo, hi):
        """Reference build only (kind == 'ref'): ESDFMap::GetPointCloud flattened to (n,3) float32."""
        f = self._f("get_point_cloud"); f.restype = C.c_long
        n = int(f(self._h, int(lo), int(hi), None, C.c_long(0)))
        out = np.empty((n, 3), np.float32)
        f(self._h, int(lo), int(hi), out.ctypes, C.c_long(n))
        return out

    def GetSliceMarker(self, slice_, max_dist):
        f = self._f("get_slice_marker"); f.restype = C.c_long
        n = int(f(self._h, int(slice_), C.c_double(max_dist), None, None, C.c_long(0)))
        xyz, rgba = np.empty((n, 3)), np.empty((n, 4), np.float32)
        f(self._h, int(slice_), C.c_double(max_dist), xyz.ctypes, rgba.ctypes, C.c_long(n))
        return xyz, rgba

    def CheckConsistency(self):
        return bool(self._f("check_consistency")(self._h))


class DepthParams(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("use_filter", C.c_int), ("margin", C.c_int),
                ("max_dist", C.c_double), ("min_dist", C.c_double), ("tolerance", C.c_double)]


def depth_conversion(img, last, image_cnt, params, m_rel, kind=None):
    """Restated Fiesta::DepthConversion (Fiesta.h:319-382): uint16 mm image -> (n,3) float32 cloud in pixel order."""
    kind = kind or best_kind()
    f = getattr(_lib(kind), _PREFIX[kind] + "depth_conversion")
    f.restype = C.c_long
    img = np.ascontiguousarray(img, np.uint16)
    rows, cols = img.shape
    last = np.ascontiguousarray(last if last is not None else img, np.uint16)
    out = np.empty((rows * cols, 3), np.float32)
    mr = np.ascontiguousarray(m_rel if m_rel is not None else np.eye(4), np.float64).reshape(16)
    n = int(f(img.ctypes, last.ctypes, rows, cols, C.c_uint(image_cnt), C.byref(params), mr.ctypes, out.ctypes))
    return out[:n].copy()


def raycast(start, end, mn, mx, kind=None):
    """Reference Raycast() (raycast.cpp:56-158): list of integer voxel coordinates, or None if it threw."""
    kind = kind or best_kind()
    L = _lib(kind)
    buf = np.empty((1502, 3))
    n = int(getattr(L, _PREFIX[kind] + "raycast")(D3(*start), D3(*end), D3(*mn), D3(*mx), buf.ctypes, C.c_long(1502)))
    if n < 0:
        return None if n == -1 else "hang"
    return buf[:n].astype(np.int64)


class FastModel:
    """CPU model of the product's FAST-mode UpdateESDF (oracle/fast_model.c).  It is driven with the occupancy state of
    some other map (the reference build on CPU tests, the GPU map on GPU tests): `update(dist, occ)` takes that map's
    distance_ / occupancy arrays as they are after UpdateOccupancy and before UpdateESDF."""
    FULL_PULL = 1
    EXIT_TEST = 2

    def __init__(self, grid_size, resolution, l_occ, tile=8):
        path = os.path.join(_HERE, "_build", "libfiesta_fastmodel.so")
        if not os.path.exists(path):
            raise RuntimeError("oracle library missing: %s (run `make -C oracle`)" % path)
        self._L = C.CDLL(path)
        self._L.fm_create_tiled.restype = C.c_void_p
        self._L.fm_fresh_left.restype = C.c_longlong
        self._L.fm_halo_ingest.restype = C.c_longlong
        self.grid_size = tuple(int(g) for g in grid_size)
        self.n = int(np.prod(self.grid_size))
        self.res = float(resolution)
        self.l_occ = float(l_occ)
        self._h = C.c_void_p(self._L.fm_create_tiled(*[C.c_int(g) for g in self.grid_size], C.c_int(tile)))
        self._exist = np.zeros(self.n, np.uint8)
        self._seen = np.zeros(self.n, bool)

    def close(self):
        if self._h is not None:
            self._L.fm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_range(self, lo, hi):
        self._L.fm_set_range(self._h, I3(*[int(x) for x in lo]), I3(*[int(x) for x in hi]))

    KEYS = ("generations", "full_visits", "retire_visits", "changed", "reset", "activations", "suppressed", "iterations",
            "evaluations", "candidates")

    def update(self, dist, occ, flags=0, reset=None):
        """One UpdateESDF.  dist: distance_ (only `!= -10000` = observed is used), occ: occupancy log-odds, reset: linear
        indices the local-map reset of UpdateOccupancy(false) set to +infinity (applied before the seeds and the delete scan)."""
        seen = np.asarray(dist) != -10000.0
        new = np.flatnonzero(seen & ~self._seen).astype(np.uint32)
        self._L.fm_observe(self._h, new.ctypes, C.c_longlong(len(new)))
        self._seen = seen
        if reset is not None and len(reset):
            r = np.ascontiguousarray(reset, dtype=np.uint32)
            self._L.fm_local_reset(self._h, r.ctypes, C.c_longlong(len(r)))
        exist = (np.asarray(occ) > self.l_occ).astype(np.uint8)
        ins = np.flatnonzero((exist == 1) & (self._exist == 0)).astype(np.uint32)
        have_del = bool(np.any((exist == 0) & (self._exist == 1)))
        self._exist = exist
        st = (C.c_longlong * 10)()
        self._L.fm_update(self._h, exist.ctypes, ins.ctypes, C.c_longlong(len(ins)), C.c_int(int(have_del)), C.c_int(int(flags)), st)
        return dict(zip(self.KEYS, [int(x) for x in st]))

    # --- x-slab sharding: mirrors ESDFMap.set_shard / shard_pack / shard_ingest / shard_relax on the model's own
    # (unpadded) layout; a layer is gy*gz records and only model instances exchange them
    def set_slab(self, tile_x_lo, tile_x_hi):
        self._L.fm_set_slab(self._h, C.c_int(int(tile_x_lo)), C.c_int(int(tile_x_hi)))

    def pack(self, x_first, nlayers):
        out = np.empty(int(nlayers) * self.grid_size[1] * self.grid_size[2], np.uint32)
        self._L.fm_pack(self._h, C.c_int(int(x_first)), C.c_int(int(nlayers)), out.ctypes)
        return out

    def halo_ingest(self, recv, x_first, nlayers, own_tile_x):
        """Takes over the received ghost records that differ; returns how many did."""
        recv = np.ascontiguousarray(recv, dtype=np.uint32)
        assert len(recv) == int(nlayers) * self.grid_size[1] * self.grid_size[2]
        return int(self._L.fm_halo_ingest(self._h, recv.ctypes, C.c_int(int(x_first)), C.c_int(int(nlayers)),
                                          C.c_int(int(own_tile_x))))

    def relax(self, flags=0):
        """E3 over the tiles the ingests queued (shard_relax)."""
        st = (C.c_longlong * 10)()
        self._L.fm_relax(self._h, C.c_int(int(flags)), st)
        return dict(zip(self.KEYS, [int(x) for x in st]))

    def export(self):
        cobs = np.empty((self.n, 3), np.int32)
        dist = np.empty(self.n)
        self._L.fm_export(self._h, cobs.ctypes, dist.ctypes, C.c_double(self.res))
        return cobs, dist

    def fresh_left(self):
        return int(self._L.fm_fresh_left(self._h))
