"""Ray casting off the friendly geometry: the general per-voxel path (maps off the voxel lattice, FIESTA_RAY_LATTICE=0),
local update boxes as the reference's local-map mode sets them, endpoints exactly on the map's faces (linear-index aliasing,
also with Gz != Pz), every observation source mixed in one order-exact epoch, and the per-frame limits and tag
wrap-arounds.  Every frame is compared with the serial reference (Fiesta.h:194-303): the rays cast, the per-voxel
(num_hit_, num_miss_) counters, the dropped rays and CheckUpdate; every integration with the reference's arrays."""
import math
import time

import numpy as np
import pytest

from tests import scenes
from tests.parity import compare, invariants

pytestmark = pytest.mark.gpu

# name -> (origin, resolution, map_size, on the lattice fast path)
MAPS = {
    "std": ((-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.2), True),
    # half a voxel off the lattice: Pos2Vox((c+0.5)*res) ties at c = -28, so every voxel centre goes through Pos2Vox
    "half": ((-3.25, -3.25, -1.65), 0.1, (6.5, 6.5, 3.3), False),
    # sizes that are no multiple of the resolution: the last voxel sticks out, and some DDA voxel centres (x = 3.25 > 3.22,
    # z = 1.55 > 1.53) lie outside the map (FB_CLS_SKIP)
    "ragged": ((-3.2, -3.2, -1.6), 0.1, (6.42, 6.47, 3.13), False),
    # dyadic: every face and voxel boundary is exact in fp64; Gz = 32, and Gz = 30 (device z pitch 32 != Gz)
    "dyadic": ((-4.0, -4.0, -2.0), 0.125, (8.0, 8.0, 4.0), True),
    "dyadic30": ((-4.0, -4.0, -2.0), 0.125, (8.0, 8.0, 3.75), True),
}

# dyadic sensor translations: world = sensor point + T_OFF is exact in fp64, and the sensor is off every lattice plane
T_OFF = (0.015625, 0.03125, 0.046875)
T_DIAG = (0.015625, 0.015625, 0.015625)   # equal start fractions on every axis: exact tMax ties along 45-degree rays
L_OCC = math.log(0.80 / 0.20)             # p_occ of both parameter sets


def lattice_path(origin, res, size):
    """Python restatement of the host predicate of fiesta_raycast_frame_device (fb_map.cu): True when every DDA voxel centre
    (c+0.5)*res inside the box lies in the map and maps to c - off on every axis, so k_ray_trace may skip Pos2Vox."""
    for k in range(3):
        G = math.ceil(size[k] / res)
        lo, hi = origin[k], origin[k] + size[k]
        clo, chi = math.ceil(lo / res), math.ceil(hi / res)
        if chi - clo > 4096 or chi <= clo:
            return False
        off = clo - math.floor(((clo + 0.5) * res - origin[k]) / res)
        for c in range(clo, chi):
            ctr = (c + 0.5) * res
            v = math.floor((ctr - origin[k]) / res)
            if ctr < lo or ctr > hi or v != c - off or v < 0 or v >= G:
                return False
    return True


def translation(t):
    T = np.eye(4)
    T[:3, 3] = t
    return T


def sensor_points(W, t):
    """float32 sensor-frame points whose world position under translation(t) is W (exact when W - t is a float32)."""
    return (np.asarray(W, np.float64).reshape(-1, 3) - np.asarray(t)).astype(np.float32)


def crafted_frames(origin, res, size, seed=0):
    """[(points, T, min_ray_length, max_ray_length, tag)] aimed at the edges of the map (origin, res, size)."""
    o = np.asarray(origin, np.float64)
    hi = o + np.asarray(size, np.float64)                        # max_range_ as the map computes it
    t = np.asarray(T_OFF)
    rng = np.random.default_rng(seed)
    frames = []
    # faces, corners, one float32 ulp outside, the sensor's own voxel, duplicates
    parts = []
    inner = rng.uniform(o + 2 * res, hi - 2 * res, (12, 3))
    for k in range(3):
        for face, out in ((o[k], -np.inf), (hi[k], np.inf)):
            W = inner.copy()
            W[:, k] = face
            on = sensor_points(W, t)
            beyond = on.copy()
            beyond[:, k] = np.nextafter(on[:, k], np.float32(out))
            parts += [on, beyond]
    corners = np.array([[(o, hi)[(m >> k) & 1][k] for k in range(3)] for m in range(8)])
    c = sensor_points(corners, t)
    parts += [c, np.nextafter(c, np.where(c > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))]
    parts.append(np.array([[0.02, 0.0, 0.0], [-0.02, 0.01, 0.0], [0.0, 0.0, 0.03], [0.01, -0.01, -0.01]], np.float32))
    body = np.concatenate(parts)
    pick = rng.choice(len(body), 24)
    frames.append((np.concatenate([body, body[pick], body[:5]]), translation(T_OFF), 0.005, 8.0, "faces"))
    # axis-aligned rays and exact 45-degree diagonals from a sensor with equal start fractions: tMax ties, z > y > x
    d = []
    for s in (0.75, 1.25, 1.5):
        for sg in ((1, 1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, -1), (-1, -1, -1), (-1, -1, 1)):
            v = s * np.asarray(sg, np.float64)
            d += [v, v * (1, 1, 0), v * (1, 0, 1), v * (0, 1, 1), v * (1, 0, 0), v * (0, 1, 0), v * (0, 0, 1)]
    frames.append((np.asarray(d, np.float32), translation(T_DIAG), 0.05, 8.0, "axes+diagonals"))
    # ray lengths: exactly max_ray_length (3-4-5 triples, exact in fp64), one ulp beyond (clipped), exactly min_ray_length,
    # one ulp below (skipped), and far points clipped inside the map
    L, Lmin = 1.875, 0.25
    e = [(L, 0, 0), (0, -L, 0), (0, 0, L), (1.125, 1.5, 0), (0, -1.125, 1.5), (-1.5, 0, -1.125), (Lmin, 0, 0), (0, 0, -Lmin)]
    e = np.asarray(e, np.float32)
    grow = np.nextafter(e, np.where(e > 0, np.float32(np.inf), np.where(e < 0, np.float32(-np.inf), np.float32(0))).astype(np.float32))
    shrink = np.nextafter(e, np.float32(0))
    far = rng.normal(size=(200, 3))
    far = (far / np.linalg.norm(far, axis=1, keepdims=True) * 4.0).astype(np.float32)
    frames.append((np.concatenate([e, grow, shrink, far]), translation(T_OFF), Lmin, L, "lengths"))
    # far points clipped at max_ray_length = 6, mostly landing outside the map
    far = rng.normal(size=(400, 3))
    far = (far / np.linalg.norm(far, axis=1, keepdims=True) * 9.0).astype(np.float32)
    frames.append((far, translation(T_OFF), 0.1, 6.0, "clipped outside"))
    return frames


def alias_frames(name):
    """[(points, T, min, max, tag, oracle ray count)]: A lies exactly on an upper face, its voxel coordinate equals G and the
    linear index aliases onto B's voxel, so A (earlier in the frame) takes B's endpoint ownership and B casts no ray."""
    if name == "dyadic":       # A on y = 4.0 in voxel x 40, z 5 -> alias (41, 0, 5)
        A, B = (1.0625, 4.0, -1.3125), (1.1875, -3.9375, -1.3125)
    elif name == "dyadic30":   # A on z = 1.75 in voxel (40, 20) -> alias (40, 21, 0): decoded with Gz, re-encoded with Pz
        A, B = (1.0625, -1.4375, 1.75), (1.0625, -1.3125, -1.9375)
    else:
        return []
    pts = sensor_points([A, B], T_OFF)
    return [(pts, translation(T_OFF), 0.1, 6.0, "alias A,B", 1), (pts[1:], translation(T_OFF), 0.1, 6.0, "B alone", 1)]


def scene_frames(name, n_depth=2, seed=3):
    origin, res, size, _ = MAPS[name]
    half = np.asarray(size) / 2
    sc = scenes.Scene(tuple(half * (0.85, 0.85, 0.8)), 8, 3, seed=seed, edge=(0.3, 0.9))
    out = []
    for f, (p, yaw) in enumerate(scenes.pose_walk(n_depth + 1, seed=seed, clamp=0.6)):
        p = p + np.asarray(origin) + half
        if f < n_depth:
            pts, T = scenes.depth_frame(sc, p, yaw, width=80, height=60, scale=0.125)
            out.append((pts, T, 0.3, 4.0, "depth %d" % f))
        else:
            pts, T = scenes.lidar_frame(sc, p, yaw, beams=16, azimuths=400)
            out.append((pts, T, 0.3, 5.0, "lidar"))
        sc.step()
    return out


# ---------------------------------------------------------------- one frame / one integration, checked
def _is_oracle(m):
    return hasattr(m, "hung_rays")


def cast(m, pts, T, lo, hi):
    """RaycastFrame -> (rays cast, rays dropped in this frame)."""
    if _is_oracle(m):
        h = m.hung_rays()
        r = m.RaycastFrame(pts, T, lo, hi)
        return r, m.hung_rays() - h
    r = m.RaycastFrame(pts, T, lo, hi)
    return r, m.stats()["rays_dropped"]


def depth_cast(m, oracle_mod, img, last_img, image_cnt, use_filter, T, m_rel, lo, hi, scale):
    """Fiesta::DepthConversion + RaycastMultithread: the device's fused DepthFrame, or the restated conversion + RaycastFrame."""
    args = (scenes.FX * scale, scenes.FY * scale, scenes.CX * scale, scenes.CY * scale, use_filter, 2, 10.0, 0.1, 0.1)
    if _is_oracle(m):
        cloud = oracle_mod.depth_conversion(img, last_img, image_cnt, oracle_mod.DepthParams(*args), m_rel, kind=m.kind)
        return cast(m, cloud, T, lo, hi) if len(cloud) else (0, 0)
    import fiesta_b200
    n = m.DepthFrame(img, fiesta_b200.DepthParams(*args), T, m_rel, lo, hi)
    return (m.stats()["rays_cast"], m.stats()["rays_dropped"]) if n else (0, 0)


def check_frame(a, b, ra, rb, tag):
    assert ra == rb, (tag, "rays cast / dropped", ra, rb)
    (h1, t1), (h2, t2) = a.export_counters(), b.export_counters()
    assert np.array_equal(h1, h2) and np.array_equal(t1, t2), (tag, "counters", int(((h1 != h2) | (t1 != t2)).sum()))
    assert a.CheckUpdate() == b.CheckUpdate(), tag


def integrate(dev, ora, mode, tag, global_map=True):
    if not dev.CheckUpdate():
        assert not ora.CheckUpdate(), tag
        return
    assert dev.UpdateOccupancy(global_map) == ora.UpdateOccupancy(global_map), tag
    dev.UpdateESDF()
    ora.UpdateESDF()
    check_arrays(dev, ora, mode, tag, global_map)


def check_arrays(dev, ora, mode, tag, global_map=True):
    r = compare(dev, ora, check_counters=True)
    assert r["occ"] == 0 and r["counters"] == 0, (tag, r)
    if mode == "exact":
        assert r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0, (tag, r)
        assert dev.stats()["expansions"] == ora.stats()["expansions"], tag
    else:
        inv = invariants(dev, L_OCC)
        if not global_map:
            # the wave stays inside the update box, so a voxel next to it may keep an obstacle farther than an occupied
            # neighbour outside the box -- the reference leaves the same states (ESDFMap.cpp:339-392 skip !VoxInRange)
            del inv["closer_occupied_neighbour"]
        assert not any(inv.values()), (tag, inv)


def make_pair(oracle_mod, name_or_geom, mode, params=scenes.PARAMS_TOGGLE):
    import fiesta_b200
    origin, res, size = MAPS[name_or_geom][:3] if isinstance(name_or_geom, str) else name_or_geom
    dev = fiesta_b200.ESDFMap(origin, res, size, mode=mode)
    ora = oracle_mod.OracleMap(origin, res, size)
    for m in (dev, ora):
        m.SetParameters(*params)
    return dev, ora


def set_lattice(monkeypatch, lattice):
    if lattice == "off":
        monkeypatch.setenv("FIESTA_RAY_LATTICE", "0")
    else:
        monkeypatch.delenv("FIESTA_RAY_LATTICE", raising=False)


@pytest.fixture(scope="module")
def timer():
    t0 = time.perf_counter()
    yield
    print("\ntest_gpu_raycast_edges.py: %.1f s" % (time.perf_counter() - t0))


# ---------------------------------------------------------------- B1 + B2: path guard and geometry matrix
@pytest.mark.parametrize("lattice", ["auto", "off"])
@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("name", list(MAPS))
def test_geometry_matrix(oracle_built, monkeypatch, timer, name, mode, lattice):
    origin, res, size, on_path = MAPS[name]
    assert lattice_path(origin, res, size) == on_path, name    # the map takes the path this case is meant to test
    set_lattice(monkeypatch, lattice)
    dev, ora = make_pair(oracle_built, name, mode)
    drive_geometry(dev, ora, name, mode)


def drive_geometry(dev, ora, name, mode):
    """Crafted edge frames, the alias pair and scene frames on map `name`; `ora` is the reference side."""
    origin, res, size, _ = MAPS[name]
    assert dev.grid_size == ora.grid_size == tuple(math.ceil(s / res) for s in size)
    frames = [f + (None,) for f in crafted_frames(origin, res, size)] + alias_frames(name) + \
             [f + (None,) for f in scene_frames(name)]
    for k, (pts, T, lo, hi, tag, want) in enumerate(frames):
        ro = cast(ora, pts, T, lo, hi)
        if want is not None:
            assert ro[0] == want, (tag, ro)                      # the reference suppresses the aliased ray
        check_frame(dev, ora, cast(dev, pts, T, lo, hi), ro, (name, tag))
        if k % 2 == 1 or k == len(frames) - 1:
            integrate(dev, ora, mode, (name, tag))


# ---------------------------------------------------------------- B3: local map as the reference runs it
@pytest.mark.parametrize("lattice", ["auto", "off"])
@pytest.mark.parametrize("mode", ["exact", "fast"])
@pytest.mark.parametrize("source", ["raycast", "depth"])
@pytest.mark.parametrize("name", ["std", "half", "dyadic30"])
def test_local_map_casting(oracle_built, monkeypatch, timer, name, source, mode, lattice):
    """Fiesta.h:482-539 with global_update_ = false: each frame is cast while the previous update's box (or a visualisation
    box set with new_vec = false, Fiesta.h:150) is in force, then SetUpdateRange(cur +- radius), UpdateOccupancy(false),
    UpdateESDF.  Voxels in the map but outside the box are stamped without being counted (ESDFMap.cpp:420-421)."""
    set_lattice(monkeypatch, lattice)
    dev, ora = make_pair(oracle_built, name, mode, params=scenes.PARAMS_DEFAULT)
    assert drive_local(dev, ora, oracle_built, name, source, mode) > 0   # some frame had stamp-only voxels


def drive_local(dev, ora, oracle_mod, name, source, mode):
    """The local-map loop on map `name`; returns the number of frames in which the reference counted fewer observations than
    the same frame gives under SetOriginalRange (voxels stamped but not counted)."""
    origin, res, size, _ = MAPS[name]
    full = oracle_mod.OracleMap(origin, res, size, kind="port")     # the same frames under SetOriginalRange
    centre = np.asarray(origin) + np.asarray(size) / 2
    radius = np.array([1.6, 1.4, 0.9])
    sc = scenes.Scene(tuple(np.asarray(size) / 2 * (0.85, 0.85, 0.8)), 8, 3, seed=5, edge=(0.3, 0.9))
    scale, use_filter = 0.125, 1
    last_img = last_T = None
    stamp_only = 0
    box = None
    for f, (p, yaw) in enumerate(scenes.pose_walk(8, seed=6, clamp=1.0)):
        p = p + centre
        tag = (name, source, f)
        before = ora.export_counters()[1].sum()
        before_full = full.export_counters()[1].sum()
        if source == "raycast":
            pts, T = scenes.depth_frame(sc, p, yaw, width=80, height=60, scale=scale)
            ro, rd = cast(ora, pts, T, 0.3, 4.0), cast(dev, pts, T, 0.3, 4.0)
            cast(full, pts, T, 0.3, 4.0)
        else:                                  # with the temporal depth filter: the first image only primes it
            img, T = scenes.depth_image(sc, p, yaw, width=80, height=60, scale=scale)
            m_rel = np.linalg.inv(last_T) @ T if last_T is not None else np.eye(4)
            ro, rd, _ = (depth_cast(m, oracle_mod, img, last_img, f + 1, use_filter, T, m_rel, 0.3, 4.0, scale) for m in (ora, dev, full))
            last_img, last_T = img, T
        check_frame(dev, ora, rd, ro, tag)
        if ora.export_counters()[1].sum() - before < full.export_counters()[1].sum() - before_full:
            stamp_only += 1
        box = (p - radius, p + radius)
        if f == 2:                             # faces on lattice planes (exact on the dyadic map); frame 3 is cast under it
            box = (np.asarray(origin) + res * np.array([10, 12, 4]), np.asarray(origin) + res * np.array([40, 36, 20]))
        if f == 4:                             # empty after clamping to the map: frame 5 only stamps
            box = (np.asarray(origin) + np.asarray(size) + 1.0, np.asarray(origin) + np.asarray(size) + 2.0)
        if ora.CheckUpdate():                  # UpdateEsdfEvent: box, UpdateOccupancy(false), UpdateESDF
            for m in (dev, ora):
                m.SetUpdateRange(*box)
            integrate(dev, ora, mode, tag, global_map=False)
        full.UpdateOccupancy(True)
        if f % 2 == 1:                         # visualisation with a newer pose moves the box, new_vec = false (Fiesta.h:150)
            for m in (dev, ora):
                m.SetUpdateRange(p + (0.3, -0.2, 0.0) - radius, p + (0.3, -0.2, 0.0) + radius, False)
        sc.step()
    full.close()
    return stamp_only


# ---------------------------------------------------------------- B4: every source in one order-exact epoch
@pytest.mark.parametrize("lattice", ["auto", "off"])
@pytest.mark.parametrize("box", [False, True])
def test_mixed_sources_one_epoch_exact(oracle_built, monkeypatch, timer, box, lattice):
    """The insert and delete queues follow the order of FIRST observation across per-call SetOccupancy, batches, ray-cast and
    depth frames (occupancy_queue_, ESDFMap.cpp:424-435): many voxels are first seen by one source and later by another."""
    set_lattice(monkeypatch, lattice)
    dev, ora = make_pair(oracle_built, "std", "exact")
    drive_mixed(dev, ora, oracle_built, box)


def drive_mixed(dev, ora, oracle_mod, box):
    gs = dev.grid_size
    rng = np.random.default_rng(8)
    sc = scenes.Scene((2.7, 2.7, 1.3), 8, 3, seed=9, edge=(0.3, 0.9))
    scale = 0.125
    last_img = last_T = None
    poses = scenes.pose_walk(6, seed=10, clamp=0.8)
    radius = np.array([1.8, 1.5, 1.0])

    def per_call(k, tag):
        pos = rng.uniform(-2.0, 2.0, (k, 3)) * (1, 1, 0.55)
        vox = np.stack([rng.integers(10, gs[i] - 10, k) for i in range(3)], -1)
        occ = rng.integers(0, 2, 2 * k)
        for j in range(k):
            assert dev.SetOccupancy(tuple(pos[j]), int(occ[j])) == ora.SetOccupancy(tuple(pos[j]), int(occ[j])), tag
            v = tuple(int(x) for x in vox[j])
            assert dev.SetOccupancy(v, int(occ[k + j])) == ora.SetOccupancy(v, int(occ[k + j])), tag

    for epoch in range(3):
        tag = ("epoch", epoch)
        (p0, y0), (p1, y1) = poses[2 * epoch], poses[2 * epoch + 1]
        if box:
            for m in (dev, ora):
                m.SetUpdateRange(p0 - radius, p0 + radius)
        per_call(150, tag)
        vox = np.stack([rng.integers(8, gs[i] - 8, 1500) for i in range(3)], -1).astype(np.int32)
        occ = (rng.random(1500) < 0.4).astype(np.uint8)
        assert np.array_equal(dev.SetOccupancyBatchVox(vox, occ), ora.SetOccupancyBatchVox(vox, occ)), tag
        pts, T = scenes.depth_frame(sc, p0, y0, width=80, height=60, scale=scale)
        check_frame(dev, ora, cast(dev, pts, T, 0.3, 4.0), cast(ora, pts, T, 0.3, 4.0), tag + ("raycast",))
        img, T = scenes.depth_image(sc, p1, y1, width=80, height=60, scale=scale)
        m_rel = np.linalg.inv(last_T) @ T if last_T is not None else np.eye(4)
        rd, ro = (depth_cast(m, oracle_mod, img, last_img, epoch + 1, 0, T, m_rel, 0.3, 4.0, scale) for m in (dev, ora))
        check_frame(dev, ora, rd, ro, tag + ("depth",))
        last_img, last_T = img, T
        per_call(150, tag)
        pts, T = scenes.lidar_frame(sc, p1, y1 + 0.4, beams=16, azimuths=400)
        check_frame(dev, ora, cast(dev, pts, T, 0.3, 5.0), cast(ora, pts, T, 0.3, 5.0), tag + ("lidar",))
        integrate(dev, ora, "exact", tag, global_map=not box)
        sc.step()


# ---------------------------------------------------------------- B5: the per-frame point limit
@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_point_limit(oracle_built, timer, mode):
    """n = 524286 (2^19 - 2) is the largest frame accepted, through the host and the device-pointer entry points; 524287 is
    refused with FIESTA_ERR_LIMIT before anything is observed.  max_ray_length 5 m keeps the ray lists near 200 MB."""
    import torch
    import fiesta_b200
    dev, ora = make_pair(oracle_built, "std", mode)
    rng = np.random.default_rng(12)
    T = scenes.body_transform((0.0137, -0.0211, 0.0093), 0.2)
    n_max = (1 << 19) - 2

    def cloud(n):
        d = rng.normal(size=(n, 3)) * (1, 1, 0.4)
        return (d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.2, 6.0, (n, 1))).astype(np.float32)

    pts = cloud(n_max)
    check_frame(dev, ora, cast(dev, pts, T, 0.3, 5.0), cast(ora, pts, T, 0.3, 5.0), "host path")
    pts = cloud(n_max)
    t = torch.from_numpy(pts).cuda()
    rd = (dev.RaycastFrame((t.data_ptr(), n_max), T, 0.3, 5.0), dev.stats()["rays_dropped"])
    check_frame(dev, ora, rd, cast(ora, pts, T, 0.3, 5.0), "device path")
    integrate(dev, ora, mode, "after the largest frames")
    before = dev.export_counters()
    pending = dev.CheckUpdate()
    over = cloud(n_max + 1)
    with pytest.raises(fiesta_b200.FiestaError, match=r"failed \(4\)"):
        dev.RaycastFrame(over, T, 0.3, 5.0)
    with pytest.raises(fiesta_b200.FiestaError, match=r"failed \(4\)"):
        dev.RaycastFrame((torch.from_numpy(over).cuda().data_ptr(), n_max + 1), T, 0.3, 5.0)
    after = dev.export_counters()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]) and dev.CheckUpdate() == pending
    pts = cloud(5000)
    check_frame(dev, ora, cast(dev, pts, T, 0.3, 5.0), cast(ora, pts, T, 0.3, 5.0), "after the refusal")
    integrate(dev, ora, mode, "after the refusal")


# ---------------------------------------------------------------- B6: wrap-arounds
SMALL = ((-1.6, -1.6, -1.6), 0.1, (3.2, 3.2, 3.2))   # 32^3


def small_cloud_pool(rng, k):
    """k endpoints that share voxels: 16 voxel centres (+- a few mm), so several points of a frame end in one voxel."""
    base = rng.uniform(-1.4, 1.4, (16, 3))
    return (base[rng.integers(0, 16, k)] + rng.uniform(-0.02, 0.02, (k, 3))).astype(np.float32)


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_owner_tag_wraps(oracle_built, timer, mode):
    """The endpoint-owner word keeps a 13-bit frame tag: after 8191 frames stamp[1] is cleared and the tag restarts.  8195
    frames of 64 points whose order changes every frame, so a stale owner of an older frame would drop the wrong ray."""
    dev, ora = make_pair(oracle_built, SMALL, mode)
    rng = np.random.default_rng(13)
    pool = small_cloud_pool(rng, 512)
    T = scenes.body_transform((0.0137, -0.0211, 0.0093), 0.0)
    for f in range(8195):
        pts = pool[rng.choice(len(pool), 64, replace=False)]
        ro, rd = cast(ora, pts, T, 0.1, 3.0), cast(dev, pts, T, 0.1, 3.0)
        assert ro == rd, (f, ro, rd)
        if 8189 <= f <= 8194:                  # the owner tag is cleared before frame 8191 (0-based)
            check_frame(dev, ora, rd, ro, f)
        if f % 100 == 99 or f == 8194:
            integrate(dev, ora, mode, f)


def test_exact_key_budget(oracle_built, timer):
    """EXACT mode: 16383 frames between two UpdateOccupancy calls (observation keys 2^30 per frame within 44 bits); per-call
    events in between use part of the last frame's room.  The last frames first-observe voxels with keys near the top of
    the key space.  The 16384th frame is refused with FIESTA_ERR_LIMIT and the map stays consistent."""
    import fiesta_b200
    dev, ora = make_pair(oracle_built, SMALL, "exact")
    rng = np.random.default_rng(14)
    pool = small_cloud_pool(rng, 256)
    late = small_cloud_pool(np.random.default_rng(15), 64)          # endpoints seen for the first time in the last frames
    T = scenes.body_transform((0.0137, -0.0211, 0.0093), 0.0)
    budget = 16383
    for f in range(budget):
        pts = pool[rng.choice(len(pool), 8, replace=False)] if f < budget - 4 else late[16 * (f - budget + 4):16 * (f - budget + 5)]
        ro, rd = cast(ora, pts, T, 0.1, 3.0), cast(dev, pts, T, 0.1, 3.0)
        assert ro == rd, (f, ro, rd)
        if f in (5000, 12000, budget - 2):
            for v in ((3, 4, 5), (20, 21, 22), (31, 0, 17)):
                assert dev.SetOccupancy(v, 1) == ora.SetOccupancy(v, 1)
        if f % 4000 == 0 or f >= budget - 3:
            check_frame(dev, ora, rd, ro, f)
    with pytest.raises(fiesta_b200.FiestaError, match=r"failed \(4\)"):
        dev.RaycastFrame(pool[:8], T, 0.1, 3.0)
    check_frame(dev, ora, 0, 0, "refused frame: nothing observed")
    integrate(dev, ora, "exact", "after the full budget")
    pts = pool[:32]
    check_frame(dev, ora, cast(dev, pts, T, 0.1, 3.0), cast(ora, pts, T, 0.1, 3.0), "next epoch")
    integrate(dev, ora, "exact", "next epoch")
