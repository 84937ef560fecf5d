"""Drivers that keep the FAST-mode CPU model (oracle/fast_model.c) in step with the reference build, and optionally with
FAST-mode ESDFMaps on the GPU, under update boxes, local-map resets and x-slab shards.

The model does not see SetUpdateRange, UpdateOccupancy(false) or the shard calls itself; these helpers restate what the
map does with them:
  vox_box    ESDFMap::SetUpdateRange (ESDFMap.cpp:792-810): the voxel box min_vec_ .. max_vec_ of a metric box;
  reset_set  the local-map reset of UpdateOccupancy(false) (ESDFMap.cpp:242-259), from the counters and the occupancy as
             they are before the call and the previous box;
  ShardedModel  one model per rank with the exchange loop of fiesta_b200.shard.sharded_update_esdf.
"""
import math

import numpy as np

from tests import scenes

def logit(p):
    return math.log(p / (1.0 - p))          # the reference's Logit, through the C library's log


def vox_box(origin, res, size, lo, hi):
    """min_vec_, max_vec_ after SetUpdateRange(lo, hi); empty along an axis when min > max."""
    origin, size = np.asarray(origin, float), np.asarray(size, float)
    mn = np.maximum(np.asarray(lo, float), origin)
    mx = np.minimum(np.asarray(hi, float), origin + size)
    vlo = np.floor((mn - origin) / res).astype(int)
    vhi = np.floor((mx - res / 2 - origin) / res).astype(int)
    return tuple(int(v) for v in vlo), tuple(int(v) for v in vhi)


def reset_set(hit, tot, occ, last, gs, params):
    """Linear indices UpdateOccupancy(false) sets to +infinity: pending observations, not skipped by the clamp test, outside
    the previous box last = (last_min_vec_, last_max_vec_)."""
    l_hit, l_miss, l_min, l_max = (logit(p) for p in params[:4])
    pending = tot > 0
    upd = np.where(hit >= tot - hit, l_hit, l_miss)
    skip = ((upd >= 0) & (occ >= l_max)) | ((upd <= 0) & (occ <= l_min))
    idx = np.indices(gs).reshape(3, -1).T
    inside = np.all((idx >= np.asarray(last[0])) & (idx <= np.asarray(last[1])), axis=1)
    return np.flatnonzero(pending & ~skip & ~inside).astype(np.uint32)


def n_diff(a, b):
    """Voxels whose closest obstacle or distance differs between two models."""
    ca, da = a.export()
    cb, db = b.export()
    return int(((ca != cb).any(axis=1) | (da != db)).sum())


def assert_identical(dev, cobs, dist, tag):
    C, D = dev.export_closest_obstacle(), dev.export_distance()
    assert np.array_equal(D, dist), (tag, int((D != dist).sum()))
    assert np.array_equal(C, cobs), (tag, int((C != cobs).any(axis=1).sum()))


class BoxDriver:
    """The reference build, three FAST models (base, every voxel pulls, exit test) and optionally a FAST-mode ESDFMap on
    the GPU, fed the same calls.  After every update the models must agree bit for bit and hold no FRESH flag; the device
    must equal the base model bit for bit (closest obstacles included) with the same changed-voxel and generation counts,
    and its occupancy and counters must equal the reference's."""

    def __init__(self, oracle_mod, origin, res, size, params, dev=None):
        self.origin, self.res, self.size = tuple(origin), float(res), tuple(size)
        self.ora = oracle_mod.OracleMap(self.origin, self.res, self.size)
        self.dev = dev
        self.gs = self.ora.grid_size
        self.full = ((0, 0, 0), tuple(g - 1 for g in self.gs))
        self.cur = self.last = self.full
        self.params = None
        mk = lambda: oracle_mod.FastModel(self.gs, self.res, logit(params[4]))
        FM = oracle_mod.FastModel
        self.base, self.pull, self.exit = mk(), mk(), mk()
        self.models = [(self.base, 0), (self.pull, FM.FULL_PULL), (self.exit, FM.EXIT_TEST)]
        self.set_params(params)
        self.updates = self.resets = self.local_updates = 0

    def maps(self):
        return (self.ora,) + ((self.dev,) if self.dev is not None else ())

    def set_params(self, params):
        assert self.params is None or params[4] == self.params[4]    # the models' occupancy threshold stays
        self.params = params
        for m in self.maps():
            m.SetParameters(*params)

    def _range(self):
        for m, _ in self.models:
            m.set_range(*self.cur)

    def set_box(self, lo, hi, new_vec=True):
        for m in self.maps():
            m.SetUpdateRange(tuple(lo), tuple(hi), new_vec)
        if new_vec:
            self.last = self.cur
        self.cur = vox_box(self.origin, self.res, self.size, lo, hi)
        self._range()

    def original(self):
        for m in self.maps():
            m.SetOriginalRange()
        self.cur = self.last = self.full
        self._range()

    def events(self, vox, occ):
        r = self.ora.SetOccupancyBatchVox(vox, occ)
        if self.dev is not None:
            assert np.array_equal(self.dev.SetOccupancyBatchVox(vox, occ), r)

    def cast(self, pts, T, lo=0.3, hi=4.0):
        r = self.ora.RaycastFrame(pts, T, lo, hi)
        if self.dev is not None:
            assert self.dev.RaycastFrame(pts, T, lo, hi) == r

    def update(self, global_map=True, tag=""):
        """UpdateOccupancy(global_map) + UpdateESDF on every side; returns the base model's statistics (None if nothing
        was pending)."""
        ora, dev = self.ora, self.dev
        if not ora.CheckUpdate():
            assert dev is None or not dev.CheckUpdate(), tag
            return None
        reset = None
        hit, tot = ora.export_counters()
        if dev is not None:
            h2, t2 = dev.export_counters()
            assert np.array_equal(hit, h2) and np.array_equal(tot, t2), ("counters", tag)
        if not global_map:
            d0 = ora.export_distance()
            reset = reset_set(hit, tot, ora.export_occupancy(), self.last, self.gs, self.params)
        r = ora.UpdateOccupancy(global_map)
        if dev is not None:
            assert dev.UpdateOccupancy(global_map) == r, tag
        dist, occ = ora.export_distance(), ora.export_occupancy()
        if dev is not None:
            assert np.array_equal(dev.export_occupancy(), occ), ("occupancy", tag)
            assert np.array_equal(dev.export_distance() != -10000.0, dist != -10000.0), ("observed", tag)
        if reset is not None:
            # the restated reset set against the reference: every finite distance that became +infinity is in it, and
            # everything in it reads +infinity
            went = (d0 >= 0) & (d0 < 10000) & (dist == 10000)
            assert np.isin(np.flatnonzero(went), reset).all(), ("reset set misses a reset voxel", tag)
            assert (dist[reset] == 10000).all(), ("reset set holds a voxel that was not reset", tag)
            self.resets += len(reset)
            self.local_updates += 1
        st = [m.update(dist, occ, f, reset) for m, f in self.models]
        ora.UpdateESDF()
        for m, _ in self.models:
            assert m.fresh_left() == 0, tag
        n = n_diff(self.base, self.pull)
        assert n == 0, ("every-voxel-pulls variant differs", tag, n)
        n = n_diff(self.base, self.exit)
        assert n == 0, ("exit-test variant differs", tag, n)
        if dev is not None:
            dev.UpdateESDF()
            cobs, d = self.base.export()
            assert_identical(dev, cobs, d, tag)
            sd = dev.stats()
            assert sd["voxels_changed"] == st[0]["changed"] and sd["generations"] == st[0]["generations"], (tag, st[0], sd)
        self.updates += 1
        return st[0]

    def distance_mismatch(self):
        """Voxels where the base model's distance differs from the reference's."""
        return int((self.base.export()[1] != self.ora.export_distance()).sum())

    def close(self):
        for m, _ in self.models:
            m.close()
        self.ora.close()


def rand_vox(rng, gs, n):
    return np.stack([rng.integers(0, gs[i], n) for i in range(3)], -1).astype(np.int32)


# ---------------------------------------------------------------- scenarios, run on the CPU and on the GPU alike
GEOM = ((-2.0, -2.0, -2.0), 0.1, (4.0, 4.0, 4.0))                # 40^3
GEOM_EDGES = ((-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.2))           # 64 x 64 x 32, the map of test_gpu_edges.py


def observe(drv, rng, observed, n_obstacles):
    allv = scenes.all_voxels(drv.gs)
    if observed < 1.0:
        allv = allv[rng.random(len(allv)) < observed]
    drv.events(allv, np.zeros(len(allv), np.uint8))
    drv.update(tag="observe")
    drv.events(rand_vox(rng, drv.gs, n_obstacles), np.ones(n_obstacles, np.uint8))
    drv.update(tag="obstacles")


def whole_grid_tail(drv, rng, n_updates=3, n_ev=600, tag=""):
    """SetOriginalRange, then whole-grid updates (the pull rule after earlier local boxes)."""
    drv.original()
    for r in range(n_updates):
        drv.events(rand_vox(rng, drv.gs, n_ev), (rng.random(n_ev) < 0.5).astype(np.uint8))
        drv.update(tag=(tag, "whole grid", r))


def scenario_fixed_box(drv, observed, seed=0):
    """(a) local boxes -- a fixed one, then random ones -- and (d) the whole grid again after them."""
    rng = np.random.default_rng(seed)
    observe(drv, rng, observed, 300)
    o, res, G = np.asarray(drv.origin), drv.res, np.asarray(drv.gs)
    for r in range(4):
        c = o + (G * res) * (0.4, 0.55, 0.5) if r < 2 else o + rng.uniform(0.5, G * res - 0.5, 3)
        drv.set_box(c - (1.0, 1.0, 0.8), c + (1.0, 1.0, 0.8))
        drv.events(rand_vox(rng, drv.gs, 600), (rng.random(600) < 0.5).astype(np.uint8))
        drv.update(tag=("box", r))
    whole_grid_tail(drv, rng, tag="fixed")


def scenario_sliding_local_map(drv, seed=7):
    """(b) the sliding local map of test_gpu_edges.py::test_local_map_moving_box_exact (UpdateOccupancy(false), resets not
    skipped under PARAMS_DEFAULT) and (d) the whole grid again after it."""
    rng = np.random.default_rng(seed)
    allv = scenes.all_voxels(drv.gs)
    idx = rng.choice(len(allv), 300, replace=False)
    drv.events(allv, np.zeros(len(allv), np.uint8)); drv.update(tag="observe")
    drv.events(allv[idx], np.ones(300, np.uint8)); drv.update(tag="obstacles")
    drv.set_params(scenes.PARAMS_DEFAULT)
    for r in range(8):
        c = np.array([-1.2 + 0.35 * r, -0.9 + 0.3 * r, 0.0])
        drv.set_box(c - (1.3, 1.2, 0.9), c + (1.3, 1.2, 0.9))
        drv.events(rand_vox(rng, drv.gs, 6000), (rng.random(6000) < 0.4).astype(np.uint8))
        drv.update(global_map=False, tag=("slide", r))
    assert drv.resets > 0
    whole_grid_tail(drv, rng, n_ev=3000, tag="sliding")


def scenario_special_boxes(drv, seed=3):
    """(c) boxes on, across and beyond the grid's faces, one voxel, and empty after clamping with events pending that were
    counted under the previous box; then (d) the whole grid again."""
    rng = np.random.default_rng(seed)
    observe(drv, rng, 1.0, 250)
    o, sz, res = np.asarray(drv.origin), np.asarray(drv.size), drv.res
    v = np.array([17, 5, 30])
    boxes = [
        ("faces", o, o + sz),                                         # exactly the grid: the whole box again
        ("max faces", o + (0.9, 1.3, 0.7), o + sz),
        ("clipped low", o - (0.7, 0.4, 1.1), o + (1.3, 2.1, 1.7)),
        ("clipped high", o + sz - (1.6, 1.2, 2.0), o + sz + (0.8, 0.3, 0.5)),
        ("clamps to the grid", o - 1.0, o + sz + 1.0),
        ("one voxel", o + res * (v + 0.25), o + res * (v + 0.75)),
        ("one x-plane", o + res * np.array([20.25, -5, -5]), o + res * np.array([20.75, 50, 50])),
    ]
    for name, lo, hi in boxes:
        drv.set_box(lo, hi)
        if name == "one voxel":
            assert drv.cur[0] == drv.cur[1] == tuple(int(x) for x in v)
        drv.events(rand_vox(rng, drv.gs, 800), (rng.random(800) < 0.5).astype(np.uint8))
        drv.update(tag=name)
    # events counted under a local box, then a box that is empty after clamping (beyond the max faces)
    drv.set_box(o + 0.5, o + 2.5)
    drv.events(rand_vox(rng, drv.gs, 1500), (rng.random(1500) < 0.5).astype(np.uint8))
    drv.set_box(o + sz + 1.0, o + sz + 2.0)
    assert any(a > b for a, b in zip(*drv.cur))
    assert drv.update(tag="empty box") is not None
    drv.events(rand_vox(rng, drv.gs, 600), (rng.random(600) < 0.5).astype(np.uint8))   # nothing is counted now
    assert drv.update(tag="empty box, no events") is None
    whole_grid_tail(drv, rng, tag="special")


def scenario_alternating_local_map(drv, seed=9):
    """(e) a local map whose box alternates between covering the whole grid (after clamping) and covering part of it."""
    rng = np.random.default_rng(seed)
    observe(drv, rng, 1.0, 300)
    drv.set_params(scenes.PARAMS_DEFAULT)
    o, sz = np.asarray(drv.origin), np.asarray(drv.size)
    for r in range(8):
        if r % 2 == 0:
            lo, hi = o - 0.5, o + sz + 0.5
        else:
            c = o + rng.uniform(0.3, 0.7, 3) * sz
            lo, hi = c - (1.1, 0.9, 1.0), c + (1.1, 0.9, 1.0)
        drv.set_box(lo, hi)
        drv.events(rand_vox(rng, drv.gs, 3000), (rng.random(3000) < 0.4).astype(np.uint8))
        drv.update(global_map=False, tag=("alternate", r))
    assert drv.resets > 0


def scenario_raycast_local_map(drv, seed=5):
    """Ray-cast local map (the UpdateEsdfEvent steps of test_gpu_raycast_edges.py::test_local_map_casting): each frame cast
    under the box in force, then SetUpdateRange(pose +- radius), UpdateOccupancy(false), UpdateESDF; visualisation boxes
    with new_vec = false in between; then global updates."""
    o, sz = np.asarray(drv.origin), np.asarray(drv.size)
    centre = o + sz / 2
    radius = np.array([1.6, 1.4, 0.9])
    sc = scenes.Scene(tuple(sz / 2 * (0.85, 0.85, 0.8)), 8, 3, seed=seed, edge=(0.3, 0.9))
    poses = list(scenes.pose_walk(10, seed=6, clamp=1.0))
    for f, (p, yaw) in enumerate(poses):
        p = p + centre
        pts, T = scenes.depth_frame(sc, p, yaw, width=80, height=60, scale=0.125)
        drv.cast(pts, T)
        if f < 7:
            drv.set_box(p - radius, p + radius)
            drv.update(global_map=False, tag=("local frame", f))
            if f % 2 == 1:
                drv.set_box(p + (0.3, -0.2, 0.0) - radius, p + (0.3, -0.2, 0.0) + radius, new_vec=False)
        else:
            if f == 7:
                drv.original()
            drv.update(tag=("global frame", f))
        sc.step()
    assert drv.local_updates > 0


# ---------------------------------------------------------------- x-slab shards
def slabs(tx, world):
    """Tile columns [lo, hi) of every rank (fiesta_set_shard)."""
    return [(tx * r // world, tx * (r + 1) // world) for r in range(world)]


class ShardedModel:
    """One FastModel per rank on its x-slab, driven through the loop of shard.sharded_update_esdf: update on every rank,
    then rounds of pack, exchange, ingest and (where something changed) relax until no rank changed a record."""

    def __init__(self, oracle_mod, grid_size, res, l_occ, world, flags=0):
        self.gs, self.world, self.flags = tuple(grid_size), int(world), flags
        tx = (self.gs[0] + 7) // 8
        self.slab = slabs(tx, world)
        self.x = [(lo * 8, min(hi * 8, self.gs[0])) for lo, hi in self.slab]
        self.ranks = [oracle_mod.FastModel(self.gs, res, l_occ) for _ in range(world)]
        for m, (lo, hi) in zip(self.ranks, self.slab):
            m.set_slab(lo, hi)
        self.rounds = 0

    def set_range(self, lo, hi):
        for m in self.ranks:
            m.set_range(lo, hi)

    def esdf(self, dist, occ):
        """UpdateESDF on every rank; the changed records per rank."""
        return [m.update(dist, occ, self.flags)["changed"] for m in self.ranks]

    def exchange_round(self):
        """One round: every rank packs, the layers travel, every rank ingests and relaxes if a ghost record changed.
        Returns the changed records of every ingest and every relax (None where a rank did not relax)."""
        self.rounds += 1
        W = self.world
        lo_out = [m.pack(x0, 2) if r > 0 else None for r, (m, (x0, _)) in enumerate(zip(self.ranks, self.x))]
        hi_out = [m.pack(x1 - 2, 2) if r + 1 < W else None for r, (m, (_, x1)) in enumerate(zip(self.ranks, self.x))]
        ing, rel = [], []
        for r, m in enumerate(self.ranks):
            (x0, x1), (t0, t1) = self.x[r], self.slab[r]
            c = 0
            if r > 0:
                c += m.halo_ingest(hi_out[r - 1], x0 - 2, 2, t0)
            if r + 1 < W:
                c += m.halo_ingest(lo_out[r + 1], x1, 2, t1 - 1)
            ing.append(c)
            rel.append(m.relax(self.flags)["changed"] if c else None)
        return ing, rel

    def update(self, dist, occ):
        """The whole loop; returns the number of records the ingests changed."""
        self.esdf(dist, occ)
        ingested = 0
        while True:
            ing, rel = self.exchange_round()
            ingested += sum(ing)
            if sum(ing) + sum(x or 0 for x in rel) == 0:
                break
        for m in self.ranks:
            assert m.fresh_left() == 0
        return ingested

    def owned(self, r):
        """Closest obstacles (gx, gy, gz, 3) and distances (gx, gy, gz) of the layers rank r owns."""
        x0, x1 = self.x[r]
        c, d = self.ranks[r].export()
        return c.reshape(self.gs + (3,))[x0:x1], d.reshape(self.gs)[x0:x1]

    def export(self):
        """Every rank contributes the x-layers it owns."""
        C = np.concatenate([self.owned(r)[0] for r in range(self.world)])
        D = np.concatenate([self.owned(r)[1] for r in range(self.world)])
        return C.reshape(-1, 3), D.reshape(-1)

    def close(self):
        for m in self.ranks:
            m.close()


def shard_geom(gx):
    """A gx x 40 x 24 map centred on the origin of the scenes."""
    size = ((gx - 0.5) * 0.1, 3.95, 2.35)
    return tuple(-s / 2 for s in size), 0.1, size


class ShardDriver:
    """The reference build (event source), the unsharded FAST model and the sharded one, and optionally -- on the GPU --
    one FAST-mode ESDFMap per rank on the same device plus an unsharded one.  After every update the gathered sharded
    model equals the unsharded model.  With maps: each rank's owned layers equal its model rank after UpdateESDF and after
    every exchange round, with the same changed-record count for every UpdateESDF, shard_ingest and shard_relax, and the
    gathered field equals the unsharded map's."""

    def __init__(self, oracle_mod, geom, params, world, device_maps=False):
        self.origin, self.res, self.size = geom
        self.ora = oracle_mod.OracleMap(*geom)
        self.ora.SetParameters(*params)
        self.gs = self.ora.grid_size
        l_occ = logit(params[4])
        self.one = oracle_mod.FastModel(self.gs, self.res, l_occ)
        self.sh = ShardedModel(oracle_mod, self.gs, self.res, l_occ, world)
        self.world = world
        self.maps, self.bufs, self.single = [], [], None
        if device_maps:
            import torch
            import fiesta_b200
            from fiesta_b200 import shard
            mk = lambda: fiesta_b200.ESDFMap(*geom, mode="fast")
            self.single = mk()
            self.single.SetParameters(*params)
            for r in range(world):
                m = mk()
                m.SetParameters(*params)
                info = m.set_shard(r, world)
                assert (info.x_begin, info.x_end) == self.sh.x[r]
                self.maps.append(m)
                self.bufs.append(shard.HaloBuffers(info.layer_words, torch.device("cuda", m.device)))
        self.ingested = 0
        # With unknown voxels as barriers the 24-neighbourhood wave has more than one fixpoint and the slab schedule may
        # settle on another one than the unsharded schedule; on fully observed grids both are the reference's field.
        self.gather_exact = True

    def all_maps(self):
        return [self.ora] + self.maps + ([self.single] if self.single is not None else [])

    def set_box(self, lo, hi):
        for m in self.all_maps():
            m.SetUpdateRange(tuple(lo), tuple(hi))
        box = vox_box(self.origin, self.res, self.size, lo, hi)
        self.one.set_range(*box)
        self.sh.set_range(*box)

    def original(self):
        for m in self.all_maps():
            m.SetOriginalRange()
        full = ((0, 0, 0), tuple(g - 1 for g in self.gs))
        self.one.set_range(*full)
        self.sh.set_range(*full)

    def events(self, vox, occ):
        for m in self.all_maps():
            m.SetOccupancyBatchVox(vox, occ)

    def cast(self, pts, T, lo=0.3, hi=4.0):
        r = self.ora.RaycastFrame(pts, T, lo, hi)
        for m in self.all_maps()[1:]:
            assert m.RaycastFrame(pts, T, lo, hi) == r

    def _check_owned(self, tag):
        for r, m in enumerate(self.maps):
            x0, x1 = self.sh.x[r]
            c, d = self.sh.owned(r)
            C = m.export_closest_obstacle().reshape(self.gs + (3,))[x0:x1]
            D = m.export_distance().reshape(self.gs)[x0:x1]
            assert np.array_equal(D, d), (tag, "rank", r, int((D != d).sum()))
            assert np.array_equal(C, c), (tag, "rank", r, int((C != c).any(axis=-1).sum()))

    def update(self, tag=""):
        if not self.ora.CheckUpdate():
            return
        self.ora.UpdateOccupancy(True)
        dist, occ = self.ora.export_distance(), self.ora.export_occupancy()
        for m in self.all_maps()[1:]:
            m.UpdateOccupancy(True)
            assert np.array_equal(m.export_occupancy(), occ), tag
        self.one.update(dist, occ)
        ch = self.sh.esdf(dist, occ)
        for r, m in enumerate(self.maps):
            m.UpdateESDF()
            assert m.stats()["voxels_changed"] == ch[r], (tag, "UpdateESDF", r)
        self._check_owned((tag, "UpdateESDF"))
        rounds = 0
        while True:
            rounds += 1
            ing, rel = self.sh.exchange_round()
            self.ingested += sum(ing)
            if self.maps:
                self._device_round(ing, rel, (tag, "round", rounds))
            if sum(ing) + sum(x or 0 for x in rel) == 0:
                break
            assert rounds < 10000, tag
        for m in self.sh.ranks:
            assert m.fresh_left() == 0, tag
        self.ora.UpdateESDF()
        C1, D1 = self.one.export()
        if self.gather_exact:
            C, D = self.sh.export()
            assert np.array_equal(D, D1) and np.array_equal(C, C1), (tag, "sharded model vs unsharded", int((D != D1).sum()))
        if self.single is not None:
            self.single.UpdateESDF()
            assert_identical(self.single, C1, D1, (tag, "unsharded map"))

    def _device_round(self, ing, rel, tag):
        """The same round on the device maps: pack on every rank, copy rank r's send_hi to rank r+1's recv_lo and rank r+1's
        send_lo to rank r's recv_hi (device to device), ingest, relax where a ghost record changed."""
        import torch
        W, B = self.world, self.bufs
        ptr = lambda t: t.data_ptr()
        for r, m in enumerate(self.maps):
            m.shard_pack(ptr(B[r].send_lo) if r > 0 else 0, ptr(B[r].send_hi) if r + 1 < W else 0)
        for r in range(W):
            if r > 0:
                B[r].recv_lo.copy_(B[r - 1].send_hi)
            if r + 1 < W:
                B[r].recv_hi.copy_(B[r + 1].send_lo)
        torch.cuda.synchronize()
        for r, m in enumerate(self.maps):
            c = m.shard_ingest(ptr(B[r].recv_lo) if r > 0 else 0, ptr(B[r].recv_hi) if r + 1 < W else 0)
            assert c == ing[r], (tag, "shard_ingest", r, c, ing[r])
            if c:
                n = m.shard_relax()
                assert n == rel[r], (tag, "shard_relax", r, n, rel[r])
        self._check_owned(tag)

    def close(self):
        self.one.close()
        self.sh.close()
        self.ora.close()
        for m in self.all_maps()[1:]:
            m.close()


def scenario_shards(drv, observed, seed=1, frames=True):
    """Random insert/delete, a wall across every internal slab face that is then deleted (dependants on both sides),
    obstacles in the ghost layers x0-2 .. x0+1 of every face, an update under a local box that crosses a face, and two
    ray-cast frames."""
    rng = np.random.default_rng(seed)
    gs = drv.gs
    allv = scenes.all_voxels(gs)
    if observed < 1.0:
        allv = allv[rng.random(len(allv)) < observed]
        drv.gather_exact = False
    drv.events(allv, np.zeros(len(allv), np.uint8))
    drv.update("observe")
    for r in range(3):
        drv.events(rand_vox(rng, gs, 500), (rng.random(500) < 0.5).astype(np.uint8))
        drv.update(("random", r))
    faces = [x0 for x0, _ in drv.sh.x[1:]]
    yy, zz = np.meshgrid(np.arange(4, gs[1] - 4), np.arange(2, gs[2] - 2), indexing="ij")
    wall = np.concatenate([np.stack([np.full(yy.size, x), yy.ravel(), zz.ravel()], -1) for f in faces for x in (f - 1, f)]).astype(np.int32)
    if len(wall):
        drv.events(wall, np.ones(len(wall), np.uint8))
        drv.update("wall")
        drv.events(wall, np.zeros(len(wall), np.uint8))
        drv.update("wall deleted")
    ghost = []
    for f in faces:
        n = 120
        ghost.append(np.stack([rng.integers(f - 2, f + 2, n), rng.integers(0, gs[1], n), rng.integers(0, gs[2], n)], -1))
    if ghost:
        ghost = np.concatenate(ghost).astype(np.int32)
        drv.events(ghost, np.ones(len(ghost), np.uint8))
        drv.update("ghost-layer obstacles")
        drv.events(ghost[::2], np.zeros(len(ghost[::2]), np.uint8))
        drv.update("ghost-layer deletes")
    f = faces[len(faces) // 2] if faces else gs[0] // 2
    o = np.asarray(drv.origin)
    lo = o + drv.res * np.array([f - 6.5, 5, 3])
    hi = o + drv.res * np.array([f + 5.5, gs[1] - 9, gs[2] - 5])
    drv.set_box(lo, hi)
    drv.events(rand_vox(rng, gs, 1500), (rng.random(1500) < 0.5).astype(np.uint8))
    drv.update("local box across a face")
    drv.original()
    drv.events(rand_vox(rng, gs, 500), (rng.random(500) < 0.5).astype(np.uint8))
    drv.update("whole grid again")
    if frames:
        sz = np.asarray(drv.size)
        sc = scenes.Scene(tuple(sz / 2 * (0.85, 0.85, 0.8)), 6, 2, seed=seed, edge=(0.2, 0.6))
        for k, (p, yaw) in enumerate(scenes.pose_walk(2, seed=seed + 1, clamp=0.3)):
            pts, T = scenes.depth_frame(sc, p, yaw, width=80, height=60, scale=0.125)
            drv.cast(pts, T)
            drv.update(("frame", k))
            sc.step()
