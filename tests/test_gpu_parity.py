"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on identical inputs.

Oracle = the unmodified reference compiled in place (oracle/_ref) when it was built (FIESTA_REFERENCE), else the C
restatement (oracle/esdf_oracle.c).  Distances are compared bit-exactly (they derive from exact integer obstacle
coordinates); closest-obstacle differences are only tolerated where both obstacles are exactly equidistant.
"""
import numpy as np
import pytest

from tests import scenes
from tests.parity import compare, assert_exact_distance

pytestmark = pytest.mark.gpu


def make_pair(oracle_built, origin, res, size, params):
    import fiesta_b200
    dev = fiesta_b200.ESDFMap(origin, res, size, mode="fast")
    ora = oracle_built.OracleMap(origin, res, size)
    dev.SetParameters(*params)
    ora.SetParameters(*params)
    assert dev.grid_total_size_ == ora.grid_total_size_ and dev.grid_size == ora.grid_size
    return dev, ora


def feed(dev, ora, vox, occ):
    a = dev.SetOccupancyBatchVox(vox, occ)
    b = ora.SetOccupancyBatchVox(vox, occ)
    assert np.array_equal(a, b)
    assert dev.CheckUpdate() == ora.CheckUpdate()
    ra, rb = dev.UpdateOccupancy(True), ora.UpdateOccupancy(True)
    assert ra == rb
    dev.UpdateESDF()
    ora.UpdateESDF()
    sd, so = dev.stats(), ora.stats()
    assert sd["occupancy_updates"] == so["occupancy_updates"]
    assert sd["inserts"] == so["inserts"] and sd["deletes"] == so["deletes"]


def test_pillar_replay_64(oracle_built):
    """SURVEY.md 8(d) config 1 (intent of test/test_ESDF_Map.cpp:42-103): observe all, 25 pillars, delete in reverse."""
    dev, ora = make_pair(oracle_built, (-6.4, -6.4, 0.0), 0.2, (12.8, 12.8, 12.8), scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(dev.grid_size)
    feed(dev, ora, allv, np.zeros(len(allv), np.uint8))
    assert_exact_distance(dev, ora, "observe")
    sites = scenes.pillar_sites()
    for k, (x, y) in enumerate(sites):
        feed(dev, ora, scenes.pillar(x, y), np.ones(25, np.uint8))
        assert_exact_distance(dev, ora, "pillar %d" % k)
    # Appendix D golden values of the unmodified reference
    assert abs(dev.GetDistance((30, 30, 10)) - 0.565685425) < 1e-9
    d, g = dev.GetDistWithGradTrilinear((0.33, -1.27, 2.51))
    do, go = ora.GetDistWithGradTrilinear((0.33, -1.27, 2.51))
    assert d == do and np.array_equal(g, go)
    assert abs(d - 0.674154485) < 1e-9
    D = dev.export_distance()
    assert abs(D[(D >= 0) & (D < 10000)].sum() - 811976.768405) < 1e-3
    for k, (x, y) in enumerate(reversed(sites)):
        feed(dev, ora, scenes.pillar(x, y), np.zeros(25, np.uint8))
        assert_exact_distance(dev, ora, "delete %d" % k)
    D = dev.export_distance()
    assert ((D >= 0) & (D < 10000)).sum() == 0


@pytest.mark.parametrize("G,res", [(40, 0.1), (33, 0.125)])
def test_random_insert_delete_fully_observed(oracle_built, G, res):
    """Mixed insert/delete rounds on a fully observed grid (also a grid whose z extent is not a multiple of 4 or 8)."""
    rng = np.random.default_rng(7)
    size = ((G - 0.5) * res,) * 3
    dev, ora = make_pair(oracle_built, (-1.0, -2.0, 0.5), res, size, scenes.PARAMS_TOGGLE)
    gs = dev.grid_size
    allv = scenes.all_voxels(gs)
    feed(dev, ora, allv, np.zeros(len(allv), np.uint8))
    for r in range(6):
        n = 500
        vox = np.stack([rng.integers(0, gs[i], n) for i in range(3)], -1).astype(np.int32)
        occ = (rng.random(n) < 0.5).astype(np.uint8)
        feed(dev, ora, vox, occ)
        res_ = assert_exact_distance(dev, ora, "round %d" % r)
    # queries agree bit-for-bit
    pos = rng.uniform(-3, 6, (4000, 3))
    assert np.array_equal(dev.GetDistanceBatch(pos), ora.GetDistanceBatch(pos))
    lo = np.array([-1.0, -2.0, 0.5]) + res
    hi = lo + np.array(size) - 3 * res
    pos = rng.uniform(lo, hi, (4000, 3))
    d1, g1 = dev.GetDistWithGradTrilinearBatch(pos)
    d2, g2 = ora.GetDistWithGradTrilinearBatch(pos)
    assert np.array_equal(d1, d2) and np.array_equal(g1, g2)


def test_raycast_counters_match_serial_reference(oracle_built):
    """Per-voxel (num_hit_, num_miss_) after one frame equal the serial reference exactly, frame after frame."""
    dev, ora = make_pair(oracle_built, (-6.4, -6.4, -3.2), 0.1, (12.8, 12.8, 6.4), scenes.PARAMS_DEFAULT)
    sc = scenes.Scene((5.0, 5.0, 2.5), 20, 5, seed=2)
    poses = scenes.pose_walk(4, seed=3)
    for f, (p, yaw) in enumerate(poses):
        pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
        pts[::53] = np.nan
        ca = dev.RaycastFrame(pts, T, 0.5, 5.0)
        cb = ora.RaycastFrame(pts, T, 0.5, 5.0)
        assert ca == cb, (f, ca, cb)
        (h1, t1), (h2, t2) = dev.export_counters(), ora.export_counters()
        assert np.array_equal(h1, h2) and np.array_equal(t1, t2), (f, int((t1 != t2).sum()))
        assert dev.CheckUpdate() == ora.CheckUpdate()
        assert dev.UpdateOccupancy(True) == ora.UpdateOccupancy(True)
        dev.UpdateESDF()
        ora.UpdateESDF()
        r = compare(dev, ora)
        assert r["occ"] == 0, (f, r)
        print("frame", f, r, dev.stats())
        sc.step()


# ----------------------------------------------------------------------------------------------------------------------
# FIESTA_MODE_EXACT: the device reproduces the reference's sequential FIFO order, so EVERYTHING is bit-exact:
# distance_, closest_obstacle_ (no tie tolerance) and the number of non-stale queue pops ("Expanding N nodes").
def make_exact_pair(oracle_built, origin, res, size, params):
    import fiesta_b200
    dev = fiesta_b200.ESDFMap(origin, res, size, mode="exact")
    ora = oracle_built.OracleMap(origin, res, size)
    dev.SetParameters(*params)
    ora.SetParameters(*params)
    return dev, ora


def assert_identical(dev, ora, tag):
    r = compare(dev, ora)
    assert r["occ"] == 0 and r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0, (tag, r)
    sd, so = dev.stats(), ora.stats()
    assert sd["expansions"] == so["expansions"], (tag, sd["expansions"], so["expansions"])
    return r


def test_exact_pillar_replay(oracle_built):
    dev, ora = make_exact_pair(oracle_built, (-6.4, -6.4, 0.0), 0.2, (12.8, 12.8, 12.8), scenes.PARAMS_TOGGLE)
    allv = scenes.all_voxels(dev.grid_size)
    feed(dev, ora, allv, np.zeros(len(allv), np.uint8))
    sites = scenes.pillar_sites()
    rng = np.random.default_rng(1)
    order = rng.permutation(len(sites))                       # shuffled variant (SURVEY.md 8(d) config 1)
    for k in order:
        feed(dev, ora, scenes.pillar(*sites[k]), np.ones(25, np.uint8))
        assert_identical(dev, ora, "pillar %d" % k)
    for k in order[::-1][:13]:
        feed(dev, ora, scenes.pillar(*sites[k]), np.zeros(25, np.uint8))
        assert_identical(dev, ora, "delete %d" % k)


@pytest.mark.parametrize("observed,two_sorts", [(1.0, False), (0.6, False), (0.6, True)])
def test_exact_random_insert_delete(oracle_built, observed, two_sorts, monkeypatch):
    """Mixed insert/delete rounds, fully and partially (salt-and-pepper) observed: the adversarial case for tie-breaks.
    two_sorts: the dependant order through the two-key fallback (rank and relink clock no longer fit one 64-bit sort key)."""
    if two_sorts:
        monkeypatch.setenv("FIESTA_X_TWO_SORTS", "1")
    rng = np.random.default_rng(21)
    dev, ora = make_exact_pair(oracle_built, (-2.0, -2.0, -2.0), 0.1, (3.95, 3.95, 3.15), scenes.PARAMS_TOGGLE)
    gs = dev.grid_size
    allv = scenes.all_voxels(gs)
    sel = allv[rng.random(len(allv)) < observed]
    sel = sel[rng.permutation(len(sel))]                      # scrambled first-observation order
    feed(dev, ora, sel, (rng.random(len(sel)) < 0.01).astype(np.uint8))
    assert_identical(dev, ora, "observe")
    for r in range(6):
        n = 1500
        vox = np.stack([rng.integers(0, gs[i], n) for i in range(3)], -1).astype(np.int32)
        feed(dev, ora, vox, (rng.random(n) < 0.5).astype(np.uint8))
        assert_identical(dev, ora, "round %d" % r)
    pos = rng.uniform(-1.9, 1.0, (2000, 3))
    d1, g1 = dev.GetDistWithGradTrilinearBatch(pos)
    d2, g2 = ora.GetDistWithGradTrilinearBatch(pos)
    assert np.array_equal(d1, d2) and np.array_equal(g1, g2)


def test_exact_raycast_frames(oracle_built):
    """Depth frames into a partially observed map: counters, occupancy, distance_, closest_obstacle_ and the expansion
    count all equal the serial reference, frame after frame."""
    dev, ora = make_exact_pair(oracle_built, (-6.4, -6.4, -3.2), 0.1, (12.8, 12.8, 6.4), scenes.PARAMS_DEFAULT)
    sc = scenes.Scene((5.0, 5.0, 2.5), 20, 5, seed=2)
    for f, (p, yaw) in enumerate(scenes.pose_walk(5, seed=3)):
        pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
        assert dev.RaycastFrame(pts, T, 0.5, 5.0) == ora.RaycastFrame(pts, T, 0.5, 5.0)
        (h1, t1), (h2, t2) = dev.export_counters(), ora.export_counters()
        assert np.array_equal(h1, h2) and np.array_equal(t1, t2)
        assert dev.UpdateOccupancy(True) == ora.UpdateOccupancy(True)
        sd, so = dev.stats(), ora.stats()
        dev.UpdateESDF()
        ora.UpdateESDF()
        sd, so = dev.stats(), ora.stats()
        assert sd["inserts"] == so["inserts"] and sd["deletes"] == so["deletes"], (f, sd, so)
        r = assert_identical(dev, ora, "frame %d" % f)
        print("exact frame", f, r, {k: sd[k] for k in ("expansions", "voxels_changed", "generations", "ms_update_esdf")})
        sc.step()


def test_exact_256_insert_delete_replay(oracle_built):
    """north_star: bit-exact closest-obstacle indices vs the reference on a 256^3 insert/delete replay (all voxels observed,
    then +20 000 inserts / -10 000 deletes per frame)."""
    rng = np.random.default_rng(6)
    dev, ora = make_exact_pair(oracle_built, (-6.4, -6.4, -6.4), 0.05, (12.8, 12.8, 12.8), scenes.PARAMS_TOGGLE)
    assert dev.grid_size == (256, 256, 256)
    allv = scenes.all_voxels(dev.grid_size)
    feed(dev, ora, allv, np.zeros(len(allv), np.uint8))
    occupied = np.empty((0, 3), np.int32)
    for f in range(2):
        ins = rng.integers(0, 256, (20000, 3)).astype(np.int32)
        dele = occupied[rng.permutation(len(occupied))[:10000]] if len(occupied) else np.empty((0, 3), np.int32)
        vox = np.concatenate([ins, dele])
        occ = np.concatenate([np.ones(len(ins), np.uint8), np.zeros(len(dele), np.uint8)])
        perm = rng.permutation(len(vox))
        feed(dev, ora, vox[perm], occ[perm])
        r = assert_identical(dev, ora, "frame %d" % f)
        print("256^3 frame", f, r, dev.stats()["expansions"], dev.stats()["ms_update_esdf"])
        occupied = np.unique(np.concatenate([occupied, ins]), axis=0)
