"""CPU tests of the FAST-mode model (oracle/fast_model.c) under update boxes, local-map resets and x-slab shards.

The model is driven with the reference build (oracle/_ref, else the C port), as in tests/test_fast_model.py.  After every
update the base model, the variant in which every queued voxel pulls and the exit-test variant must agree bit for bit and
no FRESH flag may be left -- also after earlier updates under a local box, where the pull skip used to lose values (the
whole-grid updates that follow each scenario).  The sharded model, gathered over its ranks, must equal the unsharded one.
tests/test_gpu_fast_boxes.py holds the kernels to the same model on the device.
"""
import numpy as np
import pytest

from tests import fastbox, scenes


def driver(oracle_mod, geom=fastbox.GEOM, params=scenes.PARAMS_TOGGLE):
    return fastbox.BoxDriver(oracle_mod, *geom, params)


@pytest.mark.parametrize("observed", [1.0, 0.6])
def test_fixed_box_then_whole_grid(oracle_built, observed):
    drv = driver(oracle_built)
    fastbox.scenario_fixed_box(drv, observed)
    if observed == 1.0:
        assert drv.distance_mismatch() == 0          # fully observed, whole grid: FAST equals the reference's distances
    drv.close()


def test_sliding_local_map_then_whole_grid(oracle_built):
    drv = driver(oracle_built, fastbox.GEOM_EDGES)
    fastbox.scenario_sliding_local_map(drv)
    drv.close()


def test_special_boxes(oracle_built):
    drv = driver(oracle_built)
    fastbox.scenario_special_boxes(drv)
    drv.close()


def test_alternating_local_map(oracle_built):
    drv = driver(oracle_built)
    fastbox.scenario_alternating_local_map(drv)
    drv.close()


def test_raycast_local_map(oracle_built):
    drv = driver(oracle_built, fastbox.GEOM_EDGES, scenes.PARAMS_DEFAULT)
    fastbox.scenario_raycast_local_map(drv)
    drv.close()


def test_pull_skip_is_unsafe_after_a_local_box(oracle_built):
    """The reason for the sticky pull flag (the setup of scenario (d) that found it): a voxel outside a local box never had
    its neighbours' values pushed to it (VoxInRange(new_pos), ESDFMap.cpp:351), and the first whole-grid update after the
    box phase has to pull them.  Skipping the pull there, as the model did while the box was the whole grid, left 1451
    records different from the every-voxel-pulls variant on this map."""
    drv = driver(oracle_built)
    rng = np.random.default_rng(0)
    fastbox.observe(drv, rng, 1.0, 300)
    o, G = np.asarray(drv.origin), np.asarray(drv.gs) * drv.res
    for r in range(4):
        c = o + rng.uniform(0.5, G - 0.5, 3)
        drv.set_box(c - (1.0, 1.0, 0.8), c + (1.0, 1.0, 0.8))
        drv.events(fastbox.rand_vox(rng, drv.gs, 600), (rng.random(600) < 0.5).astype(np.uint8))
        drv.update(tag=("box", r))
    drv.original()
    drv.events(fastbox.rand_vox(rng, drv.gs, 600), (rng.random(600) < 0.5).astype(np.uint8))
    st = drv.update(tag="whole grid")
    assert st["changed"] > 0
    drv.close()


# ---------------------------------------------------------------- x-slab shards
def shard_check_run(oracle_mod, world, n_updates=5):
    """The scenario of tests/gpu_shard_check.py: a 64 x 64 x 32 map, everything observed, then random insert/delete
    rounds; the sharded model against the unsharded model and the reference after every update."""
    origin, res, size = (-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.2)
    params = scenes.PARAMS_TOGGLE
    ora = oracle_mod.OracleMap(origin, res, size)
    ora.SetParameters(*params)
    gs = ora.grid_size
    l_occ = fastbox.logit(params[4])
    one = oracle_mod.FastModel(gs, res, l_occ)
    sh = fastbox.ShardedModel(oracle_mod, gs, res, l_occ, world)
    rng = np.random.default_rng(3)
    allv = scenes.all_voxels(gs)
    ingested = 0
    for r in range(n_updates):
        if r == 0:
            vox, occ = allv, np.zeros(len(allv), np.uint8)
        else:
            vox = fastbox.rand_vox(rng, gs, 400)
            occ = (rng.random(400) < 0.5).astype(np.uint8)
        ora.SetOccupancyBatchVox(vox, occ)
        ora.UpdateOccupancy(True)
        d, o = ora.export_distance(), ora.export_occupancy()
        one.update(d, o)
        ingested += sh.update(d, o)
        ora.UpdateESDF()
        C1, D1 = one.export()
        C, D = sh.export()
        assert np.array_equal(D, D1) and np.array_equal(C, C1), (world, r, int((D != D1).sum()))
        assert np.array_equal(D, ora.export_distance()), (world, r)
    sh.close(); one.close(); ora.close()
    return ingested


def test_sharded_model_world_1_equals_unsharded(oracle_built):
    assert shard_check_run(oracle_built, 1, n_updates=3) == 0


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_model_equals_unsharded_and_reference(oracle_built, world):
    assert shard_check_run(oracle_built, world) > 0         # ghost records did travel


def test_slabs_match_set_shard():
    """The slab split the model uses is fiesta_set_shard's: tile columns tx*r/world .. tx*(r+1)/world."""
    assert fastbox.slabs(3, 3) == [(0, 1), (1, 2), (2, 3)]
    assert fastbox.slabs(5, 4) == [(0, 1), (1, 2), (2, 3), (3, 5)]
    assert fastbox.slabs(8, 3) == [(0, 2), (2, 5), (5, 8)]


SHARD_CASES = [(64, 2), (64, 3), (64, 4), (33, 2), (33, 4), (24, 3), (18, 3)]


@pytest.mark.parametrize("gx,world", SHARD_CASES)
@pytest.mark.parametrize("observed", [1.0, 0.6])
def test_sharded_model_scenarios(oracle_built, gx, world, observed):
    """The shard scenarios of tests/test_gpu_fast_boxes.py on the model alone: ghost records travel, and on fully observed
    grids the gathered sharded model equals the unsharded one after every update."""
    drv = fastbox.ShardDriver(oracle_built, fastbox.shard_geom(gx), scenes.PARAMS_TOGGLE, world)
    fastbox.scenario_shards(drv, observed)
    assert drv.ingested > 0
    drv.close()
