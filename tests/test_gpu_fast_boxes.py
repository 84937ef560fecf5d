"""FAST mode on the GPU against its CPU model (oracle/fast_model.c) under update boxes, local-map resets and x-slab shards.

Boxes: the scenarios of tests/test_fast_model_boxes.py and a ray-cast local map run through a FAST ESDFMap next to the
reference build and the model.  After every update the device's closest obstacles and distances equal the model's bit for
bit, its changed-voxel and generation counts equal the model's, and its occupancy and counters equal the reference's.

Shards: N FAST maps on one device, each with set_shard(r, N), exchange their ghost layers through device copies in the loop
of fiesta_b200.shard.sharded_update_esdf, next to the sharded model.  After UpdateESDF and after every exchange round each
rank's owned layers equal the model's and every UpdateESDF, shard_ingest and shard_relax changes as many records as the
model's call did.
"""
import numpy as np
import pytest

from tests import fastbox, scenes

pytestmark = pytest.mark.gpu


def box_driver(oracle_mod, geom=fastbox.GEOM, params=scenes.PARAMS_TOGGLE):
    import fiesta_b200
    dev = fiesta_b200.ESDFMap(*geom, mode="fast")
    return fastbox.BoxDriver(oracle_mod, *geom, params, dev=dev)


@pytest.mark.parametrize("observed", [1.0, 0.6])
def test_fixed_box_then_whole_grid(oracle_built, observed):
    drv = box_driver(oracle_built)
    fastbox.scenario_fixed_box(drv, observed)
    drv.close()


def test_sliding_local_map_then_whole_grid(oracle_built):
    drv = box_driver(oracle_built, fastbox.GEOM_EDGES)
    fastbox.scenario_sliding_local_map(drv)
    drv.close()


def test_special_boxes(oracle_built):
    drv = box_driver(oracle_built)
    fastbox.scenario_special_boxes(drv)
    drv.close()


def test_alternating_local_map(oracle_built):
    drv = box_driver(oracle_built)
    fastbox.scenario_alternating_local_map(drv)
    drv.close()


def test_raycast_local_map(oracle_built):
    drv = box_driver(oracle_built, fastbox.GEOM_EDGES, scenes.PARAMS_DEFAULT)
    fastbox.scenario_raycast_local_map(drv)
    drv.close()


# ---------------------------------------------------------------- x-slab shards on one GPU
@pytest.mark.parametrize("gx,world", [(64, 2), (64, 3), (64, 4), (33, 2), (33, 4), (24, 3), (18, 3)])
@pytest.mark.parametrize("observed", [1.0, 0.6])
def test_shards_on_one_gpu_equal_sharded_model(oracle_built, gx, world, observed):
    drv = fastbox.ShardDriver(oracle_built, fastbox.shard_geom(gx), scenes.PARAMS_TOGGLE, world, device_maps=True)
    fastbox.scenario_shards(drv, observed)
    assert drv.ingested > 0
    drv.close()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_shard_check_scenario_on_one_gpu(oracle_built, world):
    """The scenario of tests/gpu_shard_check.py: the gathered field also equals the unsharded FAST map and the reference."""
    drv = fastbox.ShardDriver(oracle_built, ((-3.2, -3.2, -1.6), 0.1, (6.4, 6.4, 3.2)), scenes.PARAMS_TOGGLE, world,
                              device_maps=True)
    rng = np.random.default_rng(3)
    allv = scenes.all_voxels(drv.gs)
    for r in range(5):
        if r == 0:
            vox, occ = allv, np.zeros(len(allv), np.uint8)
        else:
            vox = fastbox.rand_vox(rng, drv.gs, 400)
            occ = (rng.random(400) < 0.5).astype(np.uint8)
        drv.events(vox, occ)
        drv.update(("shard check", r))
        D = np.concatenate([m.export_distance().reshape(drv.gs)[x0:x1] for m, (x0, x1) in zip(drv.maps, drv.sh.x)]).reshape(-1)
        assert np.array_equal(D, drv.single.export_distance()), r
        assert np.array_equal(D, drv.ora.export_distance()), r
    assert drv.ingested > 0
    drv.close()


def test_set_shard_refusals():
    import fiesta_b200

    def fast(gx):
        return fiesta_b200.ESDFMap((0.0, 0.0, 0.0), 0.1, ((gx - 0.5) * 0.1, 1.6, 1.6), mode="fast")

    m = fast(17)                                         # tiles 0-7, 8-15, 16: the last slab would be 1 voxel wide
    assert m.grid_size[0] == 17
    for r in range(3):
        with pytest.raises(fiesta_b200.FiestaError, match=r"\(4\)"):
            m.set_shard(r, 3)
    m.set_shard(1, 2)                                    # two ranks are fine on the same grid
    m.close()
    m = fast(18)
    assert m.set_shard(2, 3).x_end - m.set_shard(2, 3).x_begin == 2
    m.close()
    m = fast(24)                                         # 3 tile columns: at most 3 ranks
    m.set_shard(2, 3)
    with pytest.raises(fiesta_b200.FiestaError, match=r"\(4\)"):
        m.set_shard(0, 4)
    m.close()
    e = fiesta_b200.ESDFMap((0.0, 0.0, 0.0), 0.1, (2.35, 1.6, 1.6), mode="exact")
    with pytest.raises(fiesta_b200.FiestaError, match=r"\(1\)"):
        e.set_shard(0, 2)
    e.close()
