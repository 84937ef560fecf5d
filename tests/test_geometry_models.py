"""CPU: the FAST-mode model (oracle/fast_model.c) against the reference on the grid shapes of tests/geometry.py --
degenerate, gy == 1, smaller than a tile, padded z pitch, off-tile and long thin grids up to 2046 voxels on an axis.  The GPU
test compares the kernels with this model bit for bit, so a failure there is in the kernels when this file passes."""
import numpy as np
import pytest

from tests import scenes
from tests.parity import invariants
from tests.geometry import ORIGIN, RES, SHAPES, logit, random_voxels, shape_id, size_of, special_voxels, trilinear

CPU_SHAPES = [gs for gs in SHAPES if np.prod(gs) < 1 << 20]


class ModelView:
    """The model's records with the reference's occupancy, in the shape parity.invariants reads."""

    def __init__(self, model, ora):
        self.grid_size, self.resolution = model.grid_size, model.res
        self._cobs, self._dist = model.export()
        self._occ = ora.export_occupancy()

    def export_distance(self):
        return self._dist

    def export_closest_obstacle(self):
        return self._cobs

    def export_occupancy(self):
        return self._occ


@pytest.mark.parametrize("gs", CPU_SHAPES, ids=shape_id)
def test_model_on_shape(oracle_built, gs):
    si = SHAPES.index(gs)
    rng = np.random.default_rng(2000 + si)
    params = scenes.PARAMS_TOGGLE
    l_occ = logit(params[4])
    ora = oracle_built.OracleMap(ORIGIN, RES, size_of(gs))
    ora.SetParameters(*params)
    assert ora.grid_size == gs
    model = oracle_built.FastModel(gs, RES, l_occ)
    allv = scenes.all_voxels(gs)[rng.permutation(int(np.prod(gs)))]
    observed = 1.0 if si % 4 < 2 else 0.6
    if observed < 1.0:
        allv = allv[rng.random(len(allv)) < observed]
    spec = special_voxels(gs)
    n = min(600, 4 * int(np.prod(gs)))
    batches = [(allv, np.zeros(len(allv), np.uint8))]
    for r in range(5):
        vox = np.concatenate([random_voxels(rng, gs, n), spec[rng.random(len(spec)) < 0.5]])
        batches.append((vox, (rng.random(len(vox)) < (0.7 if r < 2 else 0.4)).astype(np.uint8)))
    batches.append((np.array([[g - 1 for g in gs]], np.int32), np.ones(1, np.uint8)))
    finite = mismatched = 0
    for k, (vox, occ) in enumerate(batches):
        ora.SetOccupancyBatchVox(vox, occ)
        if not ora.CheckUpdate():
            continue
        ora.UpdateOccupancy(True)
        model.update(ora.export_distance(), ora.export_occupancy())
        ora.UpdateESDF()
        assert model.fresh_left() == 0, k
        cobs, dist = model.export()
        R = ora.export_distance()
        # observed / unknown state and obstacles are the reference's exactly
        assert np.array_equal(dist == -10000, R == -10000), k
        occupied = ora.export_occupancy() > l_occ
        assert np.array_equal(dist == 0, occupied), k
        inv = invariants(ModelView(model, ora), l_occ)
        assert not any(inv.values()), (k, inv)
        dm = dist != R
        fin = (R >= 0) & (R < 10000)
        finite += int(fin.sum())
        mismatched += int(dm.sum())
        if observed == 1.0:
            assert dm.sum() == 0, (k, int(dm.sum()))
            assert ((cobs != ora.export_closest_obstacle()).any(axis=1) & dm).sum() == 0, k
    assert mismatched <= 0.02 * max(1, finite), (mismatched, finite)
    # tests.geometry.trilinear (the GPU test's check of GetDistWithGradTrilinear in both modes) equals the reference wherever
    # the reference's 2x2x2 stencil lies inside the grid
    q = np.asarray(ORIGIN) + rng.uniform(-0.05, 1.05, (2048, 3)) * np.asarray(size_of(gs))
    d1, g1, inside = trilinear(ora.export_distance(), gs, q)
    d2, g2 = ora.GetDistWithGradTrilinearBatch(q)
    stencil_in = np.all((q - 0.5 * RES >= np.asarray(ORIGIN)) & (q + 0.5 * RES < np.asarray(ORIGIN) + np.asarray(size_of(gs))), axis=1)
    ok = ~inside | stencil_in
    assert np.array_equal(d1[ok], d2[ok]) and np.array_equal(g1[ok & inside], g2[ok & inside])
    assert (d1 == -1).sum() == (~inside).sum()
