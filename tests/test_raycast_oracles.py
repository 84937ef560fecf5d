"""The crafted ray-casting scenes of tests/test_gpu_raycast_edges.py (off-lattice maps, faces and aliases, local update
boxes, mixed observation sources) run through both CPU oracles: the C restatement (the oracle the GPU tests fall back to)
must agree with the unmodified reference build in every frame -- rays cast, counters, SetOccupancy returns, dropped
rays -- and after every integration.  Needs oracle/_ref (built when FIESTA_REFERENCE names a FIESTA checkout)."""
import numpy as np
import pytest

from tests import scenes
from tests.test_gpu_raycast_edges import MAPS, drive_geometry, drive_local, drive_mixed, lattice_path


@pytest.fixture
def port_and_ref(oracle_built):
    if not oracle_built.available("ref"):
        pytest.skip("oracle/_ref is not built (set FIESTA_REFERENCE to a checkout of the FIESTA sources)")

    def make(name, params):
        origin, res, size, _ = MAPS[name]
        port = oracle_built.OracleMap(origin, res, size, kind="port")
        ref = oracle_built.OracleMap(origin, res, size, kind="ref")
        for m in (port, ref):
            m.SetParameters(*params)
        return port, ref
    return make


def test_lattice_path_guard():
    """The restated host predicate puts each test map on the side of the lattice fast path its tests are meant for, and the
    benchmark maps on the fast path."""
    for name, (origin, res, size, on_path) in MAPS.items():
        assert lattice_path(origin, res, size) == on_path, name
    assert {v[3] for v in MAPS.values()} == {True, False}
    for origin, res, size in (((-6.4, -6.4, -3.2), 0.1, (12.8, 12.8, 6.4)), ((-12.8, -12.8, -12.8), 0.05, (25.6, 25.6, 25.6)),
                              ((-6.4, -6.4, -6.4), 0.05, (12.8, 12.8, 12.8)), ((-25.6, -25.6, -12.8), 0.05, (51.2, 51.2, 25.6))):
        assert lattice_path(origin, res, size), origin


@pytest.mark.parametrize("name", list(MAPS))
def test_geometry_port_vs_reference(port_and_ref, name):
    port, ref = port_and_ref(name, scenes.PARAMS_TOGGLE)
    drive_geometry(port, ref, name, "exact")


@pytest.mark.parametrize("source", ["raycast", "depth"])
@pytest.mark.parametrize("name", ["std", "half", "dyadic30"])
def test_local_map_port_vs_reference(port_and_ref, oracle_built, name, source):
    port, ref = port_and_ref(name, scenes.PARAMS_DEFAULT)
    assert drive_local(port, ref, oracle_built, name, source, "exact") > 0


@pytest.mark.parametrize("box", [False, True])
def test_mixed_sources_port_vs_reference(port_and_ref, oracle_built, box):
    port, ref = port_and_ref("std", scenes.PARAMS_TOGGLE)
    drive_mixed(port, ref, oracle_built, box)
