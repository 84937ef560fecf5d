"""GPU test of the device-side visualisation extraction (SURVEY.md 8(f) next #2) against the REFERENCE's own
GetPointCloud / GetSliceMarker (tests/golden/reference_golden.json, section vis_replay, made by the compiled reference)."""
import json
import os

import pytest

from tests.golden import make_golden

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.json")))


def test_point_cloud_and_slice_marker():
    import fiesta_b200
    got = make_golden.vis_replay(lambda o, r, s: fiesta_b200.ESDFMap(o, r, s, mode="exact"))
    gold = GOLD["vis_replay"]
    assert gold["cloud_0_31"]["n"] > 50 and gold["local_slice_14"]["n"] > 0
    for k in gold:
        assert got[k] == gold[k], k
