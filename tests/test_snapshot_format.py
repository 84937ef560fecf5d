"""CPU: the map snapshot format (fiesta_b200/csrc/fb_snapshot.h) compiled with g++.  tests/cpp/snapshot_test.cpp round-trips the
header and checks that every host-side rule rejects: truncation at every length below the header (and through the stream), a
bad magic or version, a header checksum mismatch, a config whose grid differs from the stored one, grids over the limits, update
boxes outside the grid, tile lists not ascending or past the grid, a total size that does not match, and the depth section.  The
checksum is checked against known vectors and against an independent Python restatement."""
import os
import subprocess

import numpy as np
import pytest

from tests import snapshot_tool

KNOWN = [(b"", 0xE220A8397B1DCDAF), (bytes(8), 0x2A98F501AF37E97F), (bytes(range(64)), 0x452D9044068A901B),
         (b"FIESTASN" * 3, 0xF0EF91E80E4722F2)]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return snapshot_tool.build(tmp_path_factory.mktemp("snap"))


def test_header_rules(exe):
    r = subprocess.run([exe, "selftest"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("ok ")


def _sum(exe, tmp_path, data):
    p = os.path.join(str(tmp_path), "words.bin")
    with open(p, "wb") as f:
        f.write(data)
    return int(subprocess.check_output([exe, "sum", p], text=True), 16)


@pytest.mark.parametrize("data,want", KNOWN)
def test_checksum_known_vectors(exe, tmp_path, data, want):
    assert snapshot_tool.checksum(data) == want
    assert _sum(exe, tmp_path, data) == want


def test_checksum_matches_restatement(exe, tmp_path):
    rng = np.random.default_rng(7)
    for n in (1, 3, 64, 257):
        data = rng.integers(0, 256, 8 * n, dtype=np.uint8).tobytes()
        want = snapshot_tool.checksum(data)
        assert _sum(exe, tmp_path, data) == want
        flipped = bytearray(data)
        flipped[rng.integers(0, len(data))] ^= 1 << int(rng.integers(0, 8))
        assert snapshot_tool.checksum(bytes(flipped)) != want
