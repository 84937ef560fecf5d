"""CPU tests of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports every symbol that
include/fiesta_b200.h declares.  No compute is attempted here (no GPU); creating a map must fail loudly, not fall back."""
import ctypes as C
import os
import re

import pytest

import fiesta_b200
from fiesta_b200 import build as fb_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    fb_build.build()
    return fiesta_b200.load_library()


def test_header_and_library_agree(lib):
    hdr = open(os.path.join(ROOT, "include", "fiesta_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(fiesta_[a-z_0-9]+)\s*\(", hdr)))
    assert declared == sorted(fiesta_b200.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name


def test_struct_layouts_match_header():
    assert C.sizeof(fiesta_b200.Config) == 3 * 8 + 8 + 3 * 8 + 4 + 7 * 4
    assert C.sizeof(fiesta_b200.RaycastParams) == 16
    assert C.sizeof(fiesta_b200.Stats) == 14 * 8 + 6 * 4


def test_sass_is_sm90a_with_tma():
    import subprocess
    out = subprocess.run(["cuobjdump", "-sass", fiesta_b200.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "UTMALDG" in out          # the wavefront kernel stages tiles with TMA
    assert "SYNCS" in out            # mbarrier


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the no-device path cannot be exercised")
    with pytest.raises(fiesta_b200.FiestaError):
        fiesta_b200.ESDFMap((0, 0, 0), 0.1, (1, 1, 1))


def test_product_never_imports_oracle():
    """The product package and the C ABI sources must not reference oracle/ (test infrastructure)."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "fiesta_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "pyoracle" not in txt and "libfiesta_ref" not in txt and "libfiesta_oracle" not in txt, f
