"""GPU: cost matrices (fiesta_nav_matrix) against tests/navmatrixref.py evaluated on export_distance() of the same map -- matrix,
statuses and the predictable stats bit for bit, NaN included -- on ray-cast maps in both modes, on the whole grid, a local box and
boxes on every grid face, at three clearances with the unknown flag on and off, and on the serpentine maze.  Also: rows against
NavField.compute + export and NavField.paths, pass splitting, early retirement, determinism, permutations, isolation from the
map and from the field object's last compute, and argument validation."""
import ctypes as C

import numpy as np
import pytest

from tests import navmatrixref, navref
from tests.test_gpu_nav import ORIGIN, RES, SIZES, boxes, maze_map, raycast_map, same

pytestmark = pytest.mark.gpu


def expected(m, D, box, src, tgt, r, unk):
    lo = np.asarray(ORIGIN)
    return navmatrixref.matrix(D, m.grid_size, box, src, tgt, r, unk, ORIGIN, m.resolution, lo, lo + np.asarray(m.size_m))


def check(m, nav, box, src, tgt, r, unk, D=None):
    """Matrix on the device against navmatrixref, bit for bit; returns (cost, src_status, tgt_status, stats)."""
    D = m.export_distance() if D is None else D
    got = nav.matrix(box[0], box[1], src, tgt, r, unknown_blocks=unk)
    want = expected(m, D, box, src, tgt, r, unk)
    for name, a, b in zip(("cost", "src_status", "tgt_status"), got[:3], want[:3]):
        assert same(a, b), (name, box, r, unk)
    st = got[3]
    for k, v in want[3].items():
        assert st[k] == v, (k, st[k], v)
    assert st["generations"] >= (1 if st["passes"] else 0) and st["ms_compute"] > 0
    return got


def points(m, box, k, rng, extra=True):
    """k positions in the box (jittered inside their voxels), and some outside the box, outside the map and a NaN."""
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    v = np.stack([rng.integers(lo[i], hi[i] + 1, k) for i in range(3)], -1)
    p = np.asarray(ORIGIN) + (v + rng.uniform(0.05, 0.95, v.shape)) * m.resolution
    if not extra:
        return p
    out = np.asarray(ORIGIN) + np.array([[-0.05, 0.2, 0.2], [0.2, 0.2, m.size_m[2] + 0.05]])
    return np.concatenate([p, out, [[np.nan, 0.0, 0.0]], np.asarray(ORIGIN) + 0.05 + 0 * p[:1]])


@pytest.mark.parametrize("kind,mode,size", [(k, m, "gz32") for k in ("lidar", "depth") for m in ("exact", "fast")] +
                         [("lidar", m, "gz30") for m in ("exact", "fast")])
def test_matrix_on_raycast_maps(kind, mode, size):
    m, _ = raycast_map(mode, kind, SIZES[size])
    nav = m.NavField()
    rng = np.random.default_rng(17)
    D = m.export_distance()
    finite = 0
    seen = set()
    for bi, box in enumerate(boxes(m.grid_size)):
        for r in (0.0, RES, 2.5 * RES):
            for unk in (False, True):
                src = points(m, box, 5, rng)
                tgt = np.concatenate([points(m, box, 9, rng), src[:3]])
                cost, ss, ts, _ = check(m, nav, box, src, tgt, r, unk, D)
                finite += int(np.sum(np.isfinite(cost)))
                seen |= set(ss.tolist()) | set(ts.tolist())
                if r == RES and not unk and bi < 2:
                    cross_check(m, nav, box, src, tgt, r, cost, ss, ts)
    assert finite > 0 and seen == {0, 1, 2}, seen
    nav.close()


def cross_check(m, nav, box, src, tgt, r, cost, ss, ts):
    """Rows against the existing solver: compute(goals=[source]) + export() read at the targets, and paths() from the targets."""
    v, ok = navref.locate(tgt, ORIGIN, m.resolution, box)
    for i in np.nonzero(ss == 0)[0][:3]:
        nav.compute(box[0], box[1], src[i][None], r)
        F = nav.export()
        good = ts == 0
        assert np.array_equal(F[tuple(v[good].T)], cost[i, good])
        pst, _, pcost, _ = nav.paths(tgt[good], 4000)
        assert np.array_equal(pcost, cost[i, good]) and set(pst.tolist()) <= {0, 1}


def test_maze_needs_hundreds_of_generations():
    m = maze_map()
    gs = m.grid_size
    nav = m.NavField()
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    vox = np.array([[1, 0, 5], [90, 94, 2], [40, 45, 7], [60, 1, 3], [5, 93, 9]])
    p = np.asarray(ORIGIN) + (vox + 0.5) * RES
    cost, _, _, st = check(m, nav, box, p, p, 0.0, False)
    assert st["generations"] > 200, st
    assert cost[0, 1] > 80 * 32 * RES * 0.9                                # the far end is reached the long way round
    nav.close()


def test_more_than_one_pass_equals_one_call_per_source():
    m, _ = raycast_map("fast", "lidar", SIZES["gz32"], frames=2)
    nav = m.NavField()
    rng = np.random.default_rng(4)
    box = ((6, 4, 2), (57, 60, 29))
    src = points(m, box, 90, rng, extra=False)
    tgt = points(m, box, 20, rng)
    cost, ss, ts, st = check(m, nav, box, src, tgt, RES, False)
    placed = int(np.sum(ss == 0))
    assert placed > 64 and st["passes"] == 3, st
    for i in range(len(src)):
        c1, s1, t1, st1 = nav.matrix(box[0], box[1], src[i][None], tgt, RES)
        assert same(c1[0], cost[i]) and s1[0] == ss[i] and same(t1, ts)
        assert st1["passes"] == (1 if s1[0] == 0 else 0)
    nav.close()


def test_near_targets_retire_early():
    """Targets within a few voxels of their sources in a large box: sources stop long before their fields cover the box."""
    m = maze_map()
    gs = m.grid_size
    nav = m.NavField()
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    vox = np.array([[10, 0, 5], [12, 1, 6], [14, 0, 4], [11, 1, 7]])                # one corridor, a few voxels apart
    p = np.asarray(ORIGIN) + (vox + 0.5) * RES
    cost, _, _, st = check(m, nav, box, p, p, 0.0, False)
    assert st["sources_retired_early"] > 0, st
    assert np.all(np.isfinite(cost))
    st_one = nav.compute(box[0], box[1], p[:1], 0.0)
    assert st["generations"] < st_one["generations"], (st, st_one)
    nav.close()


def test_determinism_permutation_and_isolation():
    m, _ = raycast_map("exact", "lidar", SIZES["gz30"], frames=3)
    rng = np.random.default_rng(21)
    box = ((4, 7, 1), (49, 55, 26))
    D0, O0 = m.export_distance(), m.export_occupancy()
    nav = m.NavField()
    goals = points(m, box, 3, rng, extra=False)
    nav.compute(box[0], box[1], goals, RES)
    F0 = nav.export()
    starts = points(m, box, 300, rng)
    P0 = nav.paths(starts, 64)
    src, tgt = points(m, box, 12, rng), points(m, box, 15, rng)
    A = check(m, nav, box, src, tgt, RES, False)
    B = nav.matrix(box[0], box[1], src, tgt, RES)
    assert all(same(a, b) for a, b in zip(A[:3], B[:3]))
    ps, pt = rng.permutation(len(src)), rng.permutation(len(tgt))
    Cm = nav.matrix(box[0], box[1], src[ps], tgt[pt], RES)
    assert same(Cm[0], A[0][np.ix_(ps, pt)]) and same(Cm[1], A[1][ps]) and same(Cm[2], A[2][pt])
    nav.matrix((0, 0, 0), tuple(g - 1 for g in m.grid_size), src, tgt, 2.5 * RES, unknown_blocks=True)   # a larger box
    # the map and the field object's last compute are untouched
    assert np.array_equal(m.export_distance(), D0) and np.array_equal(m.export_occupancy(), O0)
    assert np.array_equal(nav.export(), F0)
    assert all(same(a, b) for a, b in zip(P0, nav.paths(starts, 64)))
    nav.close()


def test_invalid_arguments_and_empty_sets():
    import fiesta_b200
    m, _ = raycast_map("fast", "lidar", SIZES["gz30"], frames=1)
    gs = m.grid_size
    L = m._L
    nav = m.NavField()
    rng = np.random.default_rng(2)
    box = ((2, 3, 4), (40, 50, 20))
    nav.compute(box[0], box[1], points(m, box, 2, rng, extra=False), RES)
    F = nav.export()
    src, tgt = np.ascontiguousarray(points(m, box, 4, rng)), np.ascontiguousarray(points(m, box, 5, rng))
    I3 = lambda v: np.ascontiguousarray(v, np.int32)
    ss, ts, cost = np.full(len(src), 7, np.int32), np.full(len(tgt), 7, np.int32), np.full((len(src), len(tgt)), 3.5)
    st = fiesta_b200.NavMatrixStats()

    def call(lo=box[0], hi=box[1], sp=src.ctypes, ns=len(src), tp=tgt.ctypes, nt=len(tgt), r=RES, flags=0, ssp=ss.ctypes,
             tsp=ts.ctypes, cp=cost.ctypes, h=nav._h):
        return L.fiesta_nav_matrix(h, I3(lo).ctypes if lo is not None else None, I3(hi).ctypes, sp, ns, tp, nt, C.c_double(r), flags,
                                   ssp, tsp, cp, C.byref(st))

    invalid = [call(lo=(5, 3, 4), hi=(4, 50, 20)), call(lo=(-1, 3, 4)), call(hi=(gs[0], 50, 20)), call(hi=(40, 50, gs[2])),
               call(lo=None), call(h=None), call(r=float("nan")), call(r=-0.1), call(r=10000.0), call(flags=2),
               call(ns=-1), call(nt=-1), call(sp=None), call(tp=None), call(ssp=None), call(tsp=None), call(cp=None)]
    assert invalid == [1] * len(invalid), invalid                           # FIESTA_ERR_INVALID
    assert call(ns=1 << 16, nt=1 << 15) == 4 and call(ns=1 << 31, nt=1) == 4   # FIESTA_ERR_LIMIT: n_src * n_tgt >= 2^31
    assert np.all(ss == 7) and np.all(ts == 7) and np.all(cost == 3.5)
    assert np.array_equal(nav.export(), F)
    # empty sets: statuses still written, nothing else needed
    D = m.export_distance()
    c0, s0, t0, st0 = nav.matrix(box[0], box[1], np.zeros((0, 3)), tgt, RES)
    assert c0.shape == (0, len(tgt)) and same(t0, expected(m, D, box, src, tgt, RES, False)[2]) and st0["passes"] == 0
    assert call(ns=0, sp=None, ssp=None, cp=None) == 0 and np.all(ts != 7)
    c1, s1, t1, st1 = nav.matrix(box[0], box[1], src, np.zeros((0, 3)), RES)
    assert c1.shape == (len(src), 0) and same(s1, expected(m, D, box, src, tgt, RES, False)[1]) and st1["passes"] == 0
    with pytest.raises(fiesta_b200.FiestaError):
        nav.matrix((0, 0, 0), (gs[0], 1, 1), src, tgt, RES)
    check(m, nav, box, src, tgt, RES, False)                                # still usable
    assert np.array_equal(nav.export(), F)
    nav.close()
