"""CPU: the cost matrix's definition (tests/navmatrixref.py) against the cost-to-go field's (tests/navref.py), and the device
schedule with early retirement emulated on the CPU.

Every row of the matrix must be navref.field with that source as the only goal, read at the targets, with NaN wherever a point is
blocked, outside the box, outside the map or NaN.  The emulated k_navm_relax -- many channels in one work list, random tile orders,
both halo extremes, and a channel retired once its targets read <= m_c(g - 1) -- must give the same matrix, also on the crafted
cases the retirement rule is most likely to get wrong: a target in the source's voxel, unreachable targets, duplicates, sources
connected to free space only across a tile face, edge or corner, and ties where many targets sit at exactly m_c.  The move masks
of fb_nav.h (compiled with g++) must equal navref.move_mask in all 26 directions."""
import os
import subprocess

import numpy as np
import pytest

from tests import navmatrixref, navref
from tests.test_nav_oracle import BOUNDARY_CASES, CASES, boundary_grid, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.1
ORIGIN = np.array([-0.8, 0.3, -0.4])


def pos(v, rng):
    """Positions (metres) inside grid voxels v."""
    v = np.asarray(v, np.float64).reshape(-1, 3)
    return ORIGIN + (v + rng.uniform(0.1, 0.9, v.shape)) * RES


def points(gs, box, k, rng):
    """k positions in the box, a few in the grid outside the box, outside the map, a NaN, and duplicates of the first two."""
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    inside = np.stack([rng.integers(lo[i], hi[i] + 1, k) for i in range(3)], -1)
    p = [pos(inside, rng), pos([[0, 0, 0], [gs[0] - 1, gs[1] - 1, gs[2] - 1]], rng),
         ORIGIN + np.array([[-0.05, 0.1, 0.1], [0.1, gs[1] * RES + 0.05, 0.1]]), [[np.nan, 0.0, 0.0]]]
    p = np.concatenate(p)
    return np.concatenate([p, p[:2]])


def run(D, gs, box, src, tgt, r, unk):
    return navmatrixref.matrix(D, gs, box, src, tgt, r, unk, ORIGIN, RES, ORIGIN, ORIGIN + np.asarray(gs) * RES)


def check_rows(D, gs, box, src, tgt, r, unk):
    """Each row of the matrix equals the single-goal field at the targets; returns the matrix result."""
    cost, ss, ts, st = run(D, gs, box, src, tgt, r, unk)
    lo_map, hi_map = ORIGIN, ORIGIN + np.asarray(gs) * RES
    sv, sok = navref.locate(src, ORIGIN, RES, box, lo_map, hi_map)
    tv, tok = navref.locate(tgt, ORIGIN, RES, box, lo_map, hi_map)
    assert np.array_equal(ss == 2, ~sok) and np.array_equal(ts == 2, ~tok)
    for i in range(len(src)):
        want = np.full(len(tgt), np.nan)
        if ss[i] == 0:
            F = navref.field(D, gs, box, (sv[i] + np.asarray(box[0]))[None], r, unk, RES)
            assert F[tuple(sv[i])] == 0.0
            good = ts == 0
            want[good] = F[tuple(tv[good].T)]
            assert np.all(F[tuple(tv[ts == 1].T)] == -1) if np.any(ts == 1) else True
        else:
            assert np.all(np.isnan(cost[i]))
        assert np.array_equal(cost[i], want, equal_nan=True), (i, r, unk)
    assert st["sources_placed"] == int(np.sum(ss == 0)) and st["targets_placed"] == int(np.sum(ts == 0))
    return cost, ss, ts, st


def check_schedule(D, gs, box, src, tgt, r, unk, rng):
    """The emulated device schedule, with retirement and both halo extremes, gives the matrix; returns the early retirements."""
    cost, ss, ts, _ = run(D, gs, box, src, tgt, r, unk)
    T = navref.traversable(D.reshape(gs)[navref.box_slices(box)], r, unk)
    _, si = navmatrixref.status(T, box, src, ORIGIN, RES, ORIGIN, ORIGIN + np.asarray(gs) * RES)
    _, ti = navmatrixref.status(T, box, tgt, ORIGIN, RES, ORIGIN, ORIGIN + np.asarray(gs) * RES)
    rows, cols = np.nonzero(ss == 0)[0], np.nonzero(ts == 0)[0]
    early = 0
    if not len(rows) or not len(cols):
        return early
    tv = np.unravel_index(ti[cols], T.shape)
    for fresh in (True, False):
        F, _, e = navmatrixref.channel_worklist(T, si[rows], ti[cols], RES, rng, fresh)
        got = F[(slice(None),) + tv]
        assert np.array_equal(got, cost[np.ix_(rows, cols)]), (fresh, r, unk)
        early += e
    return early


@pytest.mark.parametrize("case", range(len(CASES)))
def test_rows_equal_single_goal_fields(case):
    gs, box, _ = CASES[case]
    rng = np.random.default_rng(40 + case)
    D = synth(gs, rng)
    finite = 0
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            src, tgt = points(gs, box, 5, rng), points(gs, box, 12, rng)
            cost, ss, ts, _ = check_rows(D, gs, box, src, tgt, r, unk)
            finite += int(np.sum(np.isfinite(cost)))
            assert {0, 2} <= set(ss.tolist()) | set(ts.tolist())
    assert finite > 0


@pytest.mark.parametrize("case", range(len(CASES)))
def test_emulated_schedule_with_retirement(case):
    gs, box, _ = CASES[case]
    rng = np.random.default_rng(60 + case)
    D = synth(gs, rng)
    for r in (0.0, 2.5 * RES):
        for unk in (False, True):
            check_schedule(D, gs, box, points(gs, box, 4, rng), points(gs, box, 6, rng), r, unk, rng)


def open_grid(gs=(24, 24, 16)):
    """Fully free: distances repeat, so many targets tie at exactly m_c."""
    return gs, np.ones(int(np.prod(gs)))


def test_crafted_cases_and_early_retirement():
    rng = np.random.default_rng(7)
    gs, D = open_grid()
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    c = np.array([12, 11, 8])
    ring = [c + d for d in navref.OFFSETS]                   # all 26 neighbours: 6 + 12 + 8 ties
    src = pos([c, c, [3, 3, 3]], rng)                        # a duplicate source
    tgt = np.concatenate([pos(np.concatenate([[c], ring, [c + (2, 0, 0)]]), rng), src[:1]])   # the source's own voxel twice
    cost, ss, ts, _ = check_rows(D, gs, box, src, tgt, 0.5, False)
    assert cost[0, 0] == 0.0 and cost[0, -1] == 0.0 and np.array_equal(cost[0], cost[1])
    assert np.sum(cost[0] == RES) == 6
    early = check_schedule(D, gs, box, src, tgt, 0.5, False, rng)
    assert early > 0                                         # near targets in a large free box: channels stop before the box is done
    # a target in the source's voxel only: retired at the first generation
    T = np.ones(gs, bool)
    s = np.ravel_multi_index(tuple(c), gs)
    F, gens, e = navmatrixref.channel_worklist(T, [s], [s], RES, rng, True)
    assert gens == 0 and e == 1 and F[0][tuple(c)] == 0.0
    # without the rule the same channel runs until its list is empty
    F2, gens2, e2 = navmatrixref.channel_worklist(T, [s], [s], RES, rng, True, retire=False)
    assert gens2 > 3 and e2 == 0 and F2[0][tuple(c)] == 0.0


def test_unreachable_blocked_and_outside_points():
    rng = np.random.default_rng(8)
    gs = (20, 18, 12)
    free = np.ones(gs, bool)
    free[10, :, :] = False                                   # a wall: the two halves never meet
    D = np.where(free, 1.0, 0.0).reshape(-1)
    box = ((0, 0, 0), tuple(g - 1 for g in gs))
    src = pos([[3, 4, 5], [15, 9, 2], [10, 3, 3]], rng)      # the last one on the wall: status 1
    tgt = np.concatenate([pos([[4, 4, 5], [16, 9, 2], [10, 8, 8], [0, 0, 0]], rng),
                          ORIGIN + np.array([[-1.0, 0.0, 0.0], [np.nan, np.nan, np.nan]])])
    cost, ss, ts, _ = check_rows(D, gs, box, src, tgt, 0.5, False)
    assert list(ss) == [0, 0, 1] and list(ts) == [0, 0, 1, 0, 2, 2]
    assert cost[0, 1] == np.inf and cost[1, 0] == np.inf and np.isfinite(cost[0, 0])
    assert np.all(np.isnan(cost[2])) and np.all(np.isnan(cost[:, 2])) and np.all(np.isnan(cost[:, 4:]))
    check_schedule(D, gs, box, src, tgt, 0.5, False, rng)    # a channel with an unreachable target runs until its list is empty
    # a box that cuts the grid: points in the grid but outside the box have status 2
    sub = ((0, 0, 0), (9, 17, 11))
    _, ss2, ts2, _ = check_rows(D, gs, sub, src, tgt, 0.5, False)
    assert list(ss2) == [0, 2, 2] and list(ts2) == [0, 2, 2, 0, 2, 2]


@pytest.mark.parametrize("case", range(len(BOUNDARY_CASES)))
def test_source_on_tile_face_or_corner(case):
    """A source connected to the rest of free space only across a tile face or corner: the tiles behind it must be queued."""
    lo, goal, far = BOUNDARY_CASES[case]
    gs, D = boundary_grid()
    box = (lo, tuple(g - 1 for g in gs))
    rng = np.random.default_rng(case)
    src, tgt = pos([goal], rng), pos([far, goal], rng)
    cost, _, _, _ = check_rows(D, gs, box, src, tgt, 0.5, False)
    assert np.isfinite(cost[0, 0])
    check_schedule(D, gs, box, src, tgt, 0.5, False, rng)


def test_passes():
    assert navmatrixref.passes(70, 5, 160 ** 3) == 3
    assert navmatrixref.passes(32, 5, 160 ** 3) == 1
    assert navmatrixref.passes(8, 8, 512 ** 3) == 2           # 4 per pass on the whole 512^3 grid
    assert navmatrixref.passes(5, 0, 100) == 0 and navmatrixref.passes(0, 5, 100) == 0


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("navmask") / "navmask_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "navmask_test.cpp"), "-o", out])
    return out


def test_move_bits_match_navref(exe):
    """fb_nav_move_bits equals navref.move_mask for all 26 directions, on boxes that touch every grid face."""
    rng = np.random.default_rng(13)
    checked = 0
    for gs, box, _ in CASES:
        D = synth(gs, rng)
        for r, unk in ((0.0, False), (2.5 * RES, True)):
            T = navref.traversable(D.reshape(gs)[navref.box_slices(box)], r, unk)
            txt = " ".join(str(x) for x in T.shape) + "\n" + " ".join("1" if t else "0" for t in T.reshape(-1)) + "\n"
            p = subprocess.run([exe], input=txt, capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr
            M = np.array([int(x) for x in p.stdout.split()], np.int64).reshape(T.shape)
            assert np.array_equal((M >> 13) & 1 == 1, T)
            for k, d in enumerate(navref.OFFSETS):
                bit = k if k < 13 else k + 1                  # fb_nav_dir order skips 13 (no move)
                su, _, A = navref.move_mask(T, d)
                want = np.zeros(T.shape, bool)
                want[su] = A
                assert np.array_equal((M >> bit) & 1 == 1, want), (gs, box, d)
                checked += int(want.sum())
    assert checked > 1000
