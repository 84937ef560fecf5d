"""CPU: the cost-to-go field's definition (tests/navref.py) and the path rule of fiesta_b200/csrc/fb_nav.h.

The GPU tests compare the device field with scipy's Dijkstra bit for bit.  That is only sound because the least fixpoint of
D(v) = min fl(D(u) + w) does not depend on the order relaxations run in; these tests check that claim against Gauss-Seidel sweeps in
random direction orders, check the no-corner-cutting rule, that folding the weights along an extracted path reproduces D(start)
exactly, and that the header's path rule (compiled with g++) gives navref's paths voxel for voxel.  They also run the device
solver's tile work-list rule (navref.tile_worklist) on the CPU: it must reach the same field, in particular when a goal is connected
to the rest of free space only across a tile face, edge or corner."""
import os
import subprocess

import numpy as np
import pytest

from tests import navref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.1


def synth(gs, rng, p_unknown=0.1, p_unreached=0.05):
    """An export_distance()-like array: never observed (-10000), unreached (+10000), and distances that are multiples of sqrt of
    integers times RES like real records, many of them small enough to block."""
    n = int(np.prod(gs))
    d = np.sqrt(rng.integers(0, 40, n).astype(np.float64)) * RES
    kind = rng.random(n)
    return np.where(kind < p_unknown, -10000.0, np.where(kind < p_unknown + p_unreached, 10000.0, d))


CASES = [  # grid, box (lo, hi), goals
    ((24, 20, 17), ((0, 0, 0), (23, 19, 16)), 5),
    ((13, 11, 9), ((2, 1, 0), (12, 10, 8)), 3),
    ((10, 19, 12), ((4, 0, 0), (4, 18, 11)), 3),       # 1 voxel thick in x
    ((17, 9, 21), ((0, 3, 2), (16, 3, 20)), 4),        # 1 voxel thick in y
    ((9, 30, 7), ((1, 2, 3), (8, 27, 3)), 2),          # 1 voxel thick in z
]


def goals_in(box, k, rng):
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    return np.stack([rng.integers(lo[i], hi[i] + 1, k) for i in range(3)], -1)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_dijkstra_equals_gauss_seidel_in_any_order(case):
    gs, box, ng = CASES[case]
    rng = np.random.default_rng(case)
    D = synth(gs, rng)
    reached = 0
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            goals = goals_in(box, ng, rng)
            F = navref.field(D, gs, box, goals, r, unk, RES)
            T = navref.traversable(D.reshape(gs)[navref.box_slices(box)], r, unk)
            assert np.array_equal(F < 0, ~T)
            gi = navref.goal_indices(T, box, goals)
            for seed in range(2):
                assert np.array_equal(F, navref.sweep(T, gi, RES, np.random.default_rng(seed))), (r, unk, seed)
            reached += int(np.isfinite(F[F >= 0]).sum())
    assert reached > 0


def test_diagonal_gap_is_impassable():
    res = 0.5
    T = np.zeros((2, 2, 1), bool)
    T[0, 0, 0] = T[1, 1, 0] = True                       # two diagonal obstacles between them
    D = np.where(T, 1.0, 0.0).reshape(-1)
    F = navref.field(D, (2, 2, 1), ((0, 0, 0), (1, 1, 0)), [(0, 0, 0)], 0.5, False, res)
    assert F[0, 0, 0] == 0 and F[1, 1, 0] == np.inf
    D3 = np.zeros(8)
    D3[[0, 7]] = 1.0                                     # 3-D: only two opposite corners of a 2x2x2 block are free
    F3 = navref.field(D3, (2, 2, 2), ((0, 0, 0), (1, 1, 1)), [(0, 0, 0)], 0.5, False, res)
    assert F3[1, 1, 1] == np.inf
    F4 = navref.field(np.ones(8), (2, 2, 2), ((0, 0, 0), (1, 1, 1)), [(0, 0, 0)], 0.5, False, res)
    assert F4[1, 1, 1] == res * np.sqrt(3.0) and F4[1, 1, 0] == res * np.sqrt(2.0)
    assert F4[0, 0, 1] == res


@pytest.mark.parametrize("case", range(len(CASES)))
def test_tile_worklist_equals_dijkstra(case):
    gs, box, ng = CASES[case]
    rng = np.random.default_rng(20 + case)
    D = synth(gs, rng)
    for r in (0.0, 2.5 * RES):
        for unk in (False, True):
            goals = goals_in(box, ng, rng)
            F = navref.field(D, gs, box, goals, r, unk, RES)
            T = navref.traversable(D.reshape(gs)[navref.box_slices(box)], r, unk)
            gi = navref.goal_indices(T, box, goals)
            for fresh in (True, False):
                got, _ = navref.tile_worklist(T, gi, RES, rng, fresh)
                assert np.array_equal(got, F), (r, unk, fresh)


def boundary_grid():
    """24 x 24 x 16 voxels, free only in (a) a 1-voxel corridor along x at (y, z) = (3, 3) and (b) the 2x2x2 block {7, 8}^3 plus a
    corridor along x at (y, z) = (7, 7), x = 0..7.  A goal at (8, 3, 3) lies on a tile face and (8, 8, 8) on a tile corner: the
    goal voxel is the only free voxel of its tile that touches the tiles behind it."""
    gs = (24, 24, 16)
    free = np.zeros(gs, bool)
    free[:, 3, 3] = True
    free[7:9, 7:9, 7:9] = True
    free[0:8, 7, 7] = True
    return gs, np.where(free, 1.0, 0.0).reshape(-1)


# (box lower corner, goal, a voxel that the goal reaches only through the tile boundary), grid coordinates; the box runs to the
# grid's upper corner, so its tiles start at the box corner
BOUNDARY_CASES = [((0, 0, 0), (8, 3, 3), (0, 3, 3)),       # goal on a tile face
                  ((4, 0, 0), (12, 3, 3), (4, 3, 3)),      # the same in box-local tiles
                  ((0, 0, 0), (8, 8, 8), (0, 7, 7))]       # goal on a tile corner, connected by a 3-D diagonal move only


@pytest.mark.parametrize("case", range(len(BOUNDARY_CASES)))
def test_goal_on_tile_face_or_corner(case):
    """The goal's own tile has no other voxel that improves next to the tiles across the goal's face or corner, so those tiles must
    be queued when the goal is placed."""
    lo, goal, far = BOUNDARY_CASES[case]
    gs, D = boundary_grid()
    box = (lo, tuple(g - 1 for g in gs))
    T = navref.traversable(D.reshape(gs)[navref.box_slices(box)], 0.5, False)
    F = navref.field(D, gs, box, [goal], 0.5, False, RES)
    assert np.isfinite(F[tuple(np.asarray(far) - np.asarray(lo))])
    gi = navref.goal_indices(T, box, [goal])
    for fresh in (True, False):
        got, _ = navref.tile_worklist(T, gi, RES, np.random.default_rng(1), fresh)
        assert np.array_equal(got, F), fresh


def fields(rng):
    out = []
    for gs, box, ng in CASES:
        D = synth(gs, rng, p_unknown=0.05, p_unreached=0.05)
        for r in (0.0, 4.5 * RES):                    # the larger clearance blocks half the voxels: unconnected parts
            out.append((box, navref.field(D, gs, box, goals_in(box, ng, rng), r, False, RES)))
    return out


def all_starts(F, k, rng):
    v = np.stack(np.unravel_index(np.arange(F.size), F.shape), -1)
    return v[rng.choice(len(v), min(k, len(v)), replace=False)]


def test_paths_fold_to_the_field():
    rng = np.random.default_rng(11)
    seen = set()
    for box, F in fields(rng):
        starts = all_starts(F, 400, rng)
        for max_len in (1, 6, 200):
            st, ln, cost, vox = navref.paths(F, box, RES, starts, np.ones(len(starts), bool), max_len)
            seen |= set(int(s) for s in st)
            for i in np.nonzero(st == 0)[0]:
                p = vox[i, :ln[i]]
                assert navref.fold(F, box, RES, p) == cost[i] == F[tuple(starts[i])]
                assert F[tuple(p[-1] - np.asarray(box[0]))] == 0
                assert np.all(vox[i, ln[i]:] == -1)
            assert np.all(ln[st == 3] == max_len)
            assert np.all(np.isnan(cost[st == 2])) and np.all(cost[st == 1] == np.inf)
    assert seen == {0, 1, 2, 3}, seen


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("nav") / "nav_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "nav_test.cpp"), "-o", out])
    return out


def run_header(exe, F, box, starts, max_len):
    w = navref.weights(RES)
    txt = [" ".join(str(x) for x in list(F.shape) + list(box[0])), " ".join(float(x).hex() for x in w),
           " ".join(float(x).hex() for x in F.reshape(-1)), "%d %d" % (len(starts), max_len)]
    txt += ["%d %d %d" % tuple(s) for s in starts]
    p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    lines = iter(p.stdout.splitlines())
    out = []
    for _ in starts:
        s, n, c = next(lines).split()
        out.append((int(s), int(n), float.fromhex(c), [tuple(int(x) for x in next(lines).split()) for _ in range(int(n))]))
    return out


def test_header_path_rule_matches_navref(exe):
    rng = np.random.default_rng(12)
    count = 0
    for box, F in fields(rng):
        starts = all_starts(F, 300, rng)
        for max_len in (1, 5, 300):
            want = navref.paths(F, box, RES, starts, np.ones(len(starts), bool), max_len)
            got = run_header(exe, F, box, starts, max_len)
            for i, (s, n, c, p) in enumerate(got):
                assert s == want[0][i] and n == want[1][i], (i, s, n, want[0][i], want[1][i])
                assert np.array_equal(np.float64(c), want[2][i], equal_nan=True)
                assert p == [tuple(x) for x in want[3][i, :n]]
                count += n
    assert count > 10000
