"""CPU: the cost-to-go field update (fiesta_nav_update, DESIGN.md §3.11) in its numpy model (tests/navupdref.py).

Repairing a field computed on old records -- withdraw the voxels whose finite cost lost its support, restart the re-relaxation from
the repaired start state on the seed tiles only -- must give navref.field on the new records bit for bit: on random record pairs
of test_nav_oracle.py's case shapes (1-voxel-thick boxes, several goals, three clearances, the unknown flag on and off), chained
over several updates, and on targeted cases: goals that become blocked or free, a maze door that opens and closes, a freed voxel
that opens a diagonal gap, changes on tile faces and corners and on the box faces, and no change at all.  Negative controls show
that the withdrawal rule and the seeding rule are needed, and the header's support predicate (compiled with g++) must agree with
the model on every voxel and move."""
import os
import subprocess

import numpy as np
import pytest

from tests import navref, navupdref
from tests.test_nav_oracle import CASES, RES, goals_in, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def perturb(D, rng, p):
    """New records: a fraction p of the voxels drawn again (obstacles appear and vanish, distances shift)."""
    return np.where(rng.random(D.size) < p, synth((D.size,), rng), D)


def check(D_old, D_new, gs, box, goals, r, unk, rng, fresh=True, F_old=None):
    """Update the field of D_old (or F_old) to D_new in the model; compare with the field computed on D_new.  Returns the stats."""
    F_old = navref.field(D_old, gs, box, goals, r, unk, RES) if F_old is None else F_old
    Tnew = navref.traversable(D_new.reshape(gs)[navref.box_slices(box)], r, unk)
    want = navref.field(D_new, gs, box, goals, r, unk, RES)
    got, st = navupdref.update(F_old, Tnew, navref.goal_indices(Tnew, box, goals), RES, rng, fresh)
    assert np.array_equal(got, want), (box, r, unk, int(np.sum(got != want)))
    assert st["improvable_outside_seeds"] == 0
    return got, st


@pytest.mark.parametrize("case", range(len(CASES)))
def test_update_equals_fresh_field_on_random_record_pairs(case):
    gs, box, ng = CASES[case]
    rng = np.random.default_rng(40 + case)
    totals = dict(withdrawn=0, became_blocked=0, became_free=0)
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            goals = goals_in(box, ng, rng)
            D = synth(gs, rng)
            F = None
            for step, p in enumerate((0.02, 0.1, 0.3)):                 # chained updates, each from the last repaired field
                D2 = perturb(D, rng, p)
                F, st = check(D, D2, gs, box, goals, r, unk, rng, fresh=step != 1, F_old=F)
                for k in totals:
                    totals[k] += st[k]
                D = D2
    assert all(v > 0 for v in totals.values()), totals


def free_grid(gs):
    return np.ones(gs, bool)


def records(free):
    return np.where(free, 1.0, 0.0).reshape(-1)          # clearance 0.5: 1.0 traversable, 0.0 blocked


def run_pair(free_old, free_new, goals, box=None, rng_seed=0):
    gs = free_old.shape
    box = ((0, 0, 0), tuple(g - 1 for g in gs)) if box is None else box
    rng = np.random.default_rng(rng_seed)
    out = []
    for fresh in (True, False):
        out.append(check(records(free_old), records(free_new), gs, box, goals, 0.5, False, rng, fresh)[1])
    return out[0]


def test_goal_becomes_blocked_then_free():
    free = free_grid((20, 18, 9))
    goals = [(3, 4, 4), (15, 12, 2)]
    blocked = free.copy()
    blocked[3, 4, 4] = False
    st = run_pair(free, blocked, goals)
    assert st["became_blocked"] == 1 and st["withdrawn"] > 0
    st = run_pair(blocked, free, goals)
    assert st["became_free"] == 1 and st["goals_new"] == 1


def maze(gs=(40, 31, 3)):
    """Serpentine walls along x on every third y row, a 2-voxel gap at alternating ends (test_gpu_nav.py's maze, smaller)."""
    free = np.ones(gs, bool)
    for i, y in enumerate(range(2, gs[1] - 1, 3)):
        if i % 2 == 0:
            free[0:gs[0] - 2, y, :] = False
        else:
            free[2:, y, :] = False
    return free


def test_maze_door_opens_and_closes():
    closed = maze()
    opened = closed.copy()
    opened[20, 8, :] = True                              # a door in the middle of the third wall (y = 8), through the height
    goals = [(1, 0, 1)]
    st = run_pair(closed, opened, goals)
    assert st["became_free"] == 3 and st["withdrawn"] == 0
    st = run_pair(opened, closed, goals)
    assert st["became_blocked"] == 3 and st["withdrawn"] > 100     # everything beyond the door had its shortest path through it


def test_single_freed_voxel_opens_a_diagonal_gap():
    """Two free voxels touch only diagonally, with both voxels of the 2x2 between them blocked: no move.  Freeing one of those
    voxels allows the diagonal move between the two unchanged voxels, not only moves through the freed one."""
    gs = (17, 17, 1)
    free = np.zeros(gs, bool)
    free[:8, 7, 0] = True                                # a corridor ending at (7, 7)
    free[8, 8:, 0] = True                                # another starting at (8, 8), across the tile corner (8, 8)
    new = free.copy()
    new[8, 7, 0] = True
    goals = [(0, 7, 0)]
    F_old = navref.field(records(free), gs, ((0, 0, 0), (16, 16, 0)), goals, 0.5, False, RES)
    assert F_old[8, 16, 0] == np.inf
    st = run_pair(free, new, goals)
    assert st["became_free"] == 1 and st["reached"] > 8


@pytest.mark.parametrize("where", ["face", "edge", "corner"])
def test_changes_on_tile_faces_and_corners(where):
    gs = (24, 24, 16)
    rng = np.random.default_rng(3)
    base = rng.random(gs) > 0.25
    v = {"face": (8, 3, 4), "edge": (8, 8, 5), "corner": (8, 8, 8)}[where]
    for dv in itertools_product3():
        w = tuple(v[k] + dv[k] for k in range(3))
        if all(0 <= w[k] < gs[k] for k in range(3)):
            new = base.copy()
            new[w] = not base[w]
            run_pair(base, new, [(1, 1, 1), (20, 20, 12)], rng_seed=sum(w))
    block = base.copy()
    block[7:9, 7:9, 7:9] = False                          # a 2x2x2 block around the tile corner appears, then vanishes
    run_pair(base, block, [(1, 1, 1)])
    run_pair(block, base, [(1, 1, 1)])


def itertools_product3():
    return [(a, b, c) for a in (-1, 0) for b in (-1, 0) for c in (-1, 0)]


def test_changes_on_box_faces():
    gs = (22, 19, 13)
    rng = np.random.default_rng(8)
    free = rng.random(gs) > 0.2
    for box in (((0, 0, 0), (21, 18, 12)), ((3, 2, 1), (17, 15, 10))):
        lo, hi = box
        for axis in range(3):
            for side in (lo[axis], hi[axis]):
                new = free.copy()
                sl = [slice(lo[k], hi[k] + 1) for k in range(3)]
                sl[axis] = slice(side, side + 1)
                face = new[tuple(sl)]
                face ^= rng.random(face.shape) < 0.3
                new[tuple(sl)] = face
                g = [tuple(lo), tuple((np.asarray(lo) + np.asarray(hi)) // 2)]
                run_pair(free, new, g, box=box)


def test_no_change_does_no_relaxation():
    gs, box, ng = CASES[0]
    rng = np.random.default_rng(5)
    D = synth(gs, rng)
    goals = goals_in(box, ng, rng)
    _, st = check(D, D, gs, box, goals, RES, False, rng)
    assert st == dict(st, became_blocked=0, became_free=0, withdrawn=0, goals_new=0, seed_tiles=0, generations=0, tile_visits=0)


def control_cases():
    """Record pairs of the random and targeted kinds, for the negative controls."""
    out = []
    rng = np.random.default_rng(77)
    for gs, box, ng in CASES[:2]:
        D = synth(gs, rng)
        out.append((D, perturb(D, rng, 0.1), gs, box, goals_in(box, ng, rng), RES))
    closed = maze()
    opened = closed.copy()
    opened[20, 8, :] = True
    full = ((0, 0, 0), tuple(g - 1 for g in closed.shape))
    out.append((records(opened), records(closed), closed.shape, full, [(1, 0, 1)], 0.5))
    gs = (17, 17, 1)
    free = np.zeros(gs, bool)
    free[:8, 7, 0] = True
    free[8, 8:, 0] = True
    new = free.copy()
    new[8, 7, 0] = True
    out.append((records(free), records(new), gs, ((0, 0, 0), (16, 16, 0)), [(0, 7, 0)], 0.5))
    return out


def run_variant(variant):
    wrong = outside = 0
    for D, D2, gs, box, goals, r in control_cases():
        F_old = navref.field(D, gs, box, goals, r, False, RES)
        Tnew = navref.traversable(D2.reshape(gs)[navref.box_slices(box)], r, False)
        want = navref.field(D2, gs, box, goals, r, False, RES)
        got, st = navupdref.update(F_old, Tnew, navref.goal_indices(Tnew, box, goals), RES, np.random.default_rng(1), True, variant)
        wrong += not np.array_equal(got, want)
        outside += st["improvable_outside_seeds"] > 0
    return wrong, outside


def test_negative_controls():
    assert run_variant(None) == (0, 0)
    # withdrawing only the newly blocked voxels keeps costs whose paths no longer exist: fields come out too low
    wrong, _ = run_variant("blocked_only")
    assert wrong > 0
    # seeding only a freed voxel's own tile leaves voxels outside every seed tile that can improve in the start state (the
    # diagonal gap), so k_nav_relax's invariant does not hold at generation 0.  (The fields still come out right here: the freed
    # voxel improves and queues the tiles across its faces.  The rule is kept because the correctness argument needs it.)
    _, outside = run_variant("no_free_neighbours")
    assert outside > 0


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("navu") / "navupdate_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "cpp", "navupdate_test.cpp"), "-o", out])
    return out


def test_header_support_predicate_matches_model(exe):
    rng = np.random.default_rng(13)
    count = 0
    for gs, box, ng in CASES:
        D = synth(gs, rng, p_unknown=0.05, p_unreached=0.05)
        for r in (0.0, 2.5 * RES):
            F = navref.field(D, gs, box, goals_in(box, ng, rng), r, False, RES)
            w = navref.weights(RES)
            txt = [" ".join(str(x) for x in F.shape), " ".join(float(x).hex() for x in w), " ".join(float(x).hex() for x in F.reshape(-1))]
            p = subprocess.run([exe], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr
            got = np.array([int(x) for x in p.stdout.split()], np.int64).reshape(F.shape)
            S = navupdref.supports(F, RES)
            want = np.zeros(F.shape, np.int64)
            for k in range(26):
                want |= S[k].astype(np.int64) << (k if k < 13 else k + 1)
            assert np.array_equal(got, want), int(np.sum(got != want))
            count += int(S.sum())
    assert count > 1000
