"""Every schedule of k_x_relax against the sequential reference, on small adversarial maps.

k_x_relax (fiesta_b200/csrc/fb_xrelax.cu) chooses its code paths by list sizes, and at the default thresholds the small maps
of the other GPU tests only reach SMALL generations and the one-warp-per-dependant re-seeding loop.  Two environment
variables, read once per map when it is created (fb_exact_init), move the thresholds so that small maps run every path:

  FIESTA_X_SMALL=n    a generation of more than n entries is BIG: summaries of its targets (x_claim_summaries), round 1
                      through them, commit through SUM; up to n entries it is SMALL: gathers, commit through slotc.
                      Default 32768, at most 65536; 0 makes every generation BIG.
  FIESTA_X_DENSE=n    a later round of a BIG generation whose work list has more than n entries is dense: it refreshes the
                      summaries first (only the targets of last round's flips if these are fewer than nE/4, else it claims
                      every target again), then evaluates through them.  Default 16384; 0 makes every round with work dense.
                      The first later list of at most n entries seeds the device work queue (x_async) instead, which is
                      followed by one refresh of the targets of the last round's flips (F[in]) and the queue's (F[out]).

Whatever the schedule, the result must be the reference's, bit for bit: distance_, closest_obstacle_ (ties included),
occupancy and the expansion count after every update, and the trilinear queries at the end.  Run this file after every
change to k_x_relax.  The reference does not depend on the schedule, so it runs once per scenario and every schedule is
compared with its snapshots.

Run as `python -m tests.test_gpu_xrelax_schedules <scenario>` from the repository root, the file replays one scenario on the
device under the environment it inherits and prints one JSON line (per-update counters and a digest of the final arrays).
The path-coverage tests run it with FIESTA_DEBUG_X=1 (latched once per process) and add up the phase counts of the kernel's
trace on stderr, so that a passing schedule test cannot mean that the forced path never ran.
"""
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests import scenes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X_ENV = ("FIESTA_X_SMALL", "FIESTA_X_DENSE", "FIESTA_X_TWO_SORTS")

SCHEDULES = {
    "default": {},                                                              # SMALL generations on these maps
    "big-queue": {"FIESTA_X_SMALL": "0"},                                       # every generation BIG, the queue from round 2
    # every later round with work dense, until only flips are left (nw == 0, nf > 0): then a queue phase seeded with an
    # empty list
    "dense-then-empty-queue": {"FIESTA_X_SMALL": "0", "FIESTA_X_DENSE": "0"},
    # dense rounds, then the queue: the last dense round's flips (F[in]) are refreshed after it
    "dense-then-queue": {"FIESTA_X_SMALL": "0", "FIESTA_X_DENSE": "64"},
    "mixed": {"FIESTA_X_SMALL": "256", "FIESTA_X_DENSE": "64"},                # SMALL <-> BIG hand-overs within one UpdateESDF
    "all-small": {"FIESTA_X_SMALL": "65536"},                                   # SMALL generations above the default limit
}


# ---------------------------------------------------------------------------------------------------------------------------
# Scenarios: generators over one map (device or reference) that yield (tag, results of the step) after every update; the
# final step is a trilinear query (tag "query").  Everything is seeded, so both sides see the same calls.
def feed(m, vox, occ, global_map=True):
    r = m.SetOccupancyBatchVox(vox, occ)
    u = m.UpdateOccupancy(global_map)
    m.UpdateESDF()
    return r, u


def ones(n):
    return np.ones(n, np.uint8)


def zeros(n):
    return np.zeros(n, np.uint8)


def rand_vox(rng, gs, n):
    return np.stack([rng.integers(0, gs[i], n) for i in range(3)], -1).astype(np.int32)


def interior_query(m, rng, origin, size, res, n=2000):
    lo = np.asarray(origin) + res                              # positions whose 8 trilinear neighbours lie in the grid
    hi = lo + np.asarray(size) - 3 * res
    return m.GetDistWithGradTrilinearBatch(rng.uniform(lo, hi, (n, 3)))


def salt_and_pepper(m):
    """The scene of test_exact_random_insert_delete: 60 % observed in scrambled order, unknown voxels next to everything."""
    rng = np.random.default_rng(21)
    gs = m.grid_size
    allv = scenes.all_voxels(gs)
    sel = allv[rng.random(len(allv)) < 0.6]
    sel = sel[rng.permutation(len(sel))]
    yield "observe", feed(m, sel, (rng.random(len(sel)) < 0.01).astype(np.uint8))
    for r in range(6):
        yield "round %d" % r, feed(m, rand_vox(rng, gs, 1500), (rng.random(1500) < 0.5).astype(np.uint8))
    yield "query", m.GetDistWithGradTrilinearBatch(rng.uniform(-1.9, 1.0, (2000, 3)))


FACES = dict(origin=(-1.0, -0.3, -1.0), res=0.1, size=(2.25, 0.45, 2.05))   # 23 x 5 x 21: a thin y axis, z padded to 24


def faces(m):
    """Obstacles on every face, edge and corner of a grid with a 5-voxel axis: the 129 offsets around almost every entry
    leave the grid, and the +-2 steps cross the thin axis.  10 % of the voxels are never observed."""
    rng = np.random.default_rng(3)
    gs = m.grid_size
    allv = scenes.all_voxels(gs)
    seen = allv[rng.random(len(allv)) < 0.9]
    seen = seen[rng.permutation(len(seen))]
    yield "observe", feed(m, seen, zeros(len(seen)))
    hi = np.array(gs) - 1
    nface = ((allv == 0) | (allv == hi)).sum(1)                 # 1: on a face, 2: on an edge, 3: a corner
    u = rng.random(len(allv))
    obs = allv[(nface == 3) | ((nface == 2) & (u < 0.5)) | ((nface == 1) & (u < 0.12))]
    obs = obs[rng.permutation(len(obs))]
    yield "insert", feed(m, obs, ones(len(obs)))
    yield "delete half", feed(m, obs[::2], zeros(len(obs[::2])))
    shell = allv[((allv <= 1) | (allv >= hi - 1)).any(1)]
    for r in range(2):
        v = shell[rng.integers(0, len(shell), 400)]
        yield "toggle %d" % r, feed(m, v, (rng.random(400) < 0.5).astype(np.uint8))
    yield "query", interior_query(m, rng, **FACES)


LOCAL = dict(origin=(-3.2, -3.2, -1.6), res=0.1, size=(6.4, 6.4, 3.2))


def local_box(r):
    c = np.array([-1.2 + 0.35 * r, -0.9 + 0.3 * r, 0.0])
    return c - np.array([1.3, 1.2, 0.9]), c + np.array([1.3, 1.2, 0.9])


def box_vox(lo, hi):
    """Voxel bounds of SetUpdateRange(lo, hi) on the LOCAL grid (inclusive; fiesta_set_update_range)."""
    o, res = np.asarray(LOCAL["origin"]), LOCAL["res"]
    return np.floor((lo - o) / res).astype(int), np.floor((hi - res / 2 - o) / res).astype(int)


def local_map(m):
    """The sliding local-map box of test_local_map_moving_box_exact (UpdateOccupancy(false)), then a delete of the obstacles
    just inside one face of the box: their dependants on the far side of the face are outside it (x_in_range in the gathers,
    the pushes and the re-seeding)."""
    rng = np.random.default_rng(7)
    allv = scenes.all_voxels(m.grid_size)
    idx = rng.choice(len(allv), 300, replace=False)
    yield "observe", feed(m, allv, zeros(len(allv)))
    yield "obstacles", feed(m, allv[idx], ones(300))
    m.SetParameters(*scenes.PARAMS_DEFAULT)                     # one miss no longer clamps: resets are not skipped
    for r in range(6):
        m.SetUpdateRange(*local_box(r))
        vox = rand_vox(rng, m.grid_size, 6000)
        yield "box %d" % r, feed(m, vox, (rng.random(6000) < 0.4).astype(np.uint8), global_map=False)
    m.SetParameters(*scenes.PARAMS_TOGGLE)                      # one miss deletes
    lo, hi = local_box(5)
    m.SetUpdateRange(lo, hi)
    vlo, vhi = box_vox(lo, hi)
    obs = allv[idx]
    near_face = ((obs >= vlo + 1) & (obs <= vhi - 1)).all(1) & ((obs - vlo <= 3) | (vhi - obs <= 3)).any(1)
    yield "delete at the box face", feed(m, obs[near_face], zeros(int(near_face.sum())), global_map=False)
    yield "query", m.GetDistWithGradTrilinearBatch(rng.uniform(-2.5, 2.5, (1000, 3)) * (1, 1, 0.5))


MASS = dict(origin=(-3.2, -3.2, -3.2), res=0.1, size=(6.4, 6.4, 6.4))        # 64^3


def mass_delete(m):
    """Two parallel walls with holes and sparse random obstacles, fully observed; one update deletes a whole wall, so that
    round 1 of the re-seeding is long enough for one thread per dependant, and the re-seeded values chain through the
    dependants towards the other wall.  Then half of the rest goes, and everything deleted comes back."""
    rng = np.random.default_rng(5)
    allv = scenes.all_voxels(m.grid_size)
    yield "observe", feed(m, allv, zeros(len(allv)))

    def wall(x):
        w = allv[allv[:, 0] == x]
        return w[~((w[:, 1] % 16 < 3) & (w[:, 2] % 16 < 3))]   # 3 x 3 holes every 16 voxels

    A, B = wall(14), wall(46)
    R = allv[(rng.random(len(allv)) < 0.001) & (allv[:, 0] != 14) & (allv[:, 0] != 46)]
    obs = np.concatenate([A, B, R])
    obs = obs[rng.permutation(len(obs))]
    yield "insert", feed(m, obs, ones(len(obs)))
    yield "delete wall", feed(m, A[rng.permutation(len(A))], zeros(len(A)))
    rest = np.concatenate([B, R])
    half = rest[rng.random(len(rest)) < 0.5]
    half = half[rng.permutation(len(half))]
    yield "delete half", feed(m, half, zeros(len(half)))
    back = np.concatenate([A, half])
    back = back[rng.permutation(len(back))]
    yield "re-insert", feed(m, back, ones(len(back)))
    yield "query", interior_query(m, rng, **MASS)


TIES = dict(origin=(-2.35, -2.35, -1.15), res=0.1, size=(4.65, 4.65, 2.25))    # 47 x 47 x 23: mirror planes through voxels


def ties(m):
    """A lattice of obstacles plus random ones mirrored in x and y, all inserted in one batch: many voxels have several
    equidistant candidates, and only the timestamp order decides which one they keep.  Then every other one is deleted and
    put back in reverse order."""
    rng = np.random.default_rng(9)
    gs = m.grid_size
    allv = scenes.all_voxels(gs)
    yield "observe", feed(m, allv, zeros(len(allv)))
    hi = np.array(gs) - 1
    lat = allv[((allv - 2) % 6 == 0).all(1)]
    p = rand_vox(rng, gs, 40)
    mir = np.concatenate([p, np.abs([hi[0], 0, 0] - p), np.abs([0, hi[1], 0] - p), np.abs([hi[0], hi[1], 0] - p)])
    obs = np.unique(np.concatenate([lat, mir]), axis=0).astype(np.int32)
    obs = obs[rng.permutation(len(obs))]
    yield "insert", feed(m, obs, ones(len(obs)))
    yield "delete every other", feed(m, obs[::2], zeros(len(obs[::2])))
    yield "re-insert reversed", feed(m, obs[::2][::-1], ones(len(obs[::2])))
    yield "query", interior_query(m, rng, **TIES)


RAYS = dict(origin=(-6.4, -6.4, -3.2), res=0.1, size=(12.8, 12.8, 6.4))


def raycast_frames(m):
    """Three depth frames of test_exact_raycast_frames: a realistic, partially observed map."""
    sc = scenes.Scene((5.0, 5.0, 2.5), 20, 5, seed=2)
    for f, (p, yaw) in enumerate(scenes.pose_walk(3, seed=3)):
        pts, T = scenes.depth_frame(sc, p, yaw, width=160, height=120, scale=0.25)
        n = m.RaycastFrame(pts, T, 0.5, 5.0)
        u = m.UpdateOccupancy(True)
        m.UpdateESDF()
        yield "frame %d" % f, (n, u)
        sc.step()
    yield "query", interior_query(m, np.random.default_rng(4), **RAYS)


SALT = dict(origin=(-2.0, -2.0, -2.0), res=0.1, size=(3.95, 3.95, 3.15))      # 40 x 40 x 32

# name -> (geometry, parameters, body)
SCENARIOS = {
    "salt-and-pepper": (SALT, scenes.PARAMS_TOGGLE, salt_and_pepper),
    "faces": (FACES, scenes.PARAMS_TOGGLE, faces),
    "local-box": (LOCAL, scenes.PARAMS_TOGGLE, local_map),
    "mass-delete": (MASS, scenes.PARAMS_TOGGLE, mass_delete),
    "ties": (TIES, scenes.PARAMS_TOGGLE, ties),
    "raycast-frames": (RAYS, scenes.PARAMS_DEFAULT, raycast_frames),
}
LARGE_GENERATIONS = ("mass-delete", "local-box")               # generations above 32768 entries: worth the all-small schedule


def replay(name, make):
    """Runs scenario `name` on a map made by make(origin, res, size): yields (tag, results, map) after every step."""
    geo, params, body = SCENARIOS[name]
    m = make(geo["origin"], geo["res"], geo["size"])
    m.SetParameters(*params)
    for tag, res in body(m):
        yield tag, res, m


def state(m):
    s = m.stats()
    return dict(dist=m.export_distance(), cobs=m.export_closest_obstacle(), occ=m.export_occupancy(),
                counts=(s["inserts"], s["deletes"], s["expansions"]))


def digest(st):
    h = hashlib.sha256()
    for k in ("dist", "cobs", "occ"):
        h.update(np.ascontiguousarray(st[k]).tobytes())
    return h.hexdigest()


def same(a, b):
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.shape == b.shape and np.array_equal(a, b)
    return a == b


def mismatch(got, want, gs):
    """Counts of the mismatches between two states, with the first differing voxel (none: all counts 0)."""
    dm = got["dist"] != want["dist"]
    cm = (got["cobs"] != want["cobs"]).any(axis=1)
    om = got["occ"] != want["occ"]
    r = dict(dist=int(dm.sum()), cobs_tie=int((cm & ~dm).sum()), cobs_nontie=int((cm & dm).sum()), occ=int(om.sum()))
    bad = np.flatnonzero(dm | cm | om)
    if len(bad):
        v = int(bad[0])
        r["first"] = dict(voxel=tuple(int(c) for c in np.unravel_index(v, gs)), dist=(got["dist"][v], want["dist"][v]),
                          cobs=(tuple(got["cobs"][v]), tuple(want["cobs"][v])), occ=(got["occ"][v], want["occ"][v]))
    return r


# ---------------------------------------------------------------------------------------------------------------------------
# The reference, once per scenario
def l_occ(params):
    return float(np.log(params[4] / (1 - params[4])))


def scenario_facts(name, steps, gs):
    """Checks that a scenario reaches the case it was written for (on the reference's states)."""
    if name == "local-box":
        prev, cur = steps[-3][2], steps[-2][2]                  # the state before and after the delete at the box face
        lo = l_occ(scenes.PARAMS_TOGGLE)
        gone = np.flatnonzero((prev["occ"] > lo) & ~(cur["occ"] > lo))
        assert len(gone) > 0, "no obstacle deleted at the box face"
        deps = np.isin(np.ravel_multi_index(tuple(prev["cobs"].T.clip(0)), gs), gone) & (prev["cobs"][:, 0] >= 0)
        vlo, vhi = box_vox(*local_box(5))
        xyz = np.stack(np.unravel_index(np.flatnonzero(deps), gs), -1)
        outside = int((~((xyz >= vlo) & (xyz <= vhi)).all(1)).sum())
        assert 0 < outside < len(xyz), ("dependants of the deleted obstacles outside the update box", outside, len(xyz))
    if name == "ties":
        from scipy.spatial import cKDTree
        st = steps[1][2]                                        # after the insert
        allv = scenes.all_voxels(gs)
        obs = allv[st["occ"] > l_occ(scenes.PARAMS_TOGGLE)]
        d, _ = cKDTree(obs).query(allv, k=2)
        tied = np.rint(d[:, 0] ** 2) == np.rint(d[:, 1] ** 2)
        assert tied.mean() > 0.2, ("voxels with two equidistant nearest obstacles", tied.mean())


@pytest.fixture(scope="module")
def reference(oracle_built):
    cache = {}

    def get(name):
        if name not in cache:
            steps = []
            for tag, res, m in replay(name, oracle_built.OracleMap):
                steps.append((tag, res, None if tag == "query" else state(m)))
            scenario_facts(name, steps, m.grid_size)
            cache[name] = (steps, m.grid_size)
        return cache[name]
    return get


def set_schedule(monkeypatch, env):
    for k in X_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def device_map(origin, res, size):
    import fiesta_b200
    return fiesta_b200.ESDFMap(origin, res, size, mode="exact")


def multiprocessors():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def check_against_reference(reference, scenario):
    steps, gs = reference(scenario)
    got = list(replay_checked(scenario, steps, gs))
    assert len(got) == len(steps)
    return got


def replay_checked(scenario, steps, gs):
    """Replays the scenario on the device and compares every step with the reference's snapshot; yields the device stats."""
    it = iter(steps)
    for tag, res, m in replay(scenario, device_map):
        wtag, wres, wst = next(it)
        assert tag == wtag
        assert same(res, wres), (tag, "step results differ from the reference's")
        if wst is not None:
            st = state(m)
            r = mismatch(st, wst, gs)
            assert r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0 and r["occ"] == 0, (tag, r)
            assert st["counts"] == wst["counts"], (tag, "inserts, deletes, expansions", st["counts"], wst["counts"])
        yield tag, m.stats()


MATRIX = [pytest.param(sc, sh, id="%s:%s" % (sc, sh)) for sc in SCENARIOS for sh in SCHEDULES
          if sh != "all-small" or sc in LARGE_GENERATIONS]


@pytest.mark.parametrize("scenario,schedule", MATRIX)
def test_schedule_matches_reference(reference, scenario, schedule, monkeypatch):
    set_schedule(monkeypatch, SCHEDULES[schedule])
    got = dict(check_against_reference(reference, scenario))
    if scenario == "mass-delete":
        # round 1 of the re-seeding runs one thread per dependant only above 2 warps per warp of the grid
        assert got["delete wall"]["voxels_reset"] > 2 * 32 * multiprocessors(), got["delete wall"]


def test_mass_delete_two_sorts(reference, monkeypatch):
    """The dependant order through the two-key fallback (rank and relink clock no longer fit one 64-bit sort key)."""
    set_schedule(monkeypatch, dict(SCHEDULES["big-queue"], FIESTA_X_TWO_SORTS="1"))
    got = dict(check_against_reference(reference, "mass-delete"))
    assert got["delete wall"]["voxels_reset"] > 2 * 32 * multiprocessors()


# ---------------------------------------------------------------------------------------------------------------------------
# Proof that each forced path ran: the kernel's own trace (FIESTA_DEBUG_X) in a child process
PHASES = re.compile(r"phases \(us, count\):(.*)$", re.M)
PHASE = re.compile(r"(\S+) \d+/(\d+)")
GENS = re.compile(r"^\[x\] gens .*\|(.*)$", re.M)

# schedule -> (scenario, required phase counts); the names are the trace's categories
COVERAGE = {
    "default": ("salt-and-pepper", {"round1": 0}),             # the gap this file closes: no BIG generation by default
    "big-queue": ("salt-and-pepper", {"round1": ">0", "async": ">0", "s.round1": 0, "rounds": 0}),
    "dense-then-empty-queue": ("salt-and-pepper", {"dense": ">0", "async": ">0"}),   # with DENSE=0 the queue only runs when nw == 0
    "dense-then-queue": ("salt-and-pepper", {"dense": ">0", "async": ">0", "rounds": 0}),
    "mixed": ("salt-and-pepper", {"round1": ">0", "s.round1": ">0"}),
    "all-small": ("mass-delete", {"s.round1": ">0"}),           # and generations of 32769..65536 entries (below)
}


def traced_run(scenario, env):
    e = {k: v for k, v in os.environ.items() if k not in X_ENV}
    e.update(env)
    e["FIESTA_DEBUG_X"] = "1"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.test_gpu_xrelax_schedules", scenario]
    p = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    counts = {}
    for line in PHASES.findall(p.stderr):
        for name, n in PHASE.findall(line):
            counts[name] = counts.get(name, 0) + int(n)
    gens = [int(g.split("/")[0]) for line in GENS.findall(p.stderr) for g in line.split()]
    return json.loads(p.stdout.strip().splitlines()[-1]), counts, gens


@pytest.mark.parametrize("schedule", list(COVERAGE))
def test_schedule_takes_its_path(reference, schedule):
    scenario, need = COVERAGE[schedule]
    out, counts, gens = traced_run(scenario, SCHEDULES[schedule])
    assert counts, "no FIESTA_DEBUG_X trace on stderr"
    for name, want in need.items():
        n = counts.get(name, 0)
        assert (n > 0) if want == ">0" else (n == want), (schedule, name, n, counts)
    # the trace adds synchronisations; the result stays the reference's
    steps, gs = reference(scenario)
    assert out["counts"] == [list(st["counts"]) for _, _, st in steps if st is not None], (schedule, out["counts"])
    assert out["digest"] == digest(steps[-2][2])
    if schedule == "all-small":                                 # SMALL generations above the default limit: slotc up to 2^21
        assert any(32768 < n <= 65536 for n in gens), sorted(gens)[-4:]


def main(scenario):
    counts, last = [], None
    for tag, res, m in replay(scenario, device_map):
        if tag != "query":
            last = state(m)
            counts.append(list(last["counts"]))
    print(json.dumps(dict(scenario=scenario, counts=counts, digest=digest(last))))


if __name__ == "__main__":
    main(sys.argv[1])
