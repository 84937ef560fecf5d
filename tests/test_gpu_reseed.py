"""The re-seeding of the dependants of deleted obstacles (k_x_reseed, fiesta_b200/csrc/fb_xrelax.cu) against the sequential
reference, on maps built to reach each of its stages.

k_x_reseed classifies every dependant (A), closes validity over the dependant order in rounds (B), chooses a parent (C) and
resolves the parent chains by pointer jumping (D).  The maps here give it
  * dependants with no static source several rounds deep (the inside of a deleted solid block and the free space around it),
  * a delete that leaves no obstacle at all, so that every dependant ends INF,
  * a parent chain of more than 512 dependants (a corridor of observed voxels that snakes through unknown space), so that
    D needs 10 passes or more,
  * dependants partly outside a local update box,
  * an adversarial dependant order: the block deleted from the inside out, so that the inner dependants come first.
distance_, closest_obstacle_ (ties included), occupancy and the expansion count must be the reference's after every update.
A child process with FIESTA_DEBUG_X=1 shows from the kernel's trace that B ran several rounds and D ten passes or more.

Run as `python -m tests.test_gpu_reseed <scenario>` from the repository root, the file replays one scenario on the device
and prints one JSON line (per-update counters and a digest of the final arrays).
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests import scenes
from tests.test_gpu_xrelax_schedules import X_ENV, device_map, digest, feed, l_occ, mismatch, ones, same, state, zeros

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BLOCK = dict(origin=(-2.0, -2.0, -2.0), res=0.1, size=(4.0, 4.0, 4.0))          # 40^3
BOX_LO, BOX_HI = (-2.0, -2.0, -2.0), (-0.45, 1.95, 1.95)                      # x voxels 0..14: cuts the block at x = 14


def block(m):
    """A solid 14^3 block and a wall, fully observed.  The block goes outside-in (favourable order: deep closure), comes
    back, goes inside-out (the inner dependants first), comes back, goes under a local update box whose face cuts it, and
    finally the block and the wall go together, leaving no obstacle."""
    rng = np.random.default_rng(11)
    allv = scenes.all_voxels(m.grid_size)
    yield "observe", feed(m, allv, zeros(len(allv)))
    blk = allv[((allv >= [6, 13, 13]) & (allv <= [19, 26, 26])).all(1)]
    wall = allv[allv[:, 0] == 36]
    depth = np.abs(blk - [12.5, 19.5, 19.5]).max(1)
    out_in, in_out = blk[np.argsort(-depth, kind="stable")], blk[np.argsort(depth, kind="stable")]
    both = np.concatenate([blk, wall])
    yield "insert", feed(m, both[rng.permutation(len(both))], ones(len(both)))
    yield "delete outside-in", feed(m, out_in, zeros(len(blk)))
    yield "re-insert", feed(m, blk, ones(len(blk)))
    yield "delete inside-out", feed(m, in_out, zeros(len(blk)))
    yield "re-insert 2", feed(m, blk[::-1], ones(len(blk)))
    m.SetUpdateRange(BOX_LO, BOX_HI)
    yield "delete in a box", feed(m, out_in, zeros(len(blk)), global_map=False)
    m.SetUpdateRange((-2.0, -2.0, -2.0), (2.0, 2.0, 2.0))
    yield "re-insert 3", feed(m, blk, ones(len(blk)))
    yield "delete everything", feed(m, both, zeros(len(both)))
    yield "query", m.GetDistWithGradTrilinearBatch(rng.uniform(-1.85, 1.75, (1000, 3)))


SNAKE = dict(origin=(0.0, 0.0, 0.0), res=0.1, size=(12.8, 12.8, 0.1))          # 128 x 128 x 1


def snake(m):
    """Rows y = 0, 3, ..., 126 of a 128 x 128 plane, joined at alternate ends, are the only observed voxels (the +-2 steps
    cannot cross the two unknown rows between them): one corridor of about 5 600 voxels.  A at its start and B next to row
    126 split it at y = 62.5, so A's dependants form one chain of about 2 700 voxels along the corridor, linked in the order
    the wavefront reached them.  A goes, then B."""
    gs = m.grid_size
    path = []
    for r, y in enumerate(range(0, gs[1], 3)):
        xs = range(gs[0]) if r % 2 == 0 else range(gs[0] - 1, -1, -1)
        path += [(x, y, 0) for x in xs]
        if y + 3 < gs[1]:
            xe = gs[0] - 1 if r % 2 == 0 else 0
            path += [(xe, y + 1, 0), (xe, y + 2, 0)]
    path = np.array(path, np.int32)
    a, b = np.array([[0, 0, 0]], np.int32), np.array([[0, 125, 0]], np.int32)
    yield "observe", feed(m, path, zeros(len(path)))
    yield "insert", feed(m, np.concatenate([a, b]), ones(2))
    yield "delete A", feed(m, a, zeros(1))
    yield "delete B", feed(m, b, zeros(1))
    yield "query", m.GetDistWithGradTrilinearBatch(np.random.default_rng(2).uniform(0.05, 12.6, (1000, 3)) * (1, 1, 0))


SCENARIOS = {"block": (BLOCK, scenes.PARAMS_TOGGLE, block), "snake": (SNAKE, scenes.PARAMS_TOGGLE, snake)}


def replay(name, make):
    geo, params, body = SCENARIOS[name]
    m = make(geo["origin"], geo["res"], geo["size"])
    m.SetParameters(*params)
    for tag, res in body(m):
        yield tag, res, m


def dependants(prev, cur, gs):
    """Voxels whose closest obstacle was deleted between two reference states (flat indices)."""
    lo = l_occ(scenes.PARAMS_TOGGLE)
    gone = np.flatnonzero((prev["occ"] > lo) & ~(cur["occ"] > lo))
    return np.flatnonzero(np.isin(np.ravel_multi_index(tuple(prev["cobs"].T.clip(0)), gs), gone) & (prev["cobs"][:, 0] >= 0))


def scenario_facts(name, steps, gs):
    """Checks on the reference's states that each scenario reaches the case it was written for."""
    st = {tag: s for tag, _, s in steps}
    lo = l_occ(scenes.PARAMS_TOGGLE)
    if name == "block":
        assert not (st["delete everything"]["occ"] > lo).any(), "an obstacle is left"
        deps = dependants(st["re-insert 3"], st["delete everything"], gs)
        assert len(deps) > 0 and (st["delete everything"]["cobs"][deps, 0] < 0).all()
        deps = dependants(st["re-insert 2"], st["delete in a box"], gs)
        x = np.unravel_index(deps, gs)[0]
        assert 0 < int((x > 14).sum()) < len(deps), "dependants on both sides of the update box's face"
    if name == "snake":
        deps = dependants(st["insert"], st["delete A"], gs)
        assert len(deps) > 2048, len(deps)


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


@pytest.mark.parametrize("scenario", list(SCENARIOS))
def test_reseed_matches_reference(reference, scenario, monkeypatch):
    for k in X_ENV:
        monkeypatch.delenv(k, raising=False)
    steps, gs = reference(scenario)
    it = iter(steps)
    n = 0
    for tag, res, m in replay(scenario, device_map):
        wtag, wres, wst = next(it)
        assert tag == wtag
        assert same(res, wres), (tag, "step results differ from the reference's")
        if wst is not None:
            st = state(m)
            r = mismatch(st, wst, gs)
            assert r["dist"] == 0 and r["cobs_tie"] == 0 and r["cobs_nontie"] == 0 and r["occ"] == 0, (tag, r)
            assert st["counts"] == wst["counts"], (tag, "inserts, deletes, expansions", st["counts"], wst["counts"])
        n += 1
    assert n == len(steps)


RESEED = re.compile(r"^\[x\] reseed: dependants (\d+) final after classify (\d+) closure rounds (\d+) list entries (\d+) resolve passes (\d+)$", re.M)


@pytest.mark.parametrize("scenario,rounds,passes", [("block", 3, 1), ("snake", 3, 10)])
def test_reseed_stages_ran(reference, scenario, rounds, passes):
    e = {k: v for k, v in os.environ.items() if k not in X_ENV}
    e["FIESTA_DEBUG_X"] = "1"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.test_gpu_reseed", scenario]
    p = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    lines = [tuple(int(v) for v in t) for t in RESEED.findall(p.stderr)]
    assert lines, "no re-seeding in the FIESTA_DEBUG_X trace"
    assert max(t[2] for t in lines) >= rounds and max(t[4] for t in lines) >= passes, lines
    assert any(0 < t[1] < t[0] for t in lines), lines           # some dependants final after the classification, some not
    steps, gs = reference(scenario)
    out = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["counts"] == [list(st["counts"]) for _, _, st in steps if st is not None]
    assert out["digest"] == digest(steps[-2][2])


def main(scenario):
    counts, last = [], None
    for tag, res, m in replay(scenario, device_map):
        if tag != "query":
            last = state(m)
            counts.append(list(last["counts"]))
    print(json.dumps(dict(scenario=scenario, counts=counts, digest=digest(last))))


if __name__ == "__main__":
    main(sys.argv[1])
