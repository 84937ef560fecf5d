"""SMALL generations of k_x_relax resolved entirely from the work queue: scripts/exact_async_model.c with SMALL_ASYNC = 2
seeds the queue with every element of a SMALL generation instead of running round 1 (each worker claims its own share of
the elements, IDLE -> RUNNING, and evaluates them before it pops), and refreshes nothing afterwards (the commit re-stages
the final words).  Over many seeds, with inserts, deletes with re-seeding and local update boxes, the
result must be the sequential reference's voxel for voxel and expansion for expansion.  Built with -DNO_DIRTY_RULE (a
running element that gets marked is not evaluated again), the same replays must fail."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (workers, small_async, G, obs, rounds, nops, small, local, dense_min)
CONFIGS = {
    "all-small-local": (64, 2, 40, 0.7, 6, 3000, 1000000, 1, 16),    # every generation SMALL, local update boxes
    "all-small-global": (64, 2, 32, 0.6, 5, 1500, 1000000, 0, 16),   # every generation SMALL, whole-grid updates
    "small-and-big": (64, 2, 40, 0.7, 6, 3000, 16, 1, 1024),         # SMALL <-> BIG hand-overs, BIG queue from round 2
    "few-workers": (8, 2, 32, 0.6, 5, 1500, 4096, 1, 16),
}
MUTATION_CONFIGS = ("all-small-local", "all-small-global")          # every generation SMALL: the new path alone
SEEDS = range(1, 9)


def compile_model(tmp_path_factory, name, defines=()):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("model") / name)
    subprocess.check_call([cc, "-O2", "-ffp-contract=off"] + list(defines) +
                          ["-o", exe, os.path.join(ROOT, "scripts", "exact_async_model.c"), "-lm"], stderr=subprocess.DEVNULL)
    return exe


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return compile_model(tmp_path_factory, "exact_async_model")


@pytest.fixture(scope="module")
def model_no_dirty(tmp_path_factory):
    return compile_model(tmp_path_factory, "exact_async_model_no_dirty", ["-DNO_DIRTY_RULE"])


def run(exe, cfg, seed):
    workers, small_async, G, obs, rounds, nops, small, local, dense_min = cfg
    args = [exe, str(workers), str(small_async), str(G), str(obs), str(rounds), str(nops), str(seed), str(small), str(local), str(dense_min)]
    p = subprocess.run(args, capture_output=True, text=True, timeout=300)
    ok = p.returncode == 0 and "\nOK\n" in p.stdout and all(re.search(r"dist mismatches 0 cobs mismatches 0$", line)
                                                            for line in p.stdout.splitlines() if line.startswith("[gens"))
    return ok, args, p.stdout


@pytest.mark.parametrize("name", list(CONFIGS))
def test_whole_generation_queue_matches_sequential_reference(model, name):
    seeded = 0
    for seed in SEEDS:
        ok, args, out = run(model, CONFIGS[name], seed)
        assert ok, (args, out[-2000:])
        seeded += int(re.search(r"seeded entries (\d+)", out.splitlines()[-1]).group(1))
    assert seeded > 0                                          # the queue ran


@pytest.mark.parametrize("name", MUTATION_CONFIGS)
def test_whole_generation_queue_needs_the_dirty_rule(model_no_dirty, name):
    assert any(not run(model_no_dirty, CONFIGS[name], seed)[0] for seed in SEEDS), "the replays do not catch a missed re-run"
