"""The asynchronous schedule of k_x_relax (scripts/exact_async_model.c, the CPU model of x_async on top of
oracle/exact_model.c) reproduces the sequential reference voxel for voxel and expansion for expansion, over many seeds,
in BIG generations (work queue after round 1 / the dense rounds), in SMALL generations, with and without a local update
box, with deletes (re-seeding) in every replay.  Built with -DNO_DIRTY_RULE (a running element that gets marked is not
evaluated again), replays whose generations are all BIG must fail."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (workers, G, obs, rounds, nops, small, local, dense_min)
CONFIGS = [
    (64, 40, 0.7, 6, 3000, 16, 1, 1024),     # BIG queue from round 2, SMALL generations in rounds
    (64, 40, 0.7, 6, 3000, 8, 0, 64),        # BIG queue after dense rounds, SMALL generations in rounds
    (8, 32, 0.6, 5, 1500, 64, 0, 16),        # few workers, mostly SMALL generations
]
# the BIG queue on its own (every generation BIG, local update boxes): the configurations in which the replays catch a
# missed re-run
MUTATION_CONFIGS = {
    "all-big-queue": (64, 40, 0.7, 6, 3000, 0, 1, 1024),
    "mostly-big-queue": (64, 40, 0.7, 6, 3000, 16, 1, 1024),
}
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
    workers, G, obs, rounds, nops, small, local, dense_min = cfg
    args = [exe, str(workers), str(G), str(obs), str(rounds), str(nops), str(seed), str(small), str(local), str(dense_min)]
    p = subprocess.run(args, capture_output=True, text=True, timeout=300)
    ok = p.returncode == 0 and "\nOK\n" in p.stdout and all(re.search(r"dist mismatches 0 cobs mismatches 0$", line)
                                                            for line in p.stdout.splitlines() if line.startswith("[gens"))
    return ok, args, p.stdout


@pytest.mark.parametrize("cfg", CONFIGS, ids=["big-queue+small-rounds", "big-queue-after-dense", "mostly-small-rounds"])
def test_async_schedule_matches_sequential_reference(model, cfg):
    evals = 0
    for seed in SEEDS:
        ok, args, out = run(model, cfg, seed)
        assert ok, (args, out[-2000:])
        evals += int(re.search(r"evaluations (\d+)", out.splitlines()[-1]).group(1))
    assert evals > 0                                           # the queue ran


@pytest.mark.parametrize("name", list(MUTATION_CONFIGS))
def test_async_schedule_needs_the_dirty_rule(model_no_dirty, name):
    assert any(not run(model_no_dirty, MUTATION_CONFIGS[name], seed)[0] for seed in SEEDS), "the replays do not catch a missed re-run"
