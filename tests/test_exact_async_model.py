"""The asynchronous schedule of k_x_relax (scripts/exact_async_model.c, the CPU model of x_async on top of
oracle/exact_model.c) reproduces the sequential reference voxel for voxel and expansion for expansion, over many seeds,
in BIG generations (work queue after round 1 / the dense rounds), in SMALL generations, with and without a local update
box, with deletes (re-seeding) in every replay."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (workers, small_async, G, obs, rounds, nops, small, local, dense_min)
CONFIGS = [
    (64, 1, 40, 0.7, 6, 3000, 16, 1, 1024),     # BIG queue from round 2, SMALL generations on the queue too
    (64, 0, 40, 0.7, 6, 3000, 8, 0, 64),        # BIG queue after dense rounds, SMALL generations in rounds
    (8, 1, 32, 0.6, 5, 1500, 64, 0, 16),        # few workers, mostly SMALL generations
]


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("model") / "exact_async_model")
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "scripts", "exact_async_model.c"), "-lm"])
    return exe


@pytest.mark.parametrize("cfg", CONFIGS, ids=["big+small", "big-after-dense", "small"])
def test_async_schedule_matches_sequential_reference(model, cfg):
    workers, small_async, G, obs, rounds, nops, small, local, dense_min = cfg
    evals = 0
    for seed in range(1, 9):
        args = [model, str(workers), str(small_async), str(G), str(obs), str(rounds), str(nops), str(seed), str(small), str(local), str(dense_min)]
        p = subprocess.run(args, capture_output=True, text=True, timeout=300)
        assert p.returncode == 0 and "\nOK\n" in p.stdout, (args, p.stdout[-2000:])
        for line in p.stdout.splitlines():
            if line.startswith("[gens"):
                assert re.search(r"dist mismatches 0 cobs mismatches 0$", line), line
        evals += int(re.search(r"evaluations (\d+)", p.stdout.splitlines()[-1]).group(1))
    assert evals > 0                                           # the queue ran
