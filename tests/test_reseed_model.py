"""The four-stage re-seeding of k_x_reseed (scripts/reseed_model.c, the CPU model on top of oracle/exact_model.c's replays)
gives, on every delete of every replay and on a synthetic delete of a solid block of dependants (deep closure, long parent
chains, three dependant orders, with and without an update box that cuts the block), exactly what one sequential sweep of
the reference's rule gives; and each of four wrong variants of the model fails on them."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "scripts", "reseed_model.c")
# (G, obs, rounds, nops, small, local)
CONFIGS = [(32, 0.7, 6, 1500, 64, 0), (40, 0.6, 6, 3000, 16, 1)]
SEEDS = range(1, 5)
MUTATIONS = ["MUT_B_ANY_ORDER", "MUT_C_LAST", "MUT_C_STATIC", "MUT_D_SHORT"]


def compile_model(tmp_path_factory, define=None):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("reseed") / ("reseed_model" + ("_" + define if define else "")))
    subprocess.check_call([cc, "-O2", "-ffp-contract=off"] + (["-D" + define] if define else []) + ["-o", exe, SRC, "-lm"])
    return exe


def run(exe, cfg, seed):
    if cfg[0] == "block":                                      # ("block", G, order, local)
        args = [exe, "block", str(cfg[1]), str(seed), str(cfg[2]), str(cfg[3])]
    else:
        G, obs, rounds, nops, small, local = cfg
        args = [exe, str(G), str(obs), str(rounds), str(nops), str(seed), str(small), str(local)]
    p = subprocess.run(args, capture_output=True, text=True, timeout=300)
    return p, re.search(r"^reseed (OK|FAIL): deletes (\d+) dependants (\d+) final after classify (\d+) closure rounds max (\d+) "
                        r"resolve passes max (\d+)$", p.stdout, re.M)


@pytest.mark.parametrize("cfg", CONFIGS, ids=["global", "local-box"])
def test_stages_match_one_sequential_sweep(tmp_path_factory, cfg):
    exe = compile_model(tmp_path_factory)
    deps = final = 0
    rounds = passes = 0
    for seed in SEEDS:
        p, m = run(exe, cfg, seed)
        assert p.returncode == 0 and m and m.group(1) == "OK", p.stdout[-2000:]
        assert "\nOK\n" in p.stdout                            # exact_model.c's own comparison with the reference
        deps += int(m.group(3)); final += int(m.group(4))
        rounds = max(rounds, int(m.group(5))); passes = max(passes, int(m.group(6)))
    # every stage had work: dependants that needed the closure, its pushing rounds, and pointer jumping beyond one pass
    assert 0 < final < deps and rounds >= 2 and passes >= 2, (deps, final, rounds, passes)


BLOCKS = [("block", 40, order, local) for order in (0, 1, 2) for local in (0, 1)]


@pytest.mark.parametrize("cfg", BLOCKS, ids=lambda c: "order%d-%s" % (c[2], "box" if c[3] else "global"))
def test_stages_match_one_sequential_sweep_on_a_block(tmp_path_factory, cfg):
    exe = compile_model(tmp_path_factory)
    for seed in (1, 2):
        p, m = run(exe, cfg, seed)
        assert p.returncode == 0 and m and m.group(1) == "OK", p.stdout[-2000:]
        deps, final, rounds, passes = (int(m.group(k)) for k in (3, 4, 5, 6))
        assert 0 < final < deps and rounds >= 2 and passes >= 3, (deps, final, rounds, passes)
        if cfg[2] != 1:                                        # surface inwards, or random: deep closure, long chains
            assert rounds >= 3 and passes >= 4, (deps, final, rounds, passes)


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_is_caught(tmp_path_factory, mutation):
    exe = compile_model(tmp_path_factory, mutation)
    for cfg in [CONFIGS[0]] + [c for c in BLOCKS if c[2] == 2]:   # the replays, and the block in random order
        results = [run(exe, cfg, seed) for seed in SEEDS]
        assert any(p.returncode != 0 and m and m.group(1) == "FAIL" for p, m in results), (mutation, cfg)
