"""SMALL generations of k_x_relax under their two schedules, against the sequential reference on the small adversarial maps
of tests/test_gpu_xrelax_schedules.py.

  FIESTA_X_SMALL_ASYNC=0|1  1: a SMALL generation runs its whole behaviour fixpoint from the device work queue (x_async),
                            seeded with every element instead of round 1, then commits; phase "s.async" of the trace.
                            0 (default): round 1 and later rounds ("s.round1", "s.rounds").  FIESTA_X_ASYNC=0 turns
                            every queue off.  Read when a map is created, like FIESTA_X_SMALL.

Each schedule below is compared with the reference after every update (distance_, closest_obstacle_ with ties, occupancy,
expansion counts, trilinear queries), and a child process with FIESTA_DEBUG_X=1 shows from the kernel's phase counts that
the schedule's path ran."""
import pytest

from tests.test_gpu_xrelax_schedules import (  # noqa: F401  (reference: the fixture, one reference replay per scenario)
    LARGE_GENERATIONS, SCENARIOS, X_ENV, check_against_reference, digest, reference, traced_run)

pytestmark = pytest.mark.gpu

ENV = X_ENV + ("FIESTA_X_SMALL_ASYNC",)

Q = {"FIESTA_X_SMALL_ASYNC": "1"}
SCHEDULES = {
    "small-queue": dict(Q),                                                     # SMALL generations from the queue
    "small-rounds": {},                                                         # the default: their round schedule
    "no-queue": dict(Q, FIESTA_X_ASYNC="0"),                                    # no queue anywhere, whatever SMALL_ASYNC says
    "all-small-queue": dict(Q, FIESTA_X_SMALL="65536"),                         # SMALL generations of up to 65 536 entries, queued
    "mixed-queue": dict(Q, FIESTA_X_SMALL="256", FIESTA_X_DENSE="64"),          # SMALL <-> BIG hand-overs, both queues
}

# schedule -> (scenario, required phase counts)
COVERAGE = {
    "small-queue": ("salt-and-pepper", {"s.async": ">0", "s.round1": 0, "s.rounds": 0, "round1": 0}),
    "small-rounds": ("salt-and-pepper", {"s.round1": ">0", "s.async": 0}),
    "no-queue": ("salt-and-pepper", {"s.round1": ">0", "s.async": 0, "async": 0}),
    "all-small-queue": ("mass-delete", {"s.async": ">0", "s.round1": 0}),       # and generations of 32769..65536 entries (below)
    "mixed-queue": ("salt-and-pepper", {"round1": ">0", "s.async": ">0", "s.round1": 0}),
}

MATRIX = [pytest.param(sc, sh, id="%s:%s" % (sc, sh)) for sc in SCENARIOS for sh in SCHEDULES
          if sh != "all-small-queue" or sc in LARGE_GENERATIONS]


def set_schedule(monkeypatch, env):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("scenario,schedule", MATRIX)
def test_small_schedule_matches_reference(reference, scenario, schedule, monkeypatch):  # noqa: F811
    set_schedule(monkeypatch, SCHEDULES[schedule])
    check_against_reference(reference, scenario)


@pytest.mark.parametrize("schedule", list(COVERAGE))
def test_small_schedule_takes_its_path(reference, schedule, monkeypatch):  # noqa: F811
    scenario, need = COVERAGE[schedule]
    monkeypatch.delenv("FIESTA_X_SMALL_ASYNC", raising=False)  # traced_run drops the other settings from the environment
    out, counts, gens = traced_run(scenario, SCHEDULES[schedule])
    assert counts, "no FIESTA_DEBUG_X trace on stderr"
    for name, want in need.items():
        n = counts.get(name, 0)
        assert (n > 0) if want == ">0" else (n == want), (schedule, name, n, counts)
    steps, gs = reference(scenario)
    assert out["counts"] == [list(st["counts"]) for _, _, st in steps if st is not None], (schedule, out["counts"])
    assert out["digest"] == digest(steps[-2][2])
    if schedule == "all-small-queue":
        assert any(32768 < n <= 65536 for n in gens), sorted(gens)[-4:]
