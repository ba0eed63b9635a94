"""Memory-bounded column and pedigree sweeps (DESIGN §4.3): back-pointers beyond the budget are cut into segments that share one
arena and are swept again, right to left, during the backtrace.  The result must be the one of the resident sweep, on every path
(fused trio sweep, batched two-pass sweep, sequential column sweep), for budgets from a third of the table down to about one
column; what no segment fits is refused with the bytes it needs.  WHMEC_COLUMN_ARENA_BUDGET (bytes for the shared arena;
checkpoints come on top) forces the mode on problems that fit."""
import re

import numpy as np
import pytest

from whatshap_b200 import multigpu, synth
from whatshap_b200._abi import Unsupported

pytestmark = pytest.mark.gpu

HOOK = "WHMEC_COLUMN_ARENA_BUDGET"
ENV = (HOOK, "WHMEC_PED_FUSED", "WHMEC_PED_SEQUENTIAL", "WHMEC_FORCE_COLUMN_KERNEL", "WHMEC_SOLVE_GROUPS")
PEDS = ["trio", "trio_child_first", "quartet", "three_generations", "three_children", "four_children"]
COV = {"trio": 9, "trio_child_first": 9, "quartet": 8, "three_generations": 7, "three_children": 6, "four_children": 6}
PATHS = {"default": {}, "batched": {"WHMEC_PED_FUSED": "0"}, "sequential": {"WHMEC_PED_SEQUENTIAL": "1"}}


def clean(monkeypatch, env=None):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)


def instance(ped, distrust, chains, seed):
    """A random_problem (tie-heavy weights, gaps, blanks) with several chains, or with exactly one chain."""
    for attempt in range(200):
        rng = np.random.Generator(np.random.PCG64([seed, attempt]))
        if chains == "one":
            prob = synth.random_problem(rng, 40, COV.get(ped, 10), ped, distrust=distrust, gap=0.1, mean_len=8.0, burst=4)
            if len(multigpu.independent_blocks(prob)) == 1:
                return prob
        else:
            prob = synth.random_problem(rng, 90, COV.get(ped, 10), ped, distrust=distrust)
            if len(multigpu.independent_blocks(prob)) >= 4:
                return prob
    raise AssertionError("no instance of the wanted chain structure")


def least_budget(gpu, monkeypatch, prob):
    """The refusal of a tiny budget states a lower bound; double it until a solve fits (about one column per segment)."""
    monkeypatch.setenv(HOOK, "8")
    with pytest.raises(Unsupported) as e:
        gpu.solve(prob)
    need = int(re.search(r"needs at least (\d+) bytes", str(e.value)).group(1))
    for _ in range(24):
        monkeypatch.setenv(HOOK, str(need))
        try:
            return need, gpu.solve(prob)
        except Unsupported:
            need *= 2
    raise AssertionError("no budget fits")


def check_budgets(gpu, monkeypatch, prob, path_kinds):
    """Resident solve, then bounded solves at about one column and resident/1.5, /3, /8: same solution, a smaller arena."""
    monkeypatch.delenv(HOOK, raising=False)
    whole, st = gpu.solve(prob)
    resident = st["backptr_bytes"]
    assert st["path_kind"] in path_kinds, st
    launches = {st["kernel_launches"]}
    least, (got, st2) = least_budget(gpu, monkeypatch, prob)
    assert got.same_as(whole), ("least", least, st2, got.diff(whole))
    assert st2["backptr_bytes"] < resident
    launches.add(st2["kernel_launches"])
    for divisor in (1.5, 3, 8):  # (not below the widest column of these small instances)
        monkeypatch.setenv(HOOK, str(max(int(resident / divisor), least)))
        got, st2 = gpu.solve(prob)
        assert got.same_as(whole), (divisor, st2, got.diff(whole))
        assert st2["backptr_bytes"] < resident, (divisor, st2, resident)
        assert st2["path_kind"] in path_kinds, st2
        launches.add(st2["kernel_launches"])
    assert len(launches) >= 2, launches  # other budgets, other numbers of segments swept again
    monkeypatch.delenv(HOOK, raising=False)
    return whole


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("chains", ["several", "one"])
@pytest.mark.parametrize("distrust", [False, True])
@pytest.mark.parametrize("ped", PEDS)
def test_bounded_equals_resident(gpu, monkeypatch, ped, distrust, chains, path):
    clean(monkeypatch, PATHS[path])
    prob = instance(ped, distrust, chains, seed=PEDS.index(ped) * 4 + 2 * distrust + (chains == "one"))
    # two-pass sweeps need several chains; a segment budget below one chain's back-pointers takes the column sweep (2)
    kinds = {2} if path == "sequential" or chains == "one" else {2, 3}
    check_budgets(gpu, monkeypatch, prob, kinds)


@pytest.mark.parametrize("chains", ["several", "one"])
def test_single_individual_on_the_column_kernel(gpu, monkeypatch, chains):
    clean(monkeypatch, {"WHMEC_FORCE_COLUMN_KERNEL": "1"})
    prob = instance("single", False, chains, seed=99) if chains == "several" else synth.sliding_window(120, 12, block_len=120, seed=4)
    check_budgets(gpu, monkeypatch, prob, {2})


@pytest.mark.parametrize("key,make", [
    ("cfg5-shaped trio", lambda: synth.trio(120, 5, block_len=60, seed=20250935)),  # a = 15, T = 4, 2 chains
    ("three_children", lambda: synth.nuclear_family(40, 3, 2, block_len=20, seed=7)),  # T = 64
])
@pytest.mark.parametrize("path", list(PATHS))
def test_bounded_equals_the_reference(gpu, checker, monkeypatch, key, make, path):
    """Against the compiled reference (oracle/_ref) where it was built, the C restatement elsewhere."""
    clean(monkeypatch, PATHS[path])
    prob = make()
    want = checker.solve(prob)
    monkeypatch.setenv(HOOK, "1000000000")
    _, st = gpu.solve(prob)  # (the budget holds everything: resident)
    for divisor in (2, 5):
        monkeypatch.setenv(HOOK, str(st["backptr_bytes"] // divisor))
        got, st2 = gpu.solve(prob)
        assert st2["backptr_bytes"] < st["backptr_bytes"]
        assert got.same_as(want), (key, divisor, st2, got.diff(want))


def test_impossible_budget_is_refused(gpu, monkeypatch):
    clean(monkeypatch, {HOOK: "4096"})
    prob = synth.nuclear_family(30, 4, 2, block_len=30, seed=1)  # T = 256, 12 reads: a column's back-pointers alone are 32 KiB
    with pytest.raises(Unsupported, match=r"needs at least \d+ bytes"):
        gpu.solve(prob)


def test_defaults_unchanged(gpu, monkeypatch):
    """Without the hook (or with a budget the table fits) the resident sweeps run as before."""
    clean(monkeypatch)
    trio = synth.trio(120, 5, block_len=60, seed=20250935)
    a, st = gpu.solve(trio)
    assert (st["path_kind"], st["kernel_launches"]) == (3, 3), st  # fused trio sweep: unit pass, prefix, true pass
    clean(monkeypatch, {HOOK: str(st["backptr_bytes"])})
    b, st2 = gpu.solve(trio)
    assert b.same_as(a) and (st2["path_kind"], st2["kernel_launches"], st2["backptr_bytes"]) == (3, 3, st["backptr_bytes"])
    fam = synth.nuclear_family(200, 2, 2, block_len=50, seed=3)  # T = 16: batched sweep
    clean(monkeypatch)
    c, st3 = gpu.solve(fam)
    clean(monkeypatch, {HOOK: str(st3["backptr_bytes"])})
    d, st4 = gpu.solve(fam)
    assert st3["path_kind"] == 3 and c.same_as(d)
    assert (st4["kernel_launches"], st4["backptr_bytes"]) == (st3["kernel_launches"], st3["backptr_bytes"])
