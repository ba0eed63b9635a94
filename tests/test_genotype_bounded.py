"""Memory-bounded forward-backward genotyping (DESIGN §4.5) without a GPU: a table whose backward tables exceed the budget is cut
into segments that share one arena and are swept backward again from checkpoints (gl_bounded, stepped on the host by
tests/emul).  The recomputed backward tables come from the same checkpoints through the same serial operations, so the
likelihoods equal the resident ones bit for bit, at every budget from the least that fits up to resident / 1.5."""
import re

import numpy as np
import pytest

import emul_genotype
import emul_genotype_bounded
from oracle import checker
from whatshap_b200 import synth
from whatshap_b200._abi import Unsupported

TOL_DEVICE = 1e-9
PEDS = ["single", "trio", "quartet", "three_generations", "three_children"]
COV = {"single": 8, "trio": 5, "quartet": 4, "three_generations": 4, "three_children": 4}


def tables(own):
    """(first, last + 1) of every table, and its resident cost: backward tables + two projection buffers (doubles)."""
    out, lo = [], 0
    for k, w in enumerate(own):
        if w == 0:  # a table's last column owns no backward table
            out.append((lo, k + 1, int(own[lo:k + 1].sum()) + 2 * max(1, int(own[lo:k + 1].max()))))
            lo = k + 1
    return out


def instance(ped, seed):
    """One table of 40-60 columns; for a single individual several tables, of which the longest costs the most by far."""
    for attempt in range(400):
        rng = np.random.Generator(np.random.PCG64([seed, attempt]))
        n = int(rng.integers(40, 61))
        if ped == "single":
            prob = synth.genotyping_problem(rng, 3 * n, COV[ped], ped, prior="random", gap=0.04, mean_len=5.0)
            t = sorted(c for _, _, c in tables(emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"]))
            if len(t) >= 3 and t[-1] > 3 * t[-2]:
                return prob, t[-1], t[-2]
        else:
            prob = synth.genotyping_problem(rng, n, COV[ped], ped, prior="random")
            t = tables(emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"])
            if len(t) == 1 and t[0][1] - t[0][0] == n:
                return prob, t[0][2], 0
    raise AssertionError("no instance")


def least_budget(prob):
    """A budget below one column is refused with the bytes it needs; that many bytes (in doubles) must fit."""
    with pytest.raises(Unsupported) as e:
        emul_genotype_bounded.genotype_bounded(prob, 1)
    return int(re.search(r"needs at least (\d+) bytes", str(e.value)).group(1)) // 8


@pytest.mark.parametrize("ped", PEDS)
def test_bounded_equals_resident(ped):
    prob, resident, second = instance(ped, PEDS.index(ped))
    whole, _ = emul_genotype.genotype(prob)
    want = checker.port().genotype(prob)
    assert np.all(np.abs(whole - want) <= TOL_DEVICE)
    least = least_budget(prob)
    assert least < resident
    budgets = sorted({max(least, second, int(resident / d)) for d in (1.5, 3, 8)} | {max(least, second)})
    segments = []
    for budget in budgets:
        got, info = emul_genotype_bounded.genotype_bounded(prob, budget)
        assert np.array_equal(got, whole, equal_nan=True), (ped, budget)
        assert np.all(np.abs(got - want) <= TOL_DEVICE), (ped, budget)
        assert info["segments"] > 1, (ped, budget, info)
        plan = emul_genotype_bounded.bounded_plan(prob, budget)
        assert plan["arena"] + plan["ckpt"] + plan["pool"] <= budget, (ped, budget, plan)
        cuts, own = plan["cuts"], plan["own"]
        assert len(cuts) - 1 == info["segments"]
        # the first segment, swept backward only once, is the largest that fits the arena
        first = int(own[cuts[0]:cuts[1]].sum())
        assert first <= plan["arena"] < first + int(own[cuts[1]]), (ped, budget, cuts, plan)
        segments.append(info["segments"])
    assert segments == sorted(segments, reverse=True) and segments[0] > segments[-1], (ped, budgets, segments)


def test_only_the_table_that_does_not_fit_is_cut():
    """A single individual: every other table still runs whole, in groups; the longest one is cut."""
    prob, resident, second = instance("single", 7)
    own = emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"]
    longest = max(tables(own), key=lambda t: t[2])
    plan = emul_genotype_bounded.bounded_plan(prob, max(second, resident // 2))
    assert plan["cuts"][0] == longest[0] and plan["cuts"][-1] == longest[1], (plan["cuts"], longest)
    got, info = emul_genotype_bounded.genotype_bounded(prob, max(second, resident // 2))
    assert info["segments"] > 1 and np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)


def test_resident_budget_cuts_nothing():
    prob, resident, _ = instance("trio", 11)
    got, info = emul_genotype_bounded.genotype_bounded(prob, resident)
    assert info["segments"] == 1 and len(emul_genotype_bounded.bounded_plan(prob, resident)["cuts"]) == 0
    assert np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)


def test_impossible_budget_states_what_fits():
    prob, _, _ = instance("three_children", 5)
    with pytest.raises(Unsupported, match=r"needs at least \d+ bytes"):
        emul_genotype_bounded.genotype_bounded(prob, 100)
    least = least_budget(prob)
    got, info = emul_genotype_bounded.genotype_bounded(prob, least)
    assert info["segments"] > 1 and np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)


def test_host_errors_are_unchanged():
    """Missing priors and a read on a single variant are refused with the messages of the resident path."""
    from whatshap_b200._abi import FlatProblem

    single = FlatProblem(positions=[10, 20, 30], read_off=[0, 2, 3], ent_col=[0, 1, 1], ent_allele=[0, 1, 1], ent_phred=[10, 10, 10],
                         read_ind=[0, 0], recombcost=[1, 1, 1], n_ind=1, distrust=True, gl=np.full((1, 3, 3), 1 / 3.0))
    with pytest.raises(RuntimeError, match="single variant"):
        emul_genotype_bounded.genotype_bounded(single, 1)
    prob = synth.genotyping_problem(np.random.default_rng(1), 10, 4)
    prob.gl = None
    with pytest.raises(RuntimeError, match="priors"):
        emul_genotype_bounded.genotype_bounded(prob, 1)
