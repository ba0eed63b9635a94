"""Many genotyping tables in one call on the GPU (`whmec_genotype_batch`, DESIGN §4.9): every table of mixed-shape lists against its
own `whmec_genotype` and the golden answers, the launch count of the plan, groups and a memory-bounded table under a small
WHMEC_GENOTYPE_ARENA_BUDGET, errors that stay with their table, and the objects of `GenotypeDPTable.batch`."""
import numpy as np
import pytest

import emul_genotype_batch as eb
from emul_genotype_bounded import genotype_bounded
from test_devices import objects_with_priors
from test_genotype import TOL_DEVICE, close, golden
from test_genotype_batch import bad_tables, many_chains, mixed_list, planned_launches
from whatshap_b200 import _lib, adapters, core, multigpu, synth

pytestmark = pytest.mark.gpu
TOL_SINGLE = 1e-12


@pytest.fixture(autouse=True)
def no_env(monkeypatch):
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.delenv("WHMEC_GENOTYPE_ARENA_BUDGET", raising=False)


def check_against_single(probs, got):
    for i, (p, g) in enumerate(zip(probs, got)):
        want, _ = _lib.genotype(p)
        assert isinstance(g, np.ndarray) and close(g, want, TOL_SINGLE), (i, p.n_ind, p.n_trios)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_mixed_shapes_equal_their_own_calls(seed):
    probs = mixed_list(seed, 24)
    got, (stats, total) = _lib.genotype_batch(probs, with_stats=True)
    check_against_single(probs, got)
    _, info = eb.genotype_batch(probs)
    assert info["groups"] == 1 and total["kernel_launches"] == info["launches"] == planned_launches(probs, info["group_of"])
    assert all(st["path_kind"] == 4 and st["sweep_ms"] == 0 and st["transmissions"] == 4 ** p.n_trios for st, p in zip(stats, probs))
    assert total["sweep_ms"] > 0 and total["cells"] == sum(st["cells"] for st in stats)


def test_golden_cases_and_many_single_sample_tables():
    cases = list(golden())
    rng = np.random.default_rng(9)
    singles = [synth.genotyping_problem(rng, int(rng.integers(2, 60)), int(rng.integers(2, 9)), "single") for _ in range(240)]
    probs = [p for _, p, _, _ in cases] + singles
    got, (stats, total) = _lib.genotype_batch(probs, with_stats=True)
    for (label, _, want, _), g in zip(cases, got):
        assert close(g, want, TOL_DEVICE), label
    check_against_single(probs, got)
    _, info = eb.genotype_batch(probs)
    assert total["kernel_launches"] == info["launches"]


def test_a_step_of_more_than_65535_sub_tables_is_split():
    probs = [many_chains(70000), synth.genotyping_problem(np.random.default_rng(15), 30, 4, "trio")]
    got, (stats, total) = _lib.genotype_batch(probs, with_stats=True)
    check_against_single(probs, got)
    _, info = eb.genotype_batch(probs)
    assert total["kernel_launches"] == info["launches"] > planned_launches(probs, info["group_of"])


def test_small_budget_makes_groups_and_runs_a_bounded_table_inside_the_call(monkeypatch):
    rng = np.random.default_rng(11)
    probs = [synth.genotyping_problem(rng, int(rng.integers(5, 40)), 4, ("single", "trio", "quartet", "trio_child_first")[i % 4]) for i in range(18)]
    big = synth.genotyping_problem(np.random.default_rng(12), 400, 7, "trio")
    probs.insert(7, big)
    costs = [eb.cost(p) for p in probs]
    budget = sorted(costs)[-2] + 1  # every table but the trio of 400 columns fits a group; that one runs memory-bounded
    assert costs[7] == max(costs) and genotype_bounded(big, budget)[1]["segments"] > 1
    monkeypatch.setenv("WHMEC_GENOTYPE_ARENA_BUDGET", str(budget * 8))
    got, (stats, total) = _lib.genotype_batch(probs, with_stats=True)
    _, info = eb.genotype_batch(probs, budget_doubles=budget)
    assert info["groups"] >= 3 and info["alone"] == 1 and info["group_of"][7] == -1
    assert stats[7]["kernel_launches"] > 4 * big.n_cols - 2  # bounded: backward sweeps repeated from checkpoints
    assert total["kernel_launches"] == info["launches"] + stats[7]["kernel_launches"]
    monkeypatch.delenv("WHMEC_GENOTYPE_ARENA_BUDGET")
    check_against_single(probs, got)


def test_error_tables_fail_alone():
    rng = np.random.default_rng(13)
    probs, kinds = [], []
    for p, typ, text in bad_tables():
        probs += [synth.genotyping_problem(rng, int(rng.integers(3, 30)), 4, ("single", "trio", "quartet")[len(probs) % 3]), p]
        kinds += [None, (typ, text)]
    got = _lib.genotype_batch(probs)
    for p, g, k in zip(probs, got, kinds):
        if k is None:
            assert close(g, _lib.genotype(p)[0], TOL_SINGLE)
        else:
            with pytest.raises(k[0]) as e:
                _lib.genotype(p)
            assert type(g) is type(e.value) and str(g) == str(e.value) and k[1] in str(g)


def test_objects_from_batch_equal_constructed_ones():
    rng = np.random.default_rng(14)
    Recording = adapters.recording_pedigree(core.Pedigree)
    swap = adapters.make_genotype_table_class(core)
    items = []
    for shape in ("single", "trio", "single", "quartet", "three_generations", "single"):
        prob = synth.genotyping_problem(rng, int(rng.integers(5, 60)), 5, shape)
        rs, recomb, ped = objects_with_priors(prob, Recording)
        items.append((prob, (ped.numeric_sample_ids, rs, recomb, ped, prob.positions.tolist())))
    for cls, kw in ((core.GenotypeDPTable, {}), (core.GenotypeDPTable, {"devices": [0, 0]}), (swap, {})):
        objs = cls.batch([args for _, args in items], **kw)
        for (prob, args), obj in zip(items, objs):
            one = cls(*args)
            for i in range(prob.n_ind):
                for k in range(prob.n_cols):
                    a, b = obj.get_genotype_likelihoods(i, k).as_vector(), one.get_genotype_likelihoods(i, k).as_vector()
                    assert np.allclose(a, b, rtol=0, atol=TOL_SINGLE, equal_nan=True), (cls, kw, i, k)
