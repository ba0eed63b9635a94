"""`whmec_heuristic_batch` on the GPU (DESIGN §4.10): one CTA per table must give every table what `whmec_heuristic` gives it
alone, bit for bit, and the stored answers of the reference (tests/golden/heuristic.npz) for the golden tables."""
import numpy as np
import pytest

from test_heuristic import golden_cases
from test_heuristic_batch import alone, assert_same, constructor_args, random_list, same_answers
from whatshap_b200 import _lib, adapters, core, multigpu, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def one_device(monkeypatch):
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.delenv("WHMEC_HEURISTIC_ARENA_BUDGET", raising=False)


def test_golden_vectors_in_one_call():
    cases = list(golden_cases())
    got, (stats, total) = _lib.heuristic_batch([c[1] for c in cases], [c[2] for c in cases], True, with_stats=True)
    for (i, prob, row_limit, want, n_samples), g, st in zip(cases, got, stats):
        assert_same(g, _lib.heuristic(prob, row_limit, True), i)
        for field in ("partition", "transmission"):
            assert np.array_equal(getattr(g, field), want[field]), (i, field)
        assert np.array_equal(g.haplotypes[:n_samples], want["haplotypes"]) and np.array_equal(g.mutated[:n_samples], want["mutated"]), i
    assert total["kernel_launches"] == 1 and sum(st["path_kind"] == 6 for st in stats) >= 50


def test_300_random_mixed_tables():
    probs, limits = random_list(1001, 300)
    got, (stats, total) = _lib.heuristic_batch(probs, limits, True, with_stats=True)
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)
    assert sum(st["path_kind"] == 6 for st in stats) >= 250 and total["sweep_ms"] > 0


def test_long_reads_and_synth_tables():
    probs, limits = random_list(1002, 24, row_limits=(16, 256), mean_len=30.0)
    probs += [synth.sliding_window(600, c, block_len=300, seed=s) for s, c in ((1, 20), (2, 30))]
    limits += [256, 64]
    got = _lib.heuristic_batch(probs, limits, True)
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)


def test_an_overflowing_table_and_a_table_without_mutations_leave_the_others_alone():
    probs, limits = random_list(1003, 20)
    rng = np.random.default_rng(1004)
    ties = synth.random_problem(rng, 30, 9, pedigree="trio", distrust=True, mean_len=6.0)
    ties.ent_phred = np.zeros_like(ties.ent_phred)  # every row ties at the optimum: the row buffers overflow
    ties.recombcost = np.maximum(ties.recombcost, 1).astype(np.uint32)
    probs[5], limits[5] = ties, 2
    allow = [t != 11 for t in range(len(probs))]
    limits[11] = 1
    got, (stats, _) = _lib.heuristic_batch(probs, limits, allow, with_stats=True)
    for t, (p, rl, am, g) in enumerate(zip(probs, limits, allow, got)):
        assert_same(g, alone(p, rl, am), t)
    assert stats[5]["path_kind"] == 0 and stats[11]["path_kind"] == 0
    assert sum(st["path_kind"] == 6 for st in stats) >= 15


def test_several_groups_under_the_arena_hook(monkeypatch):
    probs, limits = random_list(1005, 40, row_limits=(16, 256))
    monkeypatch.setenv("WHMEC_HEURISTIC_ARENA_BUDGET", str(1 << 20))
    got, (stats, total) = _lib.heuristic_batch(probs, limits, True, with_stats=True)
    assert total["kernel_launches"] > 2
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)


def test_batch_classmethod_equals_constructed_tables():
    items = constructor_args(1006) + constructor_args(1007)
    objs = core.PedMecHeuristic.batch([args for _, args in items])
    for (_, args), obj in zip(items, objs):
        assert isinstance(obj, core.PedMecHeuristic) and same_answers(obj, core.PedMecHeuristic(*args))
    rs, recomb, ped = items[1][1][:3]
    no_mutations = (rs, recomb, ped, 1, False, None, False)
    out = core.PedMecHeuristic.batch([items[0][1], no_mutations], return_exceptions=True)
    try:
        want = core.PedMecHeuristic(*no_mutations)
    except Exception as e:  # noqa: BLE001
        assert type(out[1]) is type(e) and str(out[1]) == str(e)
    else:
        assert same_answers(out[1], want)
    assert same_answers(out[0], core.PedMecHeuristic(*items[0][1]))


def test_swap_in_class_batch():
    cls = adapters.make_heuristic_class(core)
    items = constructor_args(1008)
    for (_, args), obj in zip(items, cls.batch([args for _, args in items])):
        assert same_answers(obj, cls(*args))
