"""Many genotyping tables in one call (`whmec_genotype_batch`, DESIGN §4.9) without a GPU: the batch plan stepped on the host
(tests/emul/emul_gl_batch.cpp, steps of different tables in random order within a launch, NaN behind the buffers)
against the emulated single-table path bit for bit and against the golden answers, the group cuts and launch counts of the
planner, per-table errors, the device assignment of `multigpu.genotype_tables` and the `batch` classmethods."""
import numpy as np
import pytest

import emul_genotype
import emul_genotype_batch as eb
from emul_genotype_bounded import genotype_bounded
from test_devices import objects_with_priors
from test_genotype import TOL_DEVICE, close, golden
from whatshap_b200 import _lib, adapters, core, multigpu, synth
from whatshap_b200._abi import FlatProblem, Unsupported

SHAPES = ("single", "trio", "trio_child_first", "quartet", "three_generations", "three_children", "four_children")


def mixed_list(seed, n_tables=14):
    """Tables of every pedigree shape, of different lengths and coverages (the largest pedigrees kept small)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_tables):
        shape = SHAPES[int(rng.integers(len(SHAPES)))] if i >= len(SHAPES) else SHAPES[i]
        big = shape in ("three_children", "four_children")
        n_cols = int(rng.integers(2, 8 if big else 40))
        cov = int(rng.integers(2, 3 if big else (9 if shape == "single" else 5)))
        out.append(synth.genotyping_problem(rng, n_cols, cov, shape, prior=("uniform", "random", "sparse")[i % 3]))
    return out


def sub_table_length(prob):
    """Columns of the longest sub-table: a single individual's longest chain, or a pedigree's whole table."""
    if prob.n_ind == 1:
        return max(hi - lo for lo, hi in multigpu.independent_blocks(prob))
    return prob.n_cols


def planned_launches(probs, group_of):
    """2 x (backward + forward steps) of the longest sub-table of every group (no group here reaches 65535 steps per launch)."""
    longest = {}
    for p, q in zip(probs, group_of):
        if q >= 0:
            longest[q] = max(longest.get(q, 0), sub_table_length(p))
    return sum(2 * ((L - 1) + L) for L in longest.values())


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_emulated_batch_equals_each_table_alone_bit_for_bit(seed):
    probs = mixed_list(seed)
    got, info = eb.genotype_batch(probs, seed=seed)
    assert info["groups"] == 1 and info["alone"] == 0
    for i, (p, g) in enumerate(zip(probs, got)):
        want, _ = emul_genotype.genotype(p)
        assert np.array_equal(g, want, equal_nan=True), (seed, i, p.n_ind, p.n_trios)
    assert info["launches"] == planned_launches(probs, info["group_of"])
    assert {p.n_trios for p in probs} == {0, 1, 2, 3, 4}


def test_golden_cases_batched_together():
    cases = list(golden())
    got, info = eb.genotype_batch([p for _, p, _, _ in cases], seed=5)
    assert info["groups"] == 1 and len(got) == 65
    for (label, prob, want, _), g in zip(cases, got):
        assert close(g, want, TOL_DEVICE), label
        assert np.array_equal(g, emul_genotype.genotype(prob)[0], equal_nan=True), label


def test_many_single_sample_tables():
    rng = np.random.default_rng(21)
    probs = [synth.genotyping_problem(rng, int(rng.integers(2, 30)), int(rng.integers(2, 7)), "single") for _ in range(120)]
    got, info = eb.genotype_batch(probs, seed=21)
    assert info["launches"] == planned_launches(probs, info["group_of"]) < sum(planned_launches([p], [0]) for p in probs)
    for p, g in zip(probs, got):
        assert np.array_equal(g, emul_genotype.genotype(p)[0], equal_nan=True)


def many_chains(n_chains, seed=0):
    """A single individual whose reads cover columns (2i, 2i + 1): n_chains chains of two columns, each a sub-table of its own."""
    rng = np.random.default_rng(seed)
    n = 2 * n_chains
    gl = rng.random((1, n, 3)) + 0.05
    return FlatProblem(positions=np.arange(1, n + 1) * 10, read_off=np.arange(0, n + 1, 2), ent_col=np.arange(n),
                       ent_allele=rng.integers(0, 2, n), ent_phred=rng.integers(5, 40, n), read_ind=np.zeros(n_chains),
                       recombcost=rng.integers(0, 30, n), n_ind=1, distrust=True, gl=gl / gl.sum(axis=2, keepdims=True))


def test_a_step_of_more_than_65535_sub_tables_is_split():
    """70000 chains in one step: every one of the 3 steps (1 backward, 2 forward) takes two launches of its kernel and of the
    rescale, 12 in all instead of the 2 x 3 of the formula without splits."""
    prob = many_chains(70000)
    (got,), info = eb.genotype_batch([prob], seed=4)
    assert info["launches"] == 2 * 2 * 3 and planned_launches([prob], [0]) == 2 * 3
    assert np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)


def test_groups_under_small_budgets_and_a_table_that_fits_none():
    probs = mixed_list(7, 16)
    big = synth.genotyping_problem(np.random.default_rng(8), 60, 5, "trio")
    probs.insert(5, big)
    costs = [eb.cost(p) for p in probs]
    whole, _ = eb.genotype_batch(probs, seed=1)
    seen = set()
    for budget in (sum(costs) + 1, sum(costs) // 3, max(costs) + 1, sorted(costs)[-2] + 1):
        got, info = eb.genotype_batch(probs, budget_doubles=budget, seed=budget)
        groups = info["group_of"]
        seen.add(info["groups"])
        members = [[t for t, q in enumerate(groups) if q == g] for g in range(info["groups"])]
        for g, ids in enumerate(members):  # consecutive, within the budget, and closed only when the next table does not fit
            assert all(groups[t] in (g, -1) for t in range(ids[0], ids[-1] + 1))
            assert sum(costs[t] for t in ids) <= budget - 1
            if g + 1 < len(members):
                assert sum(costs[t] for t in ids) + costs[members[g + 1][0]] > budget - 1
        assert info["launches"] == planned_launches(probs, groups)
        alone = [t for t, q in enumerate(groups) if q == -1]
        assert info["alone"] == len(alone) and all(costs[t] > budget - 1 for t in alone)
        for t, (p, g) in enumerate(zip(probs, got)):
            if t in alone:
                assert np.array_equal(g, genotype_bounded(p, budget)[0], equal_nan=True), (budget, t)
            else:
                assert np.array_equal(g, whole[t], equal_nan=True), (budget, t)
    assert max(seen) >= 4 and 1 in seen
    got, info = eb.genotype_batch(probs, budget_doubles=sorted(costs)[-2] + 1)
    top = int(np.argmax(costs))  # the one table above the budget: memory-bounded, the likelihoods of the resident path
    assert info["alone"] == 1 and info["group_of"][top] == -1
    assert close(got[top], emul_genotype.genotype(probs[top])[0], TOL_DEVICE)


def bad_tables():
    """(problem, expected exception type, text) for tables `whmec_genotype` refuses on the host."""
    rng = np.random.default_rng(31)
    good = synth.genotyping_problem(rng, 10, 4)
    no_priors = FlatProblem(positions=good.positions, read_off=good.read_off, ent_col=good.ent_col, ent_allele=good.ent_allele,
                            ent_phred=good.ent_phred, read_ind=good.read_ind, recombcost=good.recombcost, n_ind=1)
    single = FlatProblem(positions=[10, 20, 30], read_off=[0, 2, 3], ent_col=[0, 1, 1], ent_allele=[0, 1, 1], ent_phred=[10, 10, 10],
                         read_ind=[0, 0], recombcost=[1, 1, 1], n_ind=1, distrust=True, gl=np.full((1, 3, 3), 1 / 3.0))
    unsorted = FlatProblem(positions=[10, 20, 30], read_off=[0, 2], ent_col=[1, 0], ent_allele=[0, 1], ent_phred=[10, 10], read_ind=[0],
                           recombcost=[1, 1, 1], n_ind=1, distrust=True, gl=np.full((1, 3, 3), 1 / 3.0))
    five = FlatProblem(positions=[10, 20], read_off=[0, 2], ent_col=[0, 1], ent_allele=[0, 1], ent_phred=[10, 10], read_ind=[2],
                       recombcost=[1, 1], n_ind=7, trios=sum(([0, 1, c] for c in range(2, 7)), []),
                       distrust=True, gl=np.full((7, 2, 3), 1 / 3.0))
    wide = FlatProblem(positions=[10, 20], read_off=[0, 2], ent_col=[0, 1], ent_allele=[0, 1], ent_phred=[10, 10], read_ind=[0],
                       recombcost=[1, 1], n_ind=6, distrust=True, gl=np.full((6, 2, 3), 1 / 3.0))  # 12 founder haplotypes
    return [(no_priors, RuntimeError, "priors"), (single, RuntimeError, "single variant"), (unsorted, RuntimeError, "unsorted"),
            (five, Unsupported, "at most 4 trio relationships"), (wide, Unsupported, "founder haplotypes")]


def test_errors_are_per_table_and_leave_the_neighbours_solved():
    rng = np.random.default_rng(32)
    bad = bad_tables()
    probs, wants = [], []
    for p, typ, text in bad:
        ok = synth.genotyping_problem(rng, int(rng.integers(3, 20)), 4, SHAPES[len(probs) % 4])
        probs += [ok, p]
        wants += [emul_genotype.genotype(ok)[0], (typ, text)]
    got, info = eb.genotype_batch(probs, seed=3)
    for g, w in zip(got, wants):
        if isinstance(w, tuple):
            assert isinstance(g, w[0]) and w[1] in str(g), (g, w)
        else:
            assert np.array_equal(g, w, equal_nan=True)
    assert info["groups"] == 1 and sum(q >= 0 for q in info["group_of"]) == len(bad)


def test_c_abi_errors_need_no_gpu():
    """A list in which no table reaches the device: each gets the code and text `whmec_genotype` gives it, in input order, and
    a table without columns gives an empty result.  With a table that needs the device and none present, the call fails."""
    bad = bad_tables()
    empty = FlatProblem(positions=np.zeros(0, np.uint32), read_off=[0], ent_col=[], ent_allele=[], ent_phred=[], read_ind=[], recombcost=[],
                        n_ind=1, distrust=True, gl=np.zeros((1, 0, 3)))
    out, (stats, total) = _lib.genotype_batch([p for p, _, _ in bad] + [empty], with_stats=True)
    for (p, typ, text), got in zip(bad, out):
        with pytest.raises(typ) as e:
            _lib.genotype(p)
        assert type(got) is type(e.value) and str(got) == str(e.value) and text in str(got)
    assert out[-1].shape == (1, 0, 3) and total["kernel_launches"] == 0 and len(stats) == len(bad) + 1
    assert _lib.genotype_batch([]) == []
    if _lib.device_count() == 0:
        with pytest.raises(RuntimeError, match="CUDA"):
            _lib.genotype_batch([bad[0][0], synth.genotyping_problem(np.random.default_rng(1), 10, 4)])


def test_one_table():
    prob = synth.genotyping_problem(np.random.default_rng(41), 30, 5, "quartet")
    (got,), info = eb.genotype_batch([prob])
    assert np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True) and info["launches"] == 2 * (2 * prob.n_cols - 1)
    assert eb.genotype_batch([]) == ([], {"groups": 0, "launches": 0, "alone": 0, "group_of": []})


def test_tables_go_to_devices_by_work_and_come_back_in_input_order(monkeypatch):
    rng = np.random.default_rng(51)
    probs = [synth.genotyping_problem(rng, n, 4, shape) for n, shape in ((20, "single"), (30, "trio"), (8, "three_children"), (40, "single"),
                                                                          (10, "quartet"))]
    calls = []
    index = {id(p): i for i, p in enumerate(probs)}

    def fake_batch(problems, device=0, with_stats=False):
        calls.append((device, [index[id(p)] for p in problems]))
        return [("done", index[id(p)], device) for p in problems], ([{"device": device} for _ in problems], {})

    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.setattr(_lib, "genotype_batch", fake_batch)
    monkeypatch.setattr(_lib, "device_count", lambda: 4)
    out = multigpu.genotype_tables(probs, devices=[2, 1])
    assert [o[1] for o in out] == list(range(len(probs)))
    by_device = dict(calls)
    assert sorted(by_device) == [1, 2] and sorted(by_device[1] + by_device[2]) == list(range(len(probs)))
    heavy = next(d for d, ids in calls if 2 in ids)  # T = 64, P = 4: the heaviest table by far goes first and alone
    assert by_device[heavy] == [2]
    calls.clear()
    assert [o[2] for o in multigpu.genotype_tables(probs, devices=[3, 3])] == [3] * len(probs) and len(calls) == 1
    calls.clear()
    out, stats = multigpu.genotype_tables(probs, device=1, with_stats=True)
    assert [o[2] for o in out] == [1] * len(probs) and calls[0][0] == 1 and stats[0] == {"device": 1}
    monkeypatch.setenv(multigpu.ENV_DEVICES, "0,3")
    calls.clear()
    multigpu.genotype_tables(probs)
    assert sorted(d for d, _ in calls) == [0, 3]
    assert multigpu.genotype_tables([]) == []


def test_one_table_over_several_devices_is_genotype_table(monkeypatch):
    seen = []
    monkeypatch.setattr(multigpu, "genotype_table", lambda p, device=0, devices=None: seen.append(devices) or ("whole", {"devices": devices}))
    monkeypatch.setattr(_lib, "device_count", lambda: 4)
    prob = synth.genotyping_problem(np.random.default_rng(3), 10, 4, "trio")
    assert multigpu.genotype_tables([prob], devices=[0, 1]) == ["whole"] and seen == [[0, 1]]


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.setattr(_lib, "genotype", emul_genotype.genotype)
    monkeypatch.setattr(_lib, "genotype_batch", lambda problems, device=0, with_stats=False: (
        lambda r: (r, ([{"path_kind": 4} for _ in problems], {})) if with_stats else r)(eb.genotype_batch(problems, seed=device)[0]))


def constructor_args(seed, pedigree_class=None):
    rng = np.random.default_rng(seed)
    out = []
    for shape in ("single", "trio", "quartet", "single", "three_generations"):
        prob = synth.genotyping_problem(rng, int(rng.integers(3, 25)), 4, shape)
        rs, recomb, ped = objects_with_priors(prob, pedigree_class)
        out.append((prob, (ped.numeric_sample_ids, rs, recomb, ped, prob.positions.tolist())))
    return out


def same_answers(a, b, prob):
    return all(np.array_equal(a.get_genotype_likelihoods(i, k).as_vector(), b.get_genotype_likelihoods(i, k).as_vector(), equal_nan=True)
               for i in range(prob.n_ind) for k in range(prob.n_cols))


def test_batch_classmethod_equals_constructed_tables(emulated):
    items = constructor_args(61)
    objs = core.GenotypeDPTable.batch([args for _, args in items])
    for (prob, args), obj in zip(items, objs):
        assert isinstance(obj, core.GenotypeDPTable) and same_answers(obj, core.GenotypeDPTable(*args), prob)
        assert obj.stats == {"path_kind": 4}
    assert core.GenotypeDPTable.batch([]) == []


def test_batch_classmethod_reports_the_first_failing_table(emulated):
    items = constructor_args(62)
    prob, args = items[1]
    no_priors = (args[0], args[1], args[2], core.Pedigree(args[0]))
    for i in range(prob.n_ind):
        no_priors[3].add_individual(i, [core.Genotype([0, 1])] * prob.n_cols, [None] * prob.n_cols)
    tr = prob.trios.tolist()
    no_priors[3].add_relationship(tr[0], tr[1], tr[2])
    tables = [items[0][1], (args[0], "not a readset", args[2], args[3]), no_priors, items[2][1]]
    with pytest.raises(TypeError, match="'readset'"):
        core.GenotypeDPTable.batch(tables)
    out = core.GenotypeDPTable.batch(tables, return_exceptions=True)
    with pytest.raises(RuntimeError) as e:
        core.GenotypeDPTable(*no_priors)
    assert isinstance(out[1], TypeError) and type(out[2]) is type(e.value) and str(out[2]) == str(e.value)
    assert same_answers(out[0], core.GenotypeDPTable(*items[0][1]), items[0][0])
    assert same_answers(out[3], core.GenotypeDPTable(*items[2][1]), items[2][0])


def test_swap_in_class_batch(emulated):
    Recording = adapters.recording_pedigree(core.Pedigree)
    items = constructor_args(63, Recording)
    cls = adapters.make_genotype_table_class(core)
    objs = cls.batch([args for _, args in items])
    for (prob, args), obj in zip(items, objs):
        assert same_answers(obj, cls(*args), prob)
    with_solver = adapters.make_genotype_table_class(core, solver=lambda p: emul_genotype.genotype(p)[0])
    bad = (items[0][1][0], items[0][1][1], items[0][1][2], None)
    out = with_solver.batch([items[0][1], bad], return_exceptions=True)
    assert same_answers(out[0], cls(*items[0][1]), items[0][0]) and isinstance(out[1], Exception)
    with pytest.raises(type(out[1])):
        with_solver.batch([items[0][1], bad])
