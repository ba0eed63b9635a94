"""Many heuristic tables in one call (`whmec_heuristic_batch`, `PedMecHeuristic.batch`, DESIGN §4.10), without a GPU.

The host emulation (tests/emul_heuristic_batch.py) runs the batch's host plan and the sweep of heuristic_device.h, the very code
the kernel runs, with every phase's rows in a seeded random order.  Every table must equal `whmec_heuristic` (the host solver)
on it alone, bit for bit in every output field; tables the device cannot take, and tables it hands back, run `whmec_heuristic`
inside the call."""
import numpy as np
import pytest

import emul_heuristic_batch as eb
from test_heuristic import golden_cases
from whatshap_b200 import _lib, adapters, core, multigpu, synth
from whatshap_b200._abi import FlatProblem, Unsupported

SHAPES = ("single", "trio", "quartet", "three_generations", "two_unrelated", "trio_child_first")


def alone(prob, row_limit, allow=True):
    try:
        return _lib.heuristic(prob, row_limit, allow)
    except Exception as e:  # noqa: BLE001 - compared with the batch's entry
        return e


def assert_same(got, want, label=None):
    if isinstance(want, Exception):
        assert type(got) is type(want) and str(got) == str(want), (label, got, want)
    else:
        assert not isinstance(got, Exception), (label, got)
        assert got.same_as(want) and got.score == want.score, label


def random_list(seed, count, row_limits=(1, 2, 16, 256), mean_len=None, max_phred=None):
    rng = np.random.default_rng(seed)
    probs, limits = [], []
    for i in range(count):
        prob = synth.random_problem(rng, int(rng.integers(2, 60)), int(rng.integers(2, 9)), pedigree=SHAPES[i % len(SHAPES)],
                                    distrust=bool(rng.integers(0, 2)), max_phred=max_phred or int(rng.choice([3, 10, 40])),
                                    mean_len=mean_len or float(rng.choice([2.0, 5.0])))
        prob.recombcost = np.maximum(prob.recombcost, 1).astype(np.uint32)
        probs.append(prob)
        limits.append(int(rng.choice(row_limits)))
    return probs, limits


def test_golden_vectors_in_one_call():
    cases = list(golden_cases())
    probs, limits = [c[1] for c in cases], [c[2] for c in cases]
    for seed in (1, 2):
        got, info = eb.heuristic_batch(probs, limits, True, seed=seed)
        assert len(got) == 60 and info["groups"] == 1
        assert sum(g >= 0 for g in info["group_of"]) == 60  # every golden table reaches the sweep
        for (i, prob, row_limit, want, n_samples), g in zip(cases, got):
            assert_same(g, _lib.heuristic(prob, row_limit, True), i)
            assert np.array_equal(g.partition, want["partition"]) and np.array_equal(g.haplotypes[:n_samples], want["haplotypes"]), i


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_random_mixed_lists(seed):
    probs, limits = random_list(seed, 40)
    got, info = eb.heuristic_batch(probs, limits, True, seed=seed)
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), (seed, t))
    assert sum(g >= 0 for g in info["group_of"]) >= 30


def test_long_reads_make_wide_windows():
    probs, limits = random_list(21, 16, row_limits=(16, 256), mean_len=30.0)
    got, _ = eb.heuristic_batch(probs, limits, True, seed=5)
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)


def test_synth_shaped_single_sample_tables():
    probs = [synth.sliding_window(120, c, block_len=60, seed=s, max_phred=40) for s, c in ((1, 8), (2, 12), (3, 6))]
    got, _ = eb.heuristic_batch(probs, [256, 16, 2], True, seed=9)
    for p, rl, g in zip(probs, [256, 16, 2], got):
        assert_same(g, alone(p, rl))


def test_tie_heavy_tables_hand_back_overflowing_ones():
    """Phreds of 1 make many rows tie; phreds of 0 with distrusted genotypes make every placement useful and every row tie at
    the optimum.  All optimal rows are kept (heuristic.cpp: prune), which outgrows the row buffers: such a table is handed back
    to `whmec_heuristic`, and still equals it."""
    probs, limits = random_list(31, 24, row_limits=(1, 2), max_phred=1)
    rng = np.random.default_rng(32)
    for k in range(6):
        prob = synth.random_problem(rng, 30, 9, pedigree=SHAPES[k % 2], distrust=True, mean_len=6.0)
        prob.ent_phred = np.zeros_like(prob.ent_phred)
        prob.recombcost = np.maximum(prob.recombcost, 1).astype(np.uint32)
        probs.append(prob)
        limits.append(int(rng.choice([1, 2, 16])))
    got, info = eb.heuristic_batch(probs, limits, True, seed=4)
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)
    assert 0 < info["handed_back"] <= 6


def bad_tables():
    """(problem, row_limit, allow_mutations) of tables that fail, each with the error `whmec_heuristic` gives it."""
    rng = np.random.default_rng(5)
    base = synth.random_problem(rng, 12, 4, pedigree="trio")
    base.recombcost = np.maximum(base.recombcost, 1).astype(np.uint32)
    unsorted = synth.random_problem(rng, 12, 4)
    unsorted.read_off = np.array(unsorted.read_off)
    order = np.arange(unsorted.n_reads)[::-1]
    starts, ends = unsorted.read_off[:-1][order], unsorted.read_off[1:][order]
    unsorted = FlatProblem(positions=unsorted.positions, read_off=np.concatenate([[0], np.cumsum(ends - starts)]).astype(np.uint64),
                           ent_col=np.concatenate([unsorted.ent_col[s:e] for s, e in zip(starts, ends)]),
                           ent_allele=np.concatenate([unsorted.ent_allele[s:e] for s, e in zip(starts, ends)]),
                           ent_phred=np.concatenate([unsorted.ent_phred[s:e] for s, e in zip(starts, ends)]),
                           read_ind=unsorted.read_ind, recombcost=unsorted.recombcost, n_ind=1, distrust=False, gt=unsorted.gt)
    no_gt = synth.random_problem(rng, 12, 4)
    no_gt.gt = np.full_like(no_gt.gt, 255)
    many = synth.random_problem(rng, 6, 3)
    many = FlatProblem(positions=many.positions, read_off=many.read_off, ent_col=many.ent_col, ent_allele=many.ent_allele,
                       ent_phred=many.ent_phred, read_ind=many.read_ind, recombcost=many.recombcost, n_ind=48,
                       trios=np.array([[2 * k + 1, 2 * k + 2, 0] for k in range(16)], np.uint32).ravel(), distrust=False,
                       gt=np.ones((48, many.n_cols), np.uint8))
    outside = synth.random_problem(rng, 12, 4)
    outside.read_ind = (np.arange(outside.n_reads) % 2 * 5).astype(np.uint32)  # two samples, one individual
    return [(unsorted, 16, True), (no_gt, 16, True), (many, 16, True), (outside, 16, True), (base, 16, False)]


def test_errors_are_per_table_and_leave_the_neighbours_solved():
    bad = bad_tables()
    probs, limits, allow = [], [], []
    ok_probs, ok_limits = random_list(41, len(bad))
    for (p, rl, am), q, ql in zip(bad, ok_probs, ok_limits):
        probs += [q, p]
        limits += [ql, rl]
        allow += [True, am]
    got, info = eb.heuristic_batch(probs, limits, allow, seed=6)
    for t, (p, rl, am, g) in enumerate(zip(probs, limits, allow, got)):
        want = alone(p, rl, am)
        assert_same(g, want, t)
        if t % 2:  # (allow_mutations = False is solved, by whmec_heuristic)
            assert info["group_of"][t] == -1 and (t == 9 or isinstance(g, Exception))
    assert isinstance(got[1], RuntimeError) and "sorted" in str(got[1])
    assert isinstance(got[5], Unsupported) and "15 trio" in str(got[5])
    assert isinstance(got[7], RuntimeError) and "zero-based" in str(got[7])


def test_c_abi_without_a_device():
    """Tables that never reach the device need none: errors, allow_mutations = False, a table without reads."""
    bad = bad_tables()
    empty = FlatProblem(positions=np.zeros(3, np.uint32), read_off=[0], ent_col=[], ent_allele=[], ent_phred=[], read_ind=[],
                        recombcost=[1, 1, 1], n_ind=1, distrust=False, gt=np.ones((1, 3), np.uint8))
    probs = [p for p, _, _ in bad] + [empty]
    out = _lib.heuristic_batch(probs, [rl for _, rl, _ in bad] + [8], [am for _, _, am in bad] + [True])
    for (p, rl, am), g in zip(bad, out):
        assert_same(g, alone(p, rl, am))
    assert_same(out[-1], alone(empty, 8))
    assert _lib.heuristic_batch([]) == []
    with pytest.raises(ValueError):
        _lib.heuristic_batch(probs, [1, 2], True)
    if _lib.device_count() == 0:
        with pytest.raises(RuntimeError, match="CUDA"):
            _lib.heuristic_batch([random_list(3, 1)[0][0]])


def test_groups_under_a_small_budget():
    probs, limits = random_list(51, 24, row_limits=(16, 256))
    _, whole = eb.heuristic_batch(probs, limits, True, seed=1)
    assert whole["groups"] == 1
    got, info = eb.heuristic_batch(probs, limits, True, budget=1 << 20, seed=2)
    assert info["groups"] > 2
    for t, (p, rl, g) in enumerate(zip(probs, limits, got)):
        assert_same(g, alone(p, rl), t)
    # longest first: the group of a table never comes after that of a table with less work (columns x row_limit)
    work = [p.n_cols * rl for p, rl in zip(probs, limits)]
    grouped = [t for t in range(len(probs)) if info["group_of"][t] >= 0]
    for a in grouped:
        for b in grouped:
            if work[a] > work[b]:
                assert info["group_of"][a] <= info["group_of"][b]
    tiny, info = eb.heuristic_batch(probs[:4], limits[:4], True, budget=4096, seed=3)  # fits no group: whmec_heuristic
    assert info["groups"] == 0 and all(g == -1 for g in info["group_of"])
    for p, rl, g in zip(probs, limits, tiny):
        assert_same(g, alone(p, rl))


def test_tables_go_to_devices_by_work_and_come_back_in_input_order(monkeypatch):
    probs, _ = random_list(61, 5)
    limits = [2, 256, 16, 1, 8]
    calls = []
    index = {id(p): i for i, p in enumerate(probs)}

    def fake_batch(problems, row_limits=256, allow_mutations=True, device=0, with_stats=False):
        ids = [index[id(p)] for p in problems]
        assert list(row_limits) == [limits[i] for i in ids] and list(allow_mutations) == [i != 3 for i in ids]
        calls.append((device, ids))
        return [("done", i, device) for i in ids], ([{"device": device} for _ in problems], {})

    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.setattr(_lib, "heuristic_batch", fake_batch)
    monkeypatch.setattr(_lib, "device_count", lambda: 4)
    allow = [i != 3 for i in range(5)]
    out = multigpu.heuristic_tables(probs, limits, allow, devices=[2, 1])
    assert [o[1] for o in out] == list(range(len(probs)))
    by_device = dict(calls)
    assert sorted(by_device) == [1, 2] and sorted(by_device[1] + by_device[2]) == list(range(len(probs)))
    heaviest = int(np.argmax([p.n_cols * rl for p, rl in zip(probs, limits)]))
    assert by_device[next(d for d, ids in calls if heaviest in ids)][0] == heaviest
    calls.clear()
    out, stats = multigpu.heuristic_tables(probs, limits, allow, device=1, with_stats=True)
    assert [o[2] for o in out] == [1] * len(probs) and stats[0] == {"device": 1}
    monkeypatch.setenv(multigpu.ENV_DEVICES, "0,3")
    calls.clear()
    multigpu.heuristic_tables(probs, limits, allow)
    assert sorted(d for d, _ in calls) == [0, 3]
    calls.clear()
    assert multigpu.heuristic_tables(probs[:1], limits[:1], True, devices=[3, 0])[0][2] == 3
    assert multigpu.heuristic_tables([]) == []
    with pytest.raises(ValueError):
        multigpu.heuristic_tables(probs, [1], True)


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    monkeypatch.setattr(_lib, "heuristic_batch", lambda problems, row_limits=256, allow_mutations=True, device=0, with_stats=False: (
        lambda r: (r, ([{"path_kind": 6} for _ in problems], {})) if with_stats else r)(
            eb.heuristic_batch(problems, row_limits, allow_mutations, seed=device)[0]))


def constructor_args(seed):
    rng = np.random.default_rng(seed)
    out = []
    for k, shape in enumerate(("single", "trio", "quartet", "single", "three_generations")):
        prob = synth.random_problem(rng, int(rng.integers(3, 30)), 5, pedigree=shape, max_phred=20)
        prob.recombcost = np.maximum(prob.recombcost, 1).astype(np.uint32)
        rs, recomb, ped = synth.to_objects(prob)
        args = (rs, recomb, ped)
        if k % 2:
            args += (int(rng.choice([2, 16])), bool(k == 3), prob.positions.tolist())
        out.append((prob, args))
    return out


def same_answers(a, b):
    sa, sb = a.get_super_reads(), b.get_super_reads()
    return (sa[1] == sb[1] and [[[v.allele for v in r] for r in rs] for rs in sa[0]] == [[[v.allele for v in r] for r in rs] for rs in sb[0]]
            and a.get_optimal_partitioning() == b.get_optimal_partitioning() and a.get_mutations() == b.get_mutations()
            and a.get_optimal_cost() == b.get_optimal_cost())


def test_batch_classmethod_equals_constructed_tables(emulated):
    items = constructor_args(71)
    objs = core.PedMecHeuristic.batch([args for _, args in items])
    for (prob, args), obj in zip(items, objs):
        assert isinstance(obj, core.PedMecHeuristic) and same_answers(obj, core.PedMecHeuristic(*args))
        assert obj.stats == {"path_kind": 6}
    assert core.PedMecHeuristic.batch([]) == []


def test_batch_classmethod_reports_the_first_failing_table(emulated):
    items = constructor_args(72)
    rs, recomb, ped = items[1][1][:3]
    no_mutations = (rs, recomb, ped, 1, False, None, False)
    tables = [items[0][1], (rs, recomb, "not a pedigree"), no_mutations, items[2][1]]
    with pytest.raises(TypeError, match="'pedigree'"):
        core.PedMecHeuristic.batch(tables)
    out = core.PedMecHeuristic.batch(tables, return_exceptions=True)
    with pytest.raises(Unsupported) as e:
        core.PedMecHeuristic(*no_mutations)
    assert isinstance(out[1], TypeError) and type(out[2]) is type(e.value) and str(out[2]) == str(e.value)
    assert same_answers(out[0], core.PedMecHeuristic(*items[0][1])) and same_answers(out[3], core.PedMecHeuristic(*items[2][1]))


def test_swap_in_class_batch(emulated):
    cls = adapters.make_heuristic_class(core)
    items = constructor_args(73)
    objs = cls.batch([args for _, args in items])
    for (prob, args), obj in zip(items, objs):
        assert same_answers(obj, cls(*args))
    bad = (items[0][1][0], items[0][1][1], None)
    out = cls.batch([items[0][1], bad], return_exceptions=True)
    assert same_answers(out[0], cls(*items[0][1])) and isinstance(out[1], Exception)
    with pytest.raises(type(out[1])):
        cls.batch([items[0][1], bad])

