"""whmec_solve_batch on the GPU: every table of a list equals its own whmec_solve bit for bit (and the CPU checker), whether
it was swept in a tile group with other tables or solved by the single-table path inside the call; a table with an input
error fails alone; the switches that change the kernels and the memory budgets that change the grouping leave the answers
as they are; the container-object interface returns objects that behave like constructed ones."""
import numpy as np
import pytest

from whatshap_b200 import PedigreeDPTable, synth
from whatshap_b200._abi import FlatSolution, MendelianConflict

pytestmark = pytest.mark.gpu


def tile_tables(count, n=300, seed0=0):
    """Single-individual tables of mixed coverage (odd and even), chain lengths and weights (table 1: ties everywhere)."""
    covs = (12, 7, 15, 10, 16, 9, 13, 11)
    out = []
    for i in range(count):
        blocks = n if i == 2 else synth.geometric_blocks(n, 25.0, seed0 + i)  # table 2: a single chain
        out.append(synth.sliding_window(n, covs[i % len(covs)], block_len=blocks, seed=seed0 + i, gap=0.05 * (i % 3),
                                        max_phred=1 if i == 1 else 40))
    return out


def conflict_table():
    bad = synth.sliding_window(40, 5, block_len=20, seed=3)
    bad.gt[0, 7] = 255
    return bad


def assert_equals_single(gpu, checker, problems, out, check=True):
    assert len(out) == len(problems)
    for i, (p, got) in enumerate(zip(problems, out)):
        try:
            want, _ = gpu.solve(p)
        except RuntimeError as e:
            assert type(got) is type(e) and str(got) == str(e), (i, got, e)
            continue
        assert isinstance(got, FlatSolution), (i, got)
        assert got.same_as(want), (i, got.diff(want))
        if check:
            assert got.same_as(checker.solve(p)), i


def test_tile_group_equals_single_solves(gpu, checker):
    problems = tile_tables(8)
    out, (stats, total) = gpu.solve_batch(problems, with_stats=True)
    assert_equals_single(gpu, checker, problems, out)
    assert total["kernel_launches"] == 1 and total["sweep_ms"] > 0  # one persistent launch swept all eight tables
    assert [st["path_kind"] for st in stats] == [1] * 8 and all(st["sweep_ms"] == 0 for st in stats)
    singles = [gpu.solve(p)[1] for p in problems]
    for key in ("cells", "algorithmic_bytes", "n_chains", "max_active", "transmissions", "backptr_bytes"):
        assert [st[key] for st in stats] == [st[key] for st in singles], key
    assert total["cells"] == sum(st["cells"] for st in singles) and total["n_chains"] == sum(st["n_chains"] for st in singles)


def test_mixed_list_keeps_input_order_and_isolates_errors(gpu, checker):
    t1 = tile_tables(4, n=120, seed0=30)
    trio = synth.trio(60, 3, block_len=20, seed=5)
    quartet = synth.nuclear_family(40, children=2, c_per_sample=2, block_len=20, seed=6)
    broken_trio = synth.trio(30, 2, block_len=15, seed=7)
    broken_trio.gt[2, 4] = 255
    unsorted = synth.sliding_window(12, 3, block_len=12, seed=1)
    unsorted.ent_col[1], unsorted.ent_col[0] = unsorted.ent_col[0], unsorted.ent_col[1]
    distrusted = synth.random_problem(np.random.default_rng(11), 30, 5, pedigree="trio", distrust=True)
    problems = [t1[0], trio, conflict_table(), t1[1], synth.sliding_window(0, 4), quartet, t1[2], broken_trio, unsorted, t1[3], distrusted]
    out, (stats, total) = gpu.solve_batch(problems, with_stats=True)
    assert_equals_single(gpu, checker, problems, out)
    assert isinstance(out[10], FlatSolution) and total["path_kind"] == 0  # the parts of the call took different paths
    assert isinstance(out[2], MendelianConflict) and isinstance(out[7], MendelianConflict) and "unsorted" in str(out[8])
    kinds = [st["path_kind"] for st in stats]
    assert [kinds[i] for i in (0, 3, 6, 9)] == [1] * 4 and [kinds[i] for i in (2, 4, 7, 8)] == [0] * 4 and kinds[1] > 1 and kinds[5] > 1
    assert stats[1]["transmissions"] == 4 and stats[5]["transmissions"] == 16
    assert out[4].cost == 0


@pytest.mark.parametrize("switch", ["WHMEC_TILE_MIRROR=0", "WHMEC_TILE_PACKED_BP=0", "WHMEC_PED_CLUSTER=1", "WHMEC_PED_CLUSTER=2",
                                    "WHMEC_PED_FUSED=0", "WHMEC_FORCE_COLUMN_KERNEL=1"])
def test_batches_under_the_kernel_switches(gpu, checker, monkeypatch, switch):
    """cfg2-shaped tables (coverage 15, blocks of 500 columns) and cfg5-shaped trios, at test size."""
    name, value = switch.split("=")
    monkeypatch.setenv(name, value)
    cfg2 = [synth.sliding_window(600, 15, block_len=150, seed=20250915 + i) for i in range(3)]
    cfg5 = [synth.trio(200, 5, block_len=50, seed=20250915 + i) for i in range(3)]
    if name == "WHMEC_FORCE_COLUMN_KERNEL":
        cfg2 = [synth.sliding_window(80, 9, block_len=40, seed=i) for i in range(3)]
    problems = [cfg2[0], cfg5[0], cfg2[1], cfg5[1], cfg2[2], cfg5[2]]
    out, (stats, total) = gpu.solve_batch(problems, with_stats=True)
    assert_equals_single(gpu, checker, problems, out, check=False)
    assert [st["path_kind"] for st in stats][0::2] == [2 if name == "WHMEC_FORCE_COLUMN_KERNEL" else 1] * 3


def test_small_budgets_cut_the_list_into_groups_and_a_single_table(gpu, checker, monkeypatch):
    """About 240 KB per 300-column table: a 600 KB budget holds two of them, the 3000-column table (2.4 MB) is solved on its
    own -- by the memory-bounded sweep, which the same budget forces there."""
    small = [synth.sliding_window(300, 12, block_len=100, seed=40 + i) for i in range(5)]
    large = synth.sliding_window(3000, 12, block_len=100, seed=50)
    problems = small[:3] + [large] + small[3:]
    reference = [gpu.solve(p)[0] for p in problems]
    monkeypatch.setenv("WHMEC_TILE_ARENA_BUDGET", "600000")
    monkeypatch.setenv("WHMEC_COLUMN_ARENA_BUDGET", "600000")
    out, (stats, total) = gpu.solve_batch(problems, with_stats=True)
    for i, (got, want) in enumerate(zip(out, reference)):
        assert isinstance(got, FlatSolution) and got.same_as(want), (i, got)
    # groups {0, 1}, {2}, {4, 5}: one launch each, whatever the tables; the large table alone, as whmec_solve runs it under this
    # budget (groups of its chains one after the other: several launches)
    alone = gpu.solve(large)[1]
    assert alone["kernel_launches"] >= 2 and stats[3]["backptr_bytes"] == alone["backptr_bytes"]
    assert total["kernel_launches"] == 3 + alone["kernel_launches"]
    # trio tables under the column paths' budget: same answers, however the budget groups them
    trios = [synth.trio(200, 4, block_len=50, seed=8 + i) for i in range(3)]
    for got, p in zip(gpu.solve_batch(trios), trios):
        assert isinstance(got, FlatSolution) and got.same_as(gpu.solve(p)[0])
    assert out[3].same_as(checker.solve(large))


def test_batch_of_container_objects(gpu):
    problems = tile_tables(3, n=60, seed0=70) + [synth.trio(30, 2, block_len=15, seed=9)]
    tables = [synth.to_objects(p) for p in problems]
    singles = [PedigreeDPTable(*t) for t in tables]
    for kwargs in ({}, {"devices": [0, 0]}, {"device": 0}):
        got = PedigreeDPTable.batch(tables, **kwargs)
        assert [type(g) for g in got] == [PedigreeDPTable] * len(tables)
        for g, s in zip(got, singles):
            assert g.get_optimal_cost() == s.get_optimal_cost() and g.get_optimal_partitioning() == s.get_optimal_partitioning()
            (gr, gtv), (sr, stv) = g.get_super_reads(), s.get_super_reads()
            assert gtv == stv and [str(r) for r in gr] == [str(r) for r in sr]
    # a pedigree whose genotypes contradict each other, in the middle of the list
    contradiction = synth.trio(30, 2, block_len=15, seed=7)
    contradiction.gt[:, 4] = [0, 0, 2]  # both parents 0/0, the child 1/1
    rs, rc, ped = synth.to_objects(contradiction)
    with pytest.raises(MendelianConflict, match="Error: Mendelian conflict"):
        PedigreeDPTable(rs, rc, ped)
    mixed = tables[:2] + [(rs, rc, ped)] + tables[2:]
    with pytest.raises(MendelianConflict, match="Error: Mendelian conflict"):
        PedigreeDPTable.batch(mixed)
    got = PedigreeDPTable.batch(mixed, return_exceptions=True)
    assert isinstance(got[2], MendelianConflict) and str(got[2]) == "Error: Mendelian conflict"
    rest = got[:2] + got[3:]
    assert [g.get_optimal_cost() for g in rest] == [s.get_optimal_cost() for s in singles]
    # one table: the constructor's path
    (one,) = PedigreeDPTable.batch(tables[:1], devices=[0, 0])
    assert one.get_optimal_cost() == singles[0].get_optimal_cost()


def test_fused_trio_group_shares_the_launches(gpu, checker):
    """Trio tables of one call run pass 1, the fold and pass 2 once: three launches for all of them, per-table costs and paths."""
    trios = [synth.trio(n, c, block_len=b, seed=80 + i) for i, (n, c, b) in enumerate(((200, 5, 50), (60, 3, 60), (150, 4, 25), (90, 2, 10), (40, 3, 20)))]
    for i, p in enumerate(trios):
        p.recombcost[1:] = (49, 2, 0, 5, 1)[i]  # low costs: transmission values change along the path
    out, (stats, total) = gpu.solve_batch(trios, with_stats=True)
    assert_equals_single(gpu, checker, trios, out)
    assert total["kernel_launches"] == 3 and [st["path_kind"] for st in stats] == [3] * 5
    assert any(o.path_tv.any() for o in out)
    singles = [gpu.solve(p)[1] for p in trios]
    assert sum(st["kernel_launches"] for st in singles) > 3
    for key in ("cells", "n_chains", "transmissions"):
        assert [st[key] for st in stats] == [st[key] for st in singles], key
