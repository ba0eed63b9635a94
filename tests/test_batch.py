"""Several tables in one call (whmec_solve_batch) without a GPU.  The host code that forms a tile group -- the union of the
tables' schedules and the cut of a list of tables into groups that fit the device memory -- is the product's; a TEST-ONLY
harness (tests/emul/emul_batch.cpp) sweeps the union with the emulated schedule (work items in a seeded random order that
respects only the completion counters, from a poisoned state buffer), so a chain, panel or buffer of one table that
leaked into another shows up as a wrong result.  Input errors, the Python interface and the assignment of tables to
devices are checked through the library itself."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import golden_io
from whatshap_b200 import _lib, multigpu, synth
from whatshap_b200._abi import CProblem, CSolution, FlatSolution, MendelianConflict

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
LIBS = ("libwhemul_batch.so", "libwhemul_batch_small.so")  # tiles of 2^14 and of 2^4 entries


@pytest.fixture(scope="module")
def emul():
    subprocess.run(["make", "-C", EMUL_DIR, "-f", "batch.mk"], check=True, capture_output=True)
    libs = {}
    for name in LIBS:
        lib = C.CDLL(os.path.join(EMUL_DIR, name))
        lib.whemul_batch_solve.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(CSolution)), C.c_uint32, C.c_uint64,
                                           C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
        u64p, u32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
        lib.whemul_cut_groups.argtypes = [u64p, u64p, C.c_uint32, C.c_uint64, u32p, u32p, u32p]
        lib.whemul_cut_groups.restype = C.c_uint32
        lib.whemul_table_bytes.argtypes = [C.POINTER(CProblem), u64p]
        libs[name] = lib
    return libs


def run_group(lib, problems, seed=1):
    """(solutions, status, info) of the tables swept as one emulated tile group."""
    n = len(problems)
    sols = [FlatSolution(p.n_cols, p.n_reads, p.n_ind) for p in problems]
    cps, css = [p.as_c() for p in problems], [s.as_c() for s in sols]
    pp = (C.POINTER(CProblem) * n)(*[C.pointer(c) for c in cps])
    sp = (C.POINTER(CSolution) * n)(*[C.pointer(c) for c in css])
    status, info = (C.c_int * n)(), (C.c_uint64 * 4)()
    broken = lib.whemul_batch_solve(pp, sp, n, seed, status, info)
    assert broken == 0, "invariant %d of the union's schedule is broken" % broken
    for s, c in zip(sols, css):
        s.cost = int(c.cost)
    return sols, list(status), dict(zip(("tables", "chains", "panels", "items"), (int(v) for v in info)))


def cut(lib, sizes, items, budget):
    n = len(sizes)
    groups, alone, n_alone = (C.c_uint32 * (2 * n + 2))(), (C.c_uint32 * (n + 1))(), C.c_uint32()
    g = lib.whemul_cut_groups((C.c_uint64 * n)(*sizes), (C.c_uint64 * n)(*items), n, budget, groups, alone, C.byref(n_alone))
    return [(groups[2 * i], groups[2 * i + 1]) for i in range(g)], [alone[i] for i in range(n_alone.value)]


def test_groups_are_consecutive_and_fit_one_budget(emul):
    lib = emul[LIBS[0]]
    assert cut(lib, [], [], 100) == ([], [])
    assert cut(lib, [10, 20, 30], [1, 1, 1], 100) == ([(0, 3)], [])
    assert cut(lib, [60, 50, 40, 70], [1, 1, 1, 1], 100) == ([(0, 1), (1, 3), (3, 4)], [])
    # a table that does not fit alone takes the single-table path and closes the group in front of it
    assert cut(lib, [10, 500, 20, 30], [1, 1, 1, 1], 100) == ([(0, 1), (2, 4)], [1])
    assert cut(lib, [500], [1], 100) == ([], [0])
    # work items of a union are numbered in 32 bits
    assert cut(lib, [1, 1, 1], [1 << 30, 1 << 30, 1 << 30], 100) == ([(0, 1), (1, 2), (2, 3)], [])
    assert cut(lib, [1, 1], [1 << 31, 5], 100) == ([(1, 2)], [0])


def test_device_bytes_of_a_table(emul):
    lib = emul[LIBS[0]]
    out = (C.c_uint64 * 2)()
    assert lib.whemul_table_bytes(C.byref(synth.sliding_window(0, 4).as_c()), out) == 0 and list(out) == [0, 0]
    sizes = []
    for n in (100, 200, 400):
        assert lib.whemul_table_bytes(C.byref(synth.sliding_window(n, 10, block_len=50, seed=1).as_c()), out) == 0
        sizes.append((int(out[0]), int(out[1])))
    assert sizes[0][0] < sizes[1][0] < sizes[2][0] and sizes[2][1] == 4 * sizes[0][1] > 0


@pytest.mark.parametrize("libname", LIBS)
def test_emulated_tile_group_on_golden_vectors(emul, libname):
    """Every run of 8 single-individual golden tables as one group: each table's golden answer, the numbering of the union."""
    lib = emul[libname]
    cases = [(label, prob, want) for group in golden_io.GROUPS for label, prob, want, error in golden_io.load(group)
             if prob.n_ind == 1 and want is not None]
    assert len(cases) > 30
    solved = 0
    for lo in range(0, len(cases), 8):
        chunk = cases[lo:lo + 8]
        sols, status, info = run_group(lib, [c[1] for c in chunk], seed=lo + 1)
        assert info["tables"] == status.count(0)
        for (label, prob, want), got, st in zip(chunk, sols, status):
            assert st in (0, 100), (label, st)  # 100: no columns / the tile planner declines (single-table path in the product)
            if st == 0:
                assert got.same_as(want), (label, got.diff(want))
                solved += 1
    assert solved > 30


@pytest.mark.parametrize("mirror", ["1", "0"])
def test_emulated_group_of_ragged_tie_heavy_tables(emul, checker, monkeypatch, mirror):
    """Odd and even coverages side by side (the mirror constant km differs), weights that tie everywhere, a table of one chain
    between tables of many, a table without columns and one with a Mendelian conflict in the middle of the list."""
    monkeypatch.setenv("WHMEC_TILE_MIRROR", mirror)
    for libname, covs, n in ((LIBS[1], (6, 7, 8, 9, 5, 7), 120), (LIBS[0], (15, 16, 12), 40)):
        probs = []
        for i, cov in enumerate(covs):
            blocks = n if i == 1 else synth.geometric_blocks(n, 15.0, 10 + i)  # table 1: a single chain
            p = synth.sliding_window(n, cov, block_len=blocks, seed=20 + i, gap=0.1 * (i % 2), max_phred=1 + 2 * (i % 2))
            probs.append(p)
        bad = synth.sliding_window(30, 4, block_len=30, seed=3)
        bad.gt[0, 7] = 255
        probs[2:2] = [synth.sliding_window(0, 4), bad]
        sols, status, info = run_group(emul[libname], probs, seed=5)
        assert status[2] == 100 and status[3] == 1  # WHMEC_ERR_MENDELIAN: this table only
        assert info["tables"] == len(covs) and info["chains"] > len(covs)
        for i, (p, got) in enumerate(zip(probs, sols)):
            if i not in (2, 3):
                assert status[i] == 0
                want = checker.solve(p)
                assert got.same_as(want), (libname, i, got.diff(want))


def test_one_table_in_a_group_equals_the_table_alone(emul, checker):
    prob = synth.sliding_window(200, 9, block_len=synth.geometric_blocks(200, 20.0, 4), seed=4)
    (got,), status, info = run_group(emul[LIBS[1]], [prob], seed=9)
    assert status == [0] and got.same_as(checker.solve(prob))


def test_input_errors_are_per_table_and_need_no_gpu():
    """A list in which no table reaches the device: each gets the code and text whmec_solve gives it, in input order."""
    conflict = synth.sliding_window(12, 3, block_len=12, seed=1)
    conflict.gt[0, 5] = 255
    unsorted = synth.sliding_window(12, 3, block_len=12, seed=1)
    unsorted.ent_col[1], unsorted.ent_col[0] = unsorted.ent_col[0], unsorted.ent_col[1]
    trio = synth.trio(10, 2, block_len=10, seed=2)
    trio.gt[2, 3] = 255
    out, (stats, total) = _lib.solve_batch([synth.sliding_window(0, 4), conflict, unsorted, trio], with_stats=True)
    assert isinstance(out[0], FlatSolution) and out[0].cost == 0
    assert isinstance(out[1], MendelianConflict) and str(out[1]) == "Error: Mendelian conflict"
    assert isinstance(out[2], RuntimeError) and "unsorted variants" in str(out[2])
    assert isinstance(out[3], MendelianConflict)
    assert total["cells"] == 0 and total["kernel_launches"] == 0 and len(stats) == 4
    assert _lib.solve_batch([]) == []
    for single, batched in zip((conflict, unsorted), out[1:3]):
        with pytest.raises(type(batched)) as e:
            _lib.solve(single)
        assert str(e.value) == str(batched)


def test_tables_go_to_devices_by_work_and_come_back_in_input_order(monkeypatch):
    probs = [synth.sliding_window(n, c, block_len=20, seed=i) for i, (n, c) in enumerate(((40, 10), (40, 4), (200, 10), (20, 3), (60, 9)))]
    probs.append(synth.trio(20, 2, block_len=10, seed=9))
    calls = []
    index = {id(p): i for i, p in enumerate(probs)}

    def fake_batch(problems, device=0, with_stats=False):
        calls.append((device, [index[id(p)] for p in problems]))
        return [("solved", index[id(p)], device) for p in problems], ([{"device": device} for _ in problems], {})

    monkeypatch.setattr(_lib, "solve_batch", fake_batch)
    monkeypatch.setattr(_lib, "device_count", lambda: 4)
    out = multigpu.solve_tables(probs, devices=[2, 1])
    assert [o[1] for o in out] == list(range(len(probs)))
    by_device = dict(calls)
    assert sorted(by_device) == [1, 2] and sorted(by_device[1] + by_device[2]) == list(range(len(probs)))
    heavy = next(d for d, ids in calls if 2 in ids)  # the 200-column table: longest first, the other tables balance it
    assert 0 not in by_device[heavy] and all(ids == sorted(ids) for ids in by_device.values())
    calls.clear()
    assert [o[2] for o in multigpu.solve_tables(probs, devices=[3, 3])] == [3] * len(probs) and len(calls) == 1
    calls.clear()
    assert [o[2] for o in multigpu.solve_tables(probs, device=1)] == [1] * len(probs) and calls[0][0] == 1
    assert multigpu.solve_tables([]) == []


def test_batch_classmethod_reports_the_first_failing_table():
    from whatshap_b200 import NumericSampleIds, Pedigree, PedigreeDPTable
    from whatshap_b200.testhelpers import canonic_index_to_biallelic_gt, string_to_readset

    rs = string_to_readset("""
      11
      01
    """)
    ped = Pedigree(NumericSampleIds())
    ped.add_individual("individual0", [canonic_index_to_biallelic_gt(1)] * 2)
    tables = [(rs, [1, 1], "not a pedigree"), ("not a readset", [1, 1], ped)]
    with pytest.raises(TypeError, match="'pedigree'"):
        PedigreeDPTable.batch(tables)
    out = PedigreeDPTable.batch(tables, return_exceptions=True)
    assert [type(o) for o in out] == [TypeError, TypeError] and "'readset'" in str(out[1])
    assert PedigreeDPTable.batch([]) == []


# ---- fused-trio group ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def fused(emul):
    lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_fused_batch.so"))
    lib.whemul_fused_batch_solve.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(CSolution)), C.c_uint32, C.POINTER(C.c_int),
                                             C.POINTER(C.c_uint64)]
    u32p = C.POINTER(C.c_uint32)
    lib.whemul_fold_tables.argtypes = [u32p, u32p, C.c_uint32, u32p]
    lib.whemul_fold_tables.restype = None
    return lib


def run_fused_group(lib, problems):
    n = len(problems)
    sols = [FlatSolution(p.n_cols, p.n_reads, p.n_ind) for p in problems]
    cps, css = [p.as_c() for p in problems], [s.as_c() for s in sols]
    pp = (C.POINTER(CProblem) * n)(*[C.pointer(c) for c in cps])
    sp = (C.POINTER(CSolution) * n)(*[C.pointer(c) for c in css])
    status, info = (C.c_int * n)(), (C.c_uint64 * 2)()
    assert lib.whemul_fused_batch_solve(pp, sp, n, status, info) == 0
    for s, c in zip(sols, css):
        s.cost = int(c.cost)
    return sols, list(status), (int(info[0]), int(info[1]))


def fold(lib, rows, table_chain):
    rows = np.ascontiguousarray(rows, np.uint32)
    chain = np.ascontiguousarray(table_chain, np.uint32)
    out = np.full_like(rows, 0xDEADBEEF)
    u32p = C.POINTER(C.c_uint32)
    lib.whemul_fold_tables(rows.ctypes.data_as(u32p), chain.ctypes.data_as(u32p), len(chain) - 1, out.ctypes.data_as(u32p))
    return out


def test_fold_restarts_where_a_table_starts(fused):
    """Folding [A, B] with a table start at B equals folding A and B separately; without the restart B's inputs would carry A's costs."""
    rng = np.random.default_rng(3)
    a, b = rng.integers(0, 1000, (5, 4)).astype(np.uint32), rng.integers(0, 1000, (3, 4)).astype(np.uint32)
    a[2, 1] = b[1, 3] = 0xFFFFFFFF  # +infinity entries are skipped, not added
    both = fold(fused, np.concatenate([a, b]), [0, 5, 8])
    assert np.array_equal(both[:5], fold(fused, a, [0, 5])) and np.array_equal(both[5:], fold(fused, b, [0, 3]))
    assert not both[5].any() and not both[0].any()  # a table's first chain ignores its input: zeros
    as_one_table = fold(fused, np.concatenate([a, b]), [0, 8])
    assert np.array_equal(as_one_table[:5], both[:5]) and not np.array_equal(as_one_table[5:], both[5:])
    # a table of one chain between tables of many, and a table without chains
    three = fold(fused, np.concatenate([a, b[:1], b]), [0, 5, 6, 6, 9])
    assert np.array_equal(three[6:], both[5:]) and not three[5].any()


def test_emulated_fused_trio_group(fused, checker):
    """Trio tables as one union of chains: golden trios and generated ones, a table of one chain between tables of many,
    recombination costs low enough that transmission values change along the path (non-zero entries into chains), a table
    with a Mendelian conflict and a single individual in the list."""
    probs, wants = [], []
    for group in golden_io.GROUPS:
        for label, prob, want, error in golden_io.load(group):
            if prob.n_ind == 3 and prob.n_trios == 1 and want is not None and not prob.distrust and len(probs) < 6:
                probs.append(prob)
                wants.append(want)
    for i, (n, c, blocks) in enumerate(((60, 3, 12), (40, 2, 40), (90, 4, 15), (30, 3, 10))):  # the second: one chain
        p = synth.trio(n, c, block_len=blocks, seed=60 + i)
        p.recombcost[:] = (0, 3, 1, 7)[i]
        p.recombcost[0] = 0
        probs.append(p)
        wants.append(checker.solve(p))
    bad = synth.trio(30, 2, block_len=15, seed=7)
    bad.gt[:, 4] = [0, 0, 2]
    probs[3:3] = [bad, synth.sliding_window(20, 4, block_len=10, seed=1)]
    wants[3:3] = [None, None]
    sols, status, (tables, chains) = run_fused_group(fused, probs)
    assert status[3] == 1 and status[4] == 100
    solved = [i for i, st in enumerate(status) if st == 0]
    assert tables == len(solved) >= 5 and chains > tables
    for i in solved:
        assert sols[i].same_as(wants[i]), (i, sols[i].diff(wants[i]))
    assert any(sols[i].path_tv.any() for i in solved)  # transmission values other than 0 on some path
