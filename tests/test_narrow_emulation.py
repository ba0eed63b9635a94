"""Narrow steady-state panels (DESIGN §4.1): the tile kernel's 16-bit halfword-pair columns (tile_fast.h: narrow_column_body),
run thread by thread by the TEST-ONLY emulation (tests/emul/emul_narrow.cpp), against the 32-bit steady columns on the same inputs -- same values and same
back-pointer words, bit for bit, in every column of every narrow tile -- and inside the planner's bound; the planner's
census of which panels go narrow."""
import ctypes as C
import os
import subprocess

import pytest

import golden_io
from whatshap_b200 import synth
from whatshap_b200._abi import CProblem, CSolution, FlatSolution, raise_for

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


@pytest.fixture(scope="module")
def emul():
    subprocess.run(["make", "-C", EMUL_DIR, "-f", "narrow.mk"], check=True, capture_output=True)
    lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_narrow.so"))
    lib.whemul_narrow_solve.argtypes = [C.POINTER(CProblem), C.POINTER(CSolution), C.c_uint32, C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
    lib.whemul_last_narrow_stats.argtypes = [C.POINTER(C.c_int64)]
    lib.whemul_narrow_census.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_uint64)]
    return lib


@pytest.fixture(autouse=True)
def default_switches(monkeypatch):
    for name in ("WHMEC_TILE_NARROW", "WHMEC_TILE_MIRROR", "WHMEC_TILE_PACKED_BP", "WHEMUL_TILE_FAST"):
        monkeypatch.delenv(name, raising=False)


def run_tile(lib, prob):
    """Emulated tile solve; returns (solution or None when the planner declines, narrow statistics)."""
    sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs, err, npan = prob.as_c(), sol.as_c(), C.create_string_buffer(512), C.c_uint32(0)
    rc = lib.whemul_narrow_solve(C.byref(cp), C.byref(cs), 0, C.byref(npan), err, len(err))
    raw = (C.c_int64 * 6)()
    lib.whemul_last_narrow_stats(raw)
    stats = dict(zip(("columns", "value_mismatches", "bp_mismatches", "bound_violations", "max_spread", "min_slack"), raw[:]))
    if rc == 100:
        return None, stats
    raise_for(rc, err.value.decode())
    sol.cost = int(cs.cost)
    return sol, stats


def assert_exact(stats, label):
    assert stats["value_mismatches"] == 0 and stats["bp_mismatches"] == 0, (label, stats)
    assert stats["bound_violations"] == 0, (label, stats)
    if stats["columns"]:
        assert 0 <= stats["min_slack"] and stats["max_spread"] < 1 << 15, (label, stats)


def narrow_panels(lib, prob):
    """(steady panels, narrow panels) of the planner's schedule."""
    raw = (C.c_uint64 * 2)()
    rc = lib.whemul_narrow_census(C.byref(prob.as_c()), raw)
    assert rc == 0, rc
    return int(raw[0]), int(raw[1])


@pytest.mark.parametrize("cov,n,seed,max_phred", [(20, 48, 3, 40), (20, 52, 5, 2), (18, 44, 1, 40), (20, 50, 7, 3)])
def test_narrow_columns_equal_the_32_bit_columns_at_benchmark_coverage(emul, checker, cov, n, seed, max_phred):
    """cfg3-shaped chains (sliding windows, coverage 18 and 20) with random and tie-heavy (phred <= 2, 3) weights: every narrow column
    gives the values and back-pointer words of the 32-bit column, and the solve matches the reference."""
    prob = synth.sliding_window(n, cov, block_len=n, seed=seed, gap=0.05 * (seed % 2), max_phred=max_phred)
    got, stats = run_tile(emul, prob)
    assert got is not None and stats["columns"] > 20, stats
    assert_exact(stats, (cov, n, seed))
    want = checker.solve(prob)
    assert got.same_as(want), got.diff(want)


def test_narrow_switch_keeps_the_32_bit_path(emul, monkeypatch):
    """WHMEC_TILE_NARROW=0: no narrow panel, the same solution."""
    prob = synth.sliding_window(48, 20, block_len=48, seed=11)
    narrow, stats = run_tile(emul, prob)
    assert stats["columns"] > 0
    monkeypatch.setenv("WHMEC_TILE_NARROW", "0")
    wide, stats = run_tile(emul, prob)
    assert stats["columns"] == 0
    assert narrow.same_as(wide) and narrow.cost == wide.cost


@pytest.mark.parametrize("group", golden_io.GROUPS + ("high_coverage",))
def test_narrow_columns_on_stored_vectors(emul, group):
    """The golden vectors, the fuzz corpus and the coverage 21-25 instances (whichever reach narrow panels): every narrow column
    bit for bit equal to the 32-bit one, inside the bound, and the stored answers reproduced."""
    for label, prob, want, error in golden_io.load(group):
        if error or prob.n_ind != 1:
            continue
        got, stats = run_tile(emul, prob)
        assert_exact(stats, label)
        if got is not None and want is not None:
            assert got.same_as(want), (label, got.diff(want))


def test_census_of_narrow_panels(emul, monkeypatch):
    """cfg3's shape (coverage 20, 500-column blocks): the steady panels go narrow; with large weights (phred up to 2000) the
    bound does not fit 16 bits and they stay on the 32-bit columns; WHMEC_TILE_NARROW=0 turns the narrow panels off."""
    cfg3 = synth.sliding_window(3000, 20, block_len=500, seed=1)
    steady, narrow = narrow_panels(emul, cfg3)
    assert steady > 50 and narrow == steady, (steady, narrow)
    heavy = synth.sliding_window(3000, 20, block_len=500, seed=1, max_phred=2000)
    steady, narrow = narrow_panels(emul, heavy)
    assert steady > 50 and narrow == 0, (steady, narrow)
    monkeypatch.setenv("WHMEC_TILE_NARROW", "0")
    steady, narrow = narrow_panels(emul, cfg3)
    assert steady > 50 and narrow == 0
