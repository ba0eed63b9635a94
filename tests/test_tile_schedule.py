"""The tile kernel's schedule without a GPU.  One launch sweeps a whole segment: its CTAs claim work items from a ticket
counter, and a tile waits only until the completion counter of its producer panel (the chain's previous panel) reaches
that panel's number of tiles.  A TEST-ONLY harness (tests/emul/emul_sched.cpp) runs the work items in a seeded random
order that respects exactly those counters, starting from a poisoned state buffer; any missing dependency shows up as a
wrong result.  The planner's fields that the counters rely on are checked on their own."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import golden_io
from whatshap_b200 import synth
from whatshap_b200._abi import CProblem, CSolution, FlatSolution, raise_for

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
LIBS = ("libwhemul_sched.so", "libwhemul_sched_small.so")  # tiles of 2^14 and of 2^4 entries


@pytest.fixture(scope="module")
def sched():
    subprocess.run(["make", "-C", EMUL_DIR, "-f", "sched.mk"], check=True, capture_output=True)
    libs = {}
    for name in LIBS:
        lib = C.CDLL(os.path.join(EMUL_DIR, name))
        lib.whemul_sched_solve.argtypes = [C.POINTER(CProblem), C.POINTER(CSolution), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64),
                                           C.c_char_p, C.c_size_t]
        lib.whemul_sched_check.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_uint64)]
        libs[name] = lib
    return libs


def run_sched(lib, prob, seed, segments=1):
    """(solution, info) of the emulated schedule, or (None, None) when the planner declines the problem."""
    sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs, err, info = prob.as_c(), sol.as_c(), C.create_string_buffer(512), (C.c_uint64 * 6)()
    rc = lib.whemul_sched_solve(C.byref(cp), C.byref(cs), seed, segments, info, err, len(err))
    if rc == 100:
        return None, None
    raise_for(rc, err.value.decode())
    sol.cost = int(cs.cost)
    keys = ("items", "max_ready", "out_of_order", "canonical", "tile_major", "mirrored")
    return sol, dict(zip(keys, (int(v) for v in info)))


@pytest.mark.parametrize("libname", LIBS)
def test_out_of_order_sweep_on_golden_vectors(sched, libname):
    lib = sched[libname]
    n = 0
    for group in golden_io.GROUPS:
        for label, prob, want, error in golden_io.load(group):
            if prob.n_ind != 1 or want is None:
                continue
            got, _ = run_sched(lib, prob, seed=n + 1)
            if got is None:
                continue
            assert got.same_as(want), (label, got.diff(want))
            n += 1
    assert n > 40


@pytest.mark.parametrize("mirror", ["1", "0"])
def test_out_of_order_sweep_of_ragged_chains(sched, checker, monkeypatch, mirror):
    """The cfg3g shape at small scale (chain lengths ~ Geometric), mirrored and unmirrored panels, both hand-off layouts,
    resident and memory-bounded (segments swept again from their checkpoints during the backtrace)."""
    monkeypatch.setenv("WHMEC_TILE_MIRROR", mirror)
    seen = dict(canonical=0, tile_major=0, mirrored=0, out_of_order=0, max_ready=0)
    for libname, cov, mean, n in (("libwhemul_sched.so", 16, 12.0, 60), ("libwhemul_sched_small.so", 7, 12.0, 300),
                                  ("libwhemul_sched_small.so", 9, 30.0, 300)):
        for seed in (1, 2):
            prob = synth.sliding_window(n, cov, block_len=synth.geometric_blocks(n, mean, seed), seed=seed, gap=0.1 * (seed - 1))
            want = checker.solve(prob)
            for segments in (1, 3):
                got, info = run_sched(sched[libname], prob, seed=10 * seed + segments, segments=segments)
                assert got is not None and got.same_as(want), (libname, cov, seed, segments, got.diff(want))
                for k in seen:
                    seen[k] = max(seen[k], info[k]) if k == "max_ready" else seen[k] + info[k]
    assert seen["canonical"] > 0 and seen["tile_major"] > 0 and seen["out_of_order"] > 100 and seen["max_ready"] > 16
    assert (seen["mirrored"] > 0) == (mirror == "1")


def test_out_of_order_sweep_at_benchmark_coverage(sched, checker):
    """Coverage 18: many tiles per panel and tile-major hand-offs between them with 2^14-entry tiles."""
    prob = synth.sliding_window(40, 18, block_len=40, seed=1, gap=0.05)
    want = checker.solve(prob)
    for seed, segments in ((1, 1), (2, 4)):
        got, info = run_sched(sched["libwhemul_sched.so"], prob, seed=seed, segments=segments)
        assert got is not None and got.same_as(want), (segments, got.diff(want))
        assert info["tile_major"] > 0 and info["max_ready"] > 1


@pytest.mark.parametrize("libname", LIBS)
def test_planner_fields_behind_the_completion_counters(sched, libname):
    lib = sched[libname]
    rng = np.random.default_rng(7)
    probs = [synth.config("cfg3", 2000), synth.config("cfg3g", 3000), synth.config("cfg2", 2000), synth.config("cfg4", 120)]
    probs += [synth.sliding_window(300, int(c), block_len=synth.geometric_blocks(300, 20.0, int(s)), seed=int(s))
              for c, s in zip(rng.integers(5, 12, 4), rng.integers(1, 100, 4))]
    checked = 0
    for prob in probs:
        out = (C.c_uint64 * 2)()
        rc = lib.whemul_sched_check(C.byref(prob.as_c()), out)
        assert rc in (0, 100), rc  # 100: the planner declines (the column kernel takes such problems)
        checked += int(out[1]) if rc == 0 else 0
    assert checked > 100
