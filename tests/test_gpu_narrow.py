"""Narrow steady-state panels on the GPU (DESIGN §4.1): the 16-bit halfword-pair sweep against the 32-bit one
(WHMEC_TILE_NARROW=0) and against the reference -- cfg3-shaped tables, tie-heavy weights, the stored coverage 21-25 answers,
memory-bounded sweeps and one batch.  test_narrow_emulation.py holds the same code to the 32-bit columns without a GPU."""
import pytest

import golden_io
from whatshap_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ENV = ("WHMEC_TILE_NARROW", "WHMEC_TILE_MIRROR", "WHMEC_TILE_PACKED_BP", "WHMEC_PINNED_UPLOAD", "WHMEC_TILE_ARENA_BUDGET",
           "WHMEC_FORCE_COLUMN_KERNEL", "WHMEC_SOLVE_GROUPS")


def set_switch(monkeypatch, env):
    for k in ALL_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def both_paths(gpu, monkeypatch, prob, env=None):
    set_switch(monkeypatch, dict(env or {}))
    narrow, st = gpu.solve(prob)
    set_switch(monkeypatch, dict(env or {}, WHMEC_TILE_NARROW="0"))
    wide, st_wide = gpu.solve(prob)
    assert st["path_kind"] == 1 and st_wide["path_kind"] == 1, (st, st_wide)
    return narrow, wide, st


CFG3_SHAPES = [
    dict(n=3000, c=20, block_len=500, seed=1),
    dict(n=3000, c=20, block_len=500, seed=2, max_phred=2),   # ties everywhere
    dict(n=2000, c=20, block_len=2000, seed=3, gap=0.05),
    dict(n=2000, c=18, block_len=1000, seed=4, max_phred=3),
]


@pytest.mark.parametrize("shape", range(len(CFG3_SHAPES)))
def test_narrow_sweep_equals_the_32_bit_sweep(gpu, monkeypatch, shape):
    kw = CFG3_SHAPES[shape]
    prob = synth.sliding_window(kw["n"], kw["c"], block_len=kw["block_len"], seed=kw["seed"], gap=kw.get("gap", 0.0),
                                max_phred=kw.get("max_phred", 40))
    narrow, wide, _ = both_paths(gpu, monkeypatch, prob)
    assert narrow.same_as(wide), (kw, narrow.diff(wide))


@pytest.mark.parametrize("seed,max_phred", [(5, 40), (6, 2)])
def test_narrow_sweep_against_the_reference(gpu, checker, monkeypatch, seed, max_phred):
    prob = synth.sliding_window(60, 20, block_len=60, seed=seed, max_phred=max_phred)
    narrow, wide, _ = both_paths(gpu, monkeypatch, prob)
    want = checker.solve(prob)
    assert narrow.same_as(want), narrow.diff(want)
    assert wide.same_as(want), wide.diff(want)


def test_stored_coverage_21_to_25_answers(gpu, monkeypatch):
    for label, prob, want, _ in golden_io.load("high_coverage"):
        narrow, wide, _ = both_paths(gpu, monkeypatch, prob)
        assert narrow.same_as(want), (label, narrow.diff(want))
        assert wide.same_as(want), (label, wide.diff(want))


@pytest.mark.parametrize("divisor", [2, 5])
def test_memory_bounded_narrow_sweeps(gpu, monkeypatch, divisor):
    """An arena of 1/2 and 1/5 of the resident back-pointers: segments of rounds, re-swept from checkpoints in the backtrace."""
    prob = synth.sliding_window(2000, 20, block_len=2000, seed=7)
    set_switch(monkeypatch, {})
    resident_sol, st = gpu.solve(prob)
    resident = st["backptr_bytes"]
    narrow, wide, st = both_paths(gpu, monkeypatch, prob, {"WHMEC_TILE_ARENA_BUDGET": str(resident // divisor)})
    assert st["kernel_launches"] > 1 and st["backptr_bytes"] < resident, st
    assert narrow.same_as(wide), narrow.diff(wide)
    assert narrow.same_as(resident_sol), narrow.diff(resident_sol)


def test_one_batch_of_narrow_tables(gpu, monkeypatch):
    """Several cfg3-shaped tables in one whmec_solve_batch call (one persistent launch) against their 32-bit single solves."""
    probs = [synth.sliding_window(1500, 20, block_len=500, seed=20 + i, max_phred=(2 if i % 2 else 40)) for i in range(4)]
    probs.insert(2, synth.sliding_window(60, 17, block_len=30, seed=17))
    set_switch(monkeypatch, {"WHMEC_TILE_NARROW": "0"})
    wants = [gpu.solve(p)[0] for p in probs]
    set_switch(monkeypatch, {})
    out, (stats, total) = gpu.solve_batch(probs, with_stats=True)
    for i, (got, want) in enumerate(zip(out, wants)):
        assert not isinstance(got, Exception), (i, got)
        assert got.same_as(want), (i, got.diff(want))
    assert total["kernel_launches"] == 1, total
