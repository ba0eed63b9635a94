"""The tile kernel at coverage 21-25 against the reference's stored answers (tests/golden/high_coverage.npz): the small-chunk
hand-off (chunks under 128 bytes gathered element by element into the staging buffer) into steady and non-steady panels,
mirrored with km = 0 and km != 0 and unmirrored, the last bulk-copy shape at coverage 21, many chains of one persistent launch
waiting on each other's panels only, segments re-swept from their checkpoints, and the renumbered state offsets of a union
of tables.  Bit for bit, ties included.  test_high_coverage_golden.py checks without a GPU that the instances reach these paths.
The reference is never run here: it needs minutes for these instances."""
import sys

import pytest

import golden_io
from whatshap_b200 import synth

sys.path.insert(0, golden_io.HERE)
import make_high_coverage_golden as gen  # noqa: E402

pytestmark = pytest.mark.gpu

SWITCHES = {
    "default": {},
    "mirror_off": {"WHMEC_TILE_MIRROR": "0"},
    "ballot_bp": {"WHMEC_TILE_PACKED_BP": "0"},  # no steady panels: the generic column loops behind the same hand-offs
    "pageable_upload": {"WHMEC_PINNED_UPLOAD": "0"},
}
ALL_ENV = ("WHMEC_TILE_MIRROR", "WHMEC_TILE_PACKED_BP", "WHMEC_PINNED_UPLOAD", "WHMEC_TILE_ARENA_BUDGET", "WHMEC_FORCE_COLUMN_KERNEL",
           "WHMEC_SOLVE_GROUPS")
BOUNDED = ("sliding/n=80/c=21", "sliding/n=80/c=22", "sliding/n=80/c=23", "ragged/n=600/c=22/mean=60")
RAGGED = "ragged/n=600/c=22/mean=60"

_golden = []


def golden():
    if not _golden:
        _golden.extend((label, prob, want) for label, prob, want, _ in golden_io.load("high_coverage"))
    return _golden


def by_label(label):
    return next((prob, want) for lb, prob, want in golden() if lb == label)


def set_switch(monkeypatch, env):
    for k in ALL_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("switch", list(SWITCHES))
def test_stored_answers_under_the_kernel_switches(gpu, monkeypatch, switch):
    set_switch(monkeypatch, SWITCHES[switch])
    for label, prob, want in golden():
        got, stats = gpu.solve(prob)
        assert got.same_as(want), (switch, label, stats, got.diff(want))
        assert stats["path_kind"] == 1 and stats["max_active"] == int(gen.active_reads(prob).max()), (label, stats)


@pytest.mark.parametrize("divisor", [2, 4])
@pytest.mark.parametrize("label", BOUNDED)
def test_memory_bounded_sweeps(gpu, monkeypatch, label, divisor):
    """An arena of 1/2 and 1/4 of the resident back-pointers: segments of rounds, re-swept from checkpoints in the backtrace."""
    set_switch(monkeypatch, {})
    prob, want = by_label(label)
    resident = gpu.solve(prob)[1]["backptr_bytes"]
    monkeypatch.setenv("WHMEC_TILE_ARENA_BUDGET", str(resident // divisor))
    got, stats = gpu.solve(prob)
    assert got.same_as(want), (label, divisor, stats, got.diff(want))
    assert stats["path_kind"] == 1 and stats["kernel_launches"] > 1 and stats["backptr_bytes"] < resident, stats


def test_one_batch_of_all_stored_tables(gpu, checker, monkeypatch):
    """All stored tables in one whmec_solve_batch call, behind a one-read table and with a coverage-17 table between them:
    one persistent launch sweeps the union, whose state buffers are renumbered (and moved off their single-table alignment)."""
    set_switch(monkeypatch, {})
    one_read = synth.sliding_window(2, 2, block_len=2, seed=5)
    assert one_read.n_reads == 1
    cov17 = synth.sliding_window(60, 17, block_len=30, seed=17)
    tables = [(label, prob, want) for label, prob, want in golden()]
    items = [("one_read", one_read, checker.solve(one_read))] + tables[:3] + [("cov17", cov17, checker.solve(cov17))] + tables[3:]
    out, (stats, total) = gpu.solve_batch([p for _, p, _ in items], with_stats=True)
    for (label, _, want), got, st in zip(items, out, stats):
        assert not isinstance(got, Exception), (label, got)
        assert got.same_as(want), (label, got.diff(want))
        assert st["path_kind"] == 1, (label, st)
    assert total["kernel_launches"] == 1, total


def test_plan_swept_twice_on_many_chains(gpu, monkeypatch):
    set_switch(monkeypatch, {})
    prob, want = by_label(RAGGED)
    plan = gpu.Plan(prob)
    try:
        plan.sweep()
        first = plan.finish()
        st = plan.stats()
        plan.sweep()
        second = plan.finish()
    finally:
        plan.close()
    assert (st["path_kind"], st["kernel_launches"]) == (1, 1), st
    assert st["n_chains"] >= 10, st
    assert first.same_as(want), first.diff(want)
    assert second.same_as(want), second.diff(want)
