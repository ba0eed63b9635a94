"""The tile kernel's schedule on the device: a resident sweep is ONE persistent launch whose CTAs claim work items from a
ticket counter and wait only for the producer panel of their own chain (per-panel completion counters).  The counters and
the ticket are zeroed in front of every launch, so a plan swept twice computes the same thing twice; the column kernel,
different device code with no such schedule, must agree."""
import pytest

from whatshap_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,cols", [("cfg3", 3_000), ("cfg3g", 3_000)])
def test_resident_sweep_is_one_launch_and_sweeps_again_exactly(gpu, monkeypatch, name, cols):
    monkeypatch.delenv("WHMEC_TILE_ARENA_BUDGET", raising=False)
    monkeypatch.delenv("WHMEC_FORCE_COLUMN_KERNEL", raising=False)
    prob = synth.config(name, cols)
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
    assert second.same_as(first), second.diff(first)
    monkeypatch.setenv("WHMEC_FORCE_COLUMN_KERNEL", "1")
    col, st2 = gpu.solve(prob)
    assert st2["path_kind"] == 2
    assert col.same_as(first), col.diff(first)
