"""Five-trio pedigrees (T = 1024) on the GPU: the wide column sweep against the reference-generated golden vectors (every field,
through the C ABI), PedigreeDPTable on the same path, resident and memory-bounded sweeps, and the refusals that remain."""
import sys

import numpy as np
import pytest

import golden_io
from whatshap_b200._abi import Unsupported

sys.path.insert(0, golden_io.HERE)
import make_five_trios_golden as five  # noqa: E402

pytestmark = pytest.mark.gpu


def test_wide_sweep_reproduces_golden_vectors(gpu):
    n = 0
    for label, prob, want, error in golden_io.load("five_trios"):
        got, stats = gpu.solve(prob)
        assert got.same_as(want), (label, got.diff(want))
        assert stats["path_kind"] == 5 and stats["transmissions"] == 1024, (label, stats)
        n += 1
    assert n >= 8


def test_pedigree_dp_table_takes_the_wide_sweep(gpu):
    from whatshap_b200 import PedigreeDPTable, synth
    from whatshap_b200.core import _flatten

    n = 0
    for label, prob, want, error in golden_io.load("five_trios"):
        if prob.distrust:
            continue  # (synth.to_objects builds trusted genotypes only)
        rs, recomb, ped = synth.to_objects(prob)
        table = PedigreeDPTable(rs, recomb, ped)
        flat, stats = gpu.solve(_flatten(rs, recomb, ped, False, None))
        assert stats["path_kind"] == 5, label
        assert table.get_optimal_cost() == flat.cost, label
        assert list(table.get_optimal_partitioning()) == flat.partition.tolist(), label
        n += 1
    assert n >= 4


def _bigger(seed=21):
    return five.five_trio_problem(seed, "three_gen", 80, max_cov=7, rc_max=3)


def test_bounded_equals_resident(gpu, monkeypatch):
    prob = _bigger()
    want, st = gpu.solve(prob)
    assert st["path_kind"] == 5
    bp = st["backptr_bytes"]
    monkeypatch.setenv("WHMEC_COLUMN_ARENA_BUDGET", "64")
    with pytest.raises(Unsupported, match="needs at least") as e:
        gpu.solve(prob)
    least = int(str(e.value).split("needs at least ")[1].split()[0])
    for budget in (bp // 2, bp // 4, max(bp // 16, least), least):
        monkeypatch.setenv("WHMEC_COLUMN_ARENA_BUDGET", str(budget))
        got, stb = gpu.solve(prob)
        assert got.same_as(want), (budget, got.diff(want))
        assert stb["path_kind"] == 5 and stb["backptr_bytes"] <= max(budget, least), (budget, stb)
        assert stb["kernel_launches"] > st["kernel_launches"], budget  # the backtrace swept segments again


def test_plan_api_sweeps_repeatedly_identically(gpu):
    prob = _bigger(22)
    want, _ = gpu.solve(prob)
    with gpu.Plan(prob) as plan:
        for _ in range(3):  # from the second sweep on, a captured graph is replayed
            plan.sweep()
            got = plan.finish()
            assert got.same_as(want), got.diff(want)
            assert plan.stats()["path_kind"] == 5


def test_segments_and_genotyping_are_refused(gpu):
    prob = five.five_trio_problem(23, "nuclear5", 12, max_cov=4, distrust=True)
    with pytest.raises(Unsupported, match="at most 4 trio relationships"):
        gpu.Segment(prob, continues=False)
    prob.gl = np.full(prob.gl.shape, 1.0 / 3.0)
    with pytest.raises(Unsupported, match="at most 4 trio relationships"):
        gpu.genotype(prob)
