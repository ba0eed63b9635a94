"""Memory-bounded forward-backward genotyping on the GPU (DESIGN §4.5).  WHMEC_GENOTYPE_ARENA_BUDGET (bytes for backward tables,
checkpoints and projection buffers) forces the mode on problems that fit.  The likelihoods must equal the resident ones and the
reference to 1e-9 (the double atomicAdd makes even two resident runs differ in the last bits), with less memory for backward
tables and more launches; what no segment fits is refused with the bytes it needs; without the hook nothing changes."""
import re

import numpy as np
import pytest

import emul_genotype
import emul_genotype_bounded
from oracle import checker
from test_genotype import golden
from test_genotype_bounded import PEDS, instance, least_budget, tables
from whatshap_b200 import _lib, synth
from whatshap_b200._abi import Unsupported

pytestmark = pytest.mark.gpu

HOOK = "WHMEC_GENOTYPE_ARENA_BUDGET"
TOL = 1e-9


@pytest.fixture
def hook(monkeypatch):
    """Sets the budget (doubles -> bytes; None clears it), starting from a cleared hook."""
    monkeypatch.delenv(HOOK, raising=False)

    def set_budget(doubles):
        if doubles is None:
            monkeypatch.delenv(HOOK, raising=False)
        else:
            monkeypatch.setenv(HOOK, str(int(doubles) * 8))
    return set_budget


def close(a, b):
    return a.shape == b.shape and bool(np.all((np.abs(a - b) <= TOL) | (np.isnan(a) & np.isnan(b))))


def launches_of(plan, n_cols):
    """Two launches per step: the backward steps of the whole table, those of every segment but the first again, the forward steps."""
    cuts = plan["cuts"]
    resweep = sum(int(cuts[s + 1] - cuts[s]) - 1 for s in range(1, len(cuts) - 1))
    return 2 * ((n_cols - 1) + resweep + n_cols)


@pytest.mark.parametrize("ped", PEDS)
def test_bounded_equals_resident(hook, ped):
    prob, resident, second = instance(ped, PEDS.index(ped))
    whole, st = _lib.genotype(prob)
    want = checker.best().genotype(prob)
    assert close(whole, want)
    least = least_budget(prob)
    for budget in sorted({max(least, second, int(resident / d)) for d in (1.5, 3, 8)} | {max(least, second)}):
        hook(budget)
        got, st2 = _lib.genotype(prob)
        assert close(got, whole) and close(got, want), (ped, budget, float(np.nanmax(np.abs(got - whole))))
        assert st2["backptr_bytes"] < st["backptr_bytes"], (ped, budget, st2, st)
        assert st2["kernel_launches"] > st["kernel_launches"], (ped, budget, st2, st)
        assert st2["path_kind"] == 4
        if ped != "single":  # one table: the launches are those of its plan
            assert st2["kernel_launches"] == launches_of(emul_genotype_bounded.bounded_plan(prob, budget), prob.n_cols), (ped, budget, st2)


def test_golden_vectors_segmented(hook):
    """The reference's answers, with every table that has more than one column's backward table cut into segments."""
    cut = 0
    for label, prob, want, _ in golden():
        own = emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"]
        resident = max((c for _, _, c in tables(own)), default=0)
        if resident == 0 or np.count_nonzero(own) < 2:
            continue
        budget = max(least_budget(prob), resident // 2)
        if budget >= resident:
            continue
        hook(budget)
        got, st = _lib.genotype(prob)
        assert close(got, want), (label, float(np.nanmax(np.abs(got - want))))
        cut += 1
    assert cut >= 20, cut


def test_wide_columns(hook):
    """A trio at 15 active reads per column (32 768 cells), a few hundred columns, a quarter of the resident memory."""
    rng = np.random.default_rng(21)
    prob = synth.trio(300, 5, block_len=300, seed=21)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    whole, st = _lib.genotype(prob)
    hook(st["backptr_bytes"] // 32)  # (bytes / 4, in doubles)
    got, st2 = _lib.genotype(prob)
    assert np.allclose(got.sum(axis=2), 1.0, atol=1e-9)
    assert close(got, whole), float(np.max(np.abs(got - whole)))
    assert st2["backptr_bytes"] < st["backptr_bytes"] and st2["kernel_launches"] > st["kernel_launches"]


def test_object_level(hook):
    from whatshap_b200 import GenotypeDPTable, NumericSampleIds, Pedigree, PhredGenotypeLikelihoods
    from whatshap_b200.core import Genotype

    rng = np.random.default_rng(3)
    prob = synth.trio(60, 2, block_len=30, seed=3)  # (reads on every column)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    rs, recomb, _ = synth.to_objects(prob)
    resident = max(c for _, _, c in tables(emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"]))
    ids = NumericSampleIds()
    ped = Pedigree(ids)
    for i in range(prob.n_ind):
        ids[i]
        ped.add_individual(i, [Genotype([0, 1])] * prob.n_cols, [PhredGenotypeLikelihoods(list(prob.gl[i, k])) for k in range(prob.n_cols)])
    tr = prob.trios.tolist()
    ped.add_relationship(tr[0], tr[1], tr[2])

    def likelihoods():
        t = GenotypeDPTable(ids, rs, recomb, ped)
        return np.array([[t.get_genotype_likelihoods(i, k).as_vector() for k in range(prob.n_cols)] for i in range(prob.n_ind)])

    whole = likelihoods()
    hook(max(least_budget(prob), resident // 2))
    assert close(likelihoods(), whole)


def test_default_path_unchanged(hook):
    """Without the hook: one launch schedule, 2 x (backward + forward steps) launches, all backward tables resident."""
    prob, _, _ = instance("trio", 17)
    own = emul_genotype_bounded.bounded_plan(prob, 1 << 60)["own"]
    got, st = _lib.genotype(prob)
    assert st["kernel_launches"] == 2 * ((prob.n_cols - 1) + prob.n_cols), st
    assert st["backptr_bytes"] == int(own.sum()) * 8 and st["path_kind"] == 4, st
    assert close(got, emul_genotype.genotype(prob)[0])


def test_impossible_budget_is_refused(hook):
    prob, _, _ = instance("three_children", 5)
    hook(16)
    with pytest.raises(Unsupported, match=r"needs at least \d+ bytes") as e:
        _lib.genotype(prob)
    need = int(re.search(r"needs at least (\d+) bytes", str(e.value)).group(1))
    hook(need // 8)
    got, st = _lib.genotype(prob)
    assert close(got, emul_genotype.genotype(prob)[0]) and st["backptr_bytes"] < need
