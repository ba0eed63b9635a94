"""`whmec_realign` and `whmec_edit_distance_batch` on the GPU (DESIGN §4.11): every golden case equals the reference's stored
answers; a large random batch equals the host emulation (and the reference's compiled whatshap.align where shipped) in both
modes, with jobs on both kernels; chunked runs equal resident ones; errors name the alignment."""
import random

import numpy as np
import pytest

from scripts.realign_batch import synthetic
from test_realign import Aln, Var, check_case, emul, golden_cases, random_pairs, reference_align
from whatshap_b200 import realign

pytestmark = pytest.mark.gpu

AFFINE = dict(affine=True, gap_start=10, gap_extend=7, default_mismatch=15)


@pytest.fixture(autouse=True)
def no_budget(monkeypatch):
    monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET", raising=False)


@pytest.mark.parametrize("index", range(len(golden_cases())))
def test_golden_case(gpu, index):
    check_case(golden_cases()[index], realign.detect_alleles)


@pytest.fixture(scope="module")
def batch():
    reference, variants, alns = synthetic(1.2, seed=5)
    long_ins = Var(1000, reference[1000], [reference[1000] + "ACGT" * 300])  # a 1200-base insertion read through
    variants = sorted(variants + [long_ins], key=lambda v: v.position)
    alns.append(Aln(900, [(0, 101), (1, 1200), (0, 300)], reference[900:1001] + "ACGT" * 300 + reference[1001:1301]))
    return reference, variants, alns


@pytest.mark.parametrize("mode", ["unit", "affine"])
def test_large_batch_equals_emulation(gpu, batch, mode):
    reference, variants, alns = batch
    kw = AFFINE if mode == "affine" else {}
    st, st_e = {}, {}
    got = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
    want = realign.detect_alleles(alns, variants, reference, stats=st_e, library=emul(), **kw)
    assert got == want
    assert st["items"] > 200000 and st["short_jobs"] > 0 and st["long_jobs"] > 0 and st["long_items"] > 0


def test_chunked_equals_resident(gpu, batch, monkeypatch):
    reference, variants, alns = batch
    alns = alns[:3000] + alns[-1:]
    for kw in ({}, AFFINE):
        st = {}
        whole = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
        assert st["chunks"] == 1
        for budget in ("1", "100000"):
            monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", budget)
            st_b = {}
            assert realign.detect_alleles(alns, variants, reference, stats=st_b, **kw) == whole
            assert st_b["chunks"] > 1 and (budget != "1" or st_b["chunks"] == st["items"])
        monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET")


def test_distances_equal_reference_and_emulation(gpu):
    rng = random.Random(11)
    qs, ts = random_pairs(rng, 300000, long_share=0.01)
    st = {}
    unit = realign.edit_distances(qs, ts, stats=st)
    assert st["long_jobs"] > 0 and st["short_jobs"] > 0
    assert np.array_equal(unit, realign.edit_distances(qs, ts, library=emul()))
    aff = realign.edit_distances_affine_gap(qs, ts, 2.5, 10.9, 3.5)
    assert np.array_equal(aff, realign.edit_distances_affine_gap(qs, ts, 2.5, 10.9, 3.5, library=emul()))
    align = reference_align()
    if align is not None:
        k = 20000
        assert list(unit[:k]) == [align.edit_distance(q, t) for q, t in zip(qs[:k], ts[:k])]
        assert list(aff[:k]) == [align.edit_distance_affine_gap(q, t, [2.5] * len(q), 10, 3) for q, t in zip(qs[:k], ts[:k])]


def test_errors_name_the_alignment(gpu):
    reference = "ACGT" * 50
    variants = [Var(50, "G", ["C"]), Var(100, "A", ["T"])]
    good = Aln(40, [(0, 30)], reference[40:70])
    with pytest.raises(ValueError, match=r"^alignment 1\b.*Unsupported CIGAR operation"):
        realign.detect_alleles([good, Aln(40, [(0, 5), (9, 2), (0, 30)], reference[40:77])], variants, reference)
    with pytest.raises(ValueError, match=r"^alignment 1, variant 0: unknown CIGAR operator 9"):  # inside the window
        realign.detect_alleles([good, Aln(40, [(0, 20), (9, 2), (0, 10)], reference[40:72])], variants, reference)
    with pytest.raises(ValueError, match=r"^alignment 2, variant 0\b"):
        realign.detect_alleles([good, good, Aln(50, [(0, 30)], reference[50:80])], variants, reference, overhang=0)
