"""`whmec_realign_kmerald` and `whmec_kmer_align_batch` on the GPU (DESIGN §4.12): every golden case equals the reference's stored
answers; a large synthetic batch with long insertions equals the host emulation, with jobs on both kernels and in several
chunks; many random pairs equal the emulation and, where oracle/_ref/pyref ships it, the reference's compiled kmer_align."""
import random

import numpy as np
import pytest

from scripts.kmerald_batch import costs_table, workload
from test_kmerald import GOLDEN, Aln, Biallelic, check_case, cost_dict, emul, same_f32
from test_realign import reference_align
from whatshap_b200 import realign

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_budget(monkeypatch):
    monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET", raising=False)


@pytest.mark.parametrize("index", range(len(GOLDEN["detect"])))
def test_golden_case(gpu, index):
    check_case(GOLDEN["detect"][index], realign.detect_alleles)


@pytest.mark.parametrize("table", range(len(GOLDEN["pairs"])))
def test_golden_pairs(gpu, table):
    t = GOLDEN["pairs"][table]
    s1, s2 = zip(*t["seqs"])
    got = realign.kmer_distances(s1, s2, cost_dict(t["costs"]), t["gap"], t["k"])
    assert same_f32(got, [np.float32(float(w)) for w in t["want"]])


@pytest.fixture(scope="module")
def batch():
    reference, variants, alns = workload(0.3, seed=5)
    long_ins = Biallelic(1000, reference[1000], reference[1000] + "ACGT" * 300)  # a 1200-base insertion read through
    variants = sorted(variants + [long_ins], key=lambda v: v.position)
    alns.append(Aln(900, [(0, 101), (1, 1200), (0, 300)], reference[900:1001] + "ACGT" * 300 + reference[1001:1301]))
    costs = realign.KmerCosts(costs_table(7, 16))
    return reference, variants, alns, costs


def test_large_batch_equals_emulation(gpu, batch):
    reference, variants, alns, costs = batch
    kw = dict(use_kmerald=True, kmerald_costs=costs, kmerald_window=40, kmerald_gappenalty=12.5)
    st, st_e = {}, {}
    got = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
    want = realign.detect_alleles(alns, variants, reference, stats=st_e, library=emul(), **kw)
    assert got == want
    assert st["items"] >= 50000 and st["short_jobs"] > 0 and st["long_jobs"] > 0 and st["long_items"] > 0
    assert sum(len(g) for g in got) > st["items"] // 2


def test_chunked_equals_resident(gpu, batch, monkeypatch):
    reference, variants, alns, costs = batch
    alns = alns[:1500] + alns[-1:]
    kw = dict(use_kmerald=True, kmerald_costs=costs)
    st = {}
    whole = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
    assert st["chunks"] == 1 and st["long_jobs"] > 0
    for budget in (1, 200000 + len(costs) * 12):
        monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", str(budget))
        st_b = {}
        assert realign.detect_alleles(alns, variants, reference, stats=st_b, **kw) == whole
        assert st_b["chunks"] > 1 and (budget != 1 or st_b["chunks"] == st["items"])


def random_pairs(rng, n, long_share=0.01):
    s1, s2 = [], []
    for _ in range(n):
        a = "".join(rng.choice("ACGTACGTACGTN") for _ in range(rng.randrange(0, 70)))
        b = list(a)
        for _ in range(rng.randrange(0, 5)):
            if b:
                k = rng.randrange(len(b))
                b[k:k + rng.randrange(0, 3)] = rng.choice(["", "A", "C", "GT"])
        b = "".join(b)
        if rng.random() < long_share:
            a = a + "".join(rng.choice("ACGT") for _ in range(rng.randrange(65, 1200)))
        if rng.random() < 0.5:
            a, b = b, a
        s1.append(a)
        s2.append(b)
    return s1, s2


def test_distances_equal_emulation_and_reference(gpu):
    rng = random.Random(12)
    s1, s2 = random_pairs(rng, 30000)
    mapping = costs_table(5, 8)
    mapping[(27, -5)] = "nan"
    costs = realign.KmerCosts(mapping)
    st = {}
    got = realign.kmer_distances(s1, s2, costs, 7.3, 5, stats=st)
    assert st["long_jobs"] > 0 and st["short_jobs"] > 0
    assert same_f32(got, realign.kmer_distances(s1, s2, costs, 7.3, 5, library=emul()))
    align = reference_align()
    if align is not None:
        k = 20000
        want = [align.kmer_align(align.enumerate_all_kmers(a.encode(), 5), align.enumerate_all_kmers(b.encode(), 5), mapping, 7.3)
                for a, b in zip(s1[:k], s2[:k])]
        assert same_f32(got[:k], np.array(want, np.float32))
