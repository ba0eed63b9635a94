"""SURVEY.md 8(f) rank 1 on the GPU: REAL `whatshap.core.ReadSet` / `Pedigree` objects (the compiled reference binding,
built by oracle/build_pyref.py into oracle/_ref/pyref where the reference sources are available) go through
`adapters.make_dp_table_class` into the CUDA solve, and everything the swap-in returns is compared with what the real
`whatshap.core.PedigreeDPTable` returns on the same objects — the call `whatshap phase` makes at whatshap/cli/phase.py:604-612.
The real class's answers are stored in tests/golden/real_containers_answers.json; without the binding the same inputs are
built from this package's containers and the swap-in's answers are compared with the stored ones."""
import json
import random

import pytest

import golden_io
import test_pedigreephasing as tp
import test_phasing as ts
from whatshap_b200 import adapters, components
from whatshap_b200 import core as mine
from whatshap_b200.testhelpers import string_to_readset, string_to_readset_pedigree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def real_core():
    """The reference binding, or None where it was not built."""
    from oracle import build_pyref

    return build_pyref.shipped_core()


def to_real(core, rs):
    out = core.ReadSet()
    for r in rs:
        read = core.Read(r.name, r.mapqs[0], r.source_id, r.sample_id)
        for v in r:
            read.add_variant(v.position, v.allele, v.quality)
        out.add(read)
    return out


def real_pedigree(core, case, recording=True):
    cls = adapters.recording_pedigree(core.Pedigree) if recording else core.Pedigree
    ped = cls(core.NumericSampleIds())
    for i, gts in enumerate(case["genotypes"]):
        genotypes = [core.Genotype([0] * (2 - g) + [1] * g) if 0 <= g <= 2 else core.Genotype([]) for g in gts]
        gls = [core.PhredGenotypeLikelihoods(g) for g in case["gls"][i]] if "gls" in case else None
        ped.add_individual("individual{}".format(i), genotypes, gls)
    for f, m, c in case["trios"]:
        ped.add_relationship("individual{}".format(f), "individual{}".format(m), "individual{}".format(c))
    return ped


def same_answers(a, b):
    assert a.get_optimal_cost() == b.get_optimal_cost()
    assert a.get_optimal_partitioning() == b.get_optimal_partitioning()
    (sa, ta), (sb, tb) = a.get_super_reads(), b.get_super_reads()
    assert ta == tb and len(sa) == len(sb)
    for ra, rb in zip(sa, sb):
        assert type(ra) is type(rb) and len(ra) == len(rb) == 2
        for x, y in zip(ra, rb):
            assert (x.name, x.mapqs, x.source_id, x.sample_id) == (y.name, y.mapqs, y.source_id, y.sample_id)
            assert [(v.position, v.allele, v.quality) for v in x] == [(v.position, v.allele, v.quality) for v in y]
    return sa


def answers(table):
    """Everything a table answers, as JSON-like data."""
    superreads, tv = table.get_super_reads()
    return {"cost": table.get_optimal_cost(), "partitioning": list(table.get_optimal_partitioning()), "tv": list(tv),
            "superreads": [[[x.name, list(x.mapqs), x.source_id, x.sample_id, [[v.position, v.allele, v.quality] for v in x]]
                            for x in rs] for rs in superreads]}


def check_against_reference(key, a, b):
    """`a` (the swap-in) answers like `b` (the real class, None without the binding) and like its stored answers."""
    if b is not None:
        same_answers(a, b)
    want = golden_io.reference_answer("real_containers", key, None if b is None else answers(b))
    assert json.loads(json.dumps(answers(a))) == want, key


@pytest.mark.parametrize("recording", [True, False])
@pytest.mark.parametrize("name", sorted(tp.CASES))
def test_pedigree_cases_real_objects_cuda_vs_real_dp_table(gpu, real_core, name, recording):
    case = tp.CASES[name]
    core = real_core or mine
    my_rs = string_to_readset_pedigree(case["reads"]) if case["reads"].strip() else mine.ReadSet()
    real_rs = to_real(core, my_rs)
    ped = real_pedigree(core, case, recording)
    distrust, positions = case.get("distrust", False), case.get("positions")
    Table = adapters.make_dp_table_class(core)  # default solver: the CUDA path
    a = Table(real_rs, case["recomb"], ped, distrust, positions)
    recomb = list(case["recomb"]) + [case["recomb"][-1]] * 4  # the real class reads recombcost[k] unchecked
    b = real_core.PedigreeDPTable(real_rs, recomb, ped, distrust, positions) if real_core else None
    assert a.get_optimal_cost() == case["cost"]
    check_against_reference(f"pedigree/{name}/{recording}", a, b)


def test_single_individual_matrices_real_objects(gpu, real_core):
    core = real_core or mine
    Table = adapters.make_dp_table_class(core)
    for name in sorted(ts.MATRICES):
        reads, weights = ts.MATRICES[name]
        real_rs = to_real(core, string_to_readset(reads, weights))
        positions = real_rs.get_positions()
        for het in (True, False):
            ped = core.Pedigree(core.NumericSampleIds())
            gls = [None if het else core.PhredGenotypeLikelihoods([0, 0, 0])] * len(positions)
            ped.add_individual("individual0", [core.Genotype([0, 1])] * len(positions), gls)
            b = real_core.PedigreeDPTable(real_rs, [1] * len(positions), ped, not het) if real_core else None
            check_against_reference(f"matrix/{name}/{het}", Table(real_rs, [1] * len(positions), ped, not het), b)


def random_real_readset(core, rng, n_cols, coverage, samples):
    """Reads with random spans and gaps over positions 100, 200, ...; sorted the way `whatshap phase` sorts them."""
    rs = core.ReadSet()
    idx = 0
    for start in range(-6, n_cols):
        for _ in range(coverage if rng.random() < 0.7 else 1):
            if rng.random() < 0.45:
                continue
            first, length = max(start, 0), rng.randint(2, 9)
            cols = [c for c in range(first, min(first + length, n_cols)) if c == first or rng.random() > 0.15]
            if len(cols) < 2:
                continue
            read = core.Read("read%05d" % idx, 60, 0, rng.randrange(samples))
            for c in cols:
                read.add_variant(100 * (c + 1), rng.randint(0, 1), rng.randint(1, 35))
            rs.add(read)
            idx += 1
    rs.sort()
    return rs


@pytest.mark.parametrize("seed", range(4))
def test_random_real_readsets_single_and_trio(gpu, real_core, seed):
    rng = random.Random(seed)
    core = real_core or mine
    Table = adapters.make_dp_table_class(core)
    for samples in (1, 3):
        n_cols = rng.randint(30, 70)
        rs = random_real_readset(core, rng, n_cols, 3 if samples == 1 else 2, samples)
        positions = rs.get_positions()
        n = len(positions)
        ped = adapters.recording_pedigree(core.Pedigree)(core.NumericSampleIds())
        distrust = bool(seed & 1)
        for s in range(samples):
            gls = [core.PhredGenotypeLikelihoods([rng.randint(0, 30) for _ in range(3)]) for _ in range(n)] if distrust else None
            ped.add_individual(s, [core.Genotype([0, 1])] * n, gls)
        if samples == 3:
            ped.add_relationship(0, 1, 2)
        recomb = [rng.randint(1, 30) for _ in range(n)] + [1] * 4
        a = Table(rs, recomb, ped, distrust, positions)
        b = real_core.PedigreeDPTable(rs, recomb, ped, distrust, positions) if real_core else None
        check_against_reference(f"random/{seed}/{samples}", a, b)
        superreads = a.get_super_reads()[0]
        # the step after the DP (whatshap/cli/phase.py:676-714) on the swap-in's super-reads
        family = list(range(samples))
        ids = {s: s for s in family}
        comp = components.compute_overall_components(positions, rs, distrust, family, samples > 1, [], ids, superreads)
        assert set(comp) == set(positions) and all(comp[p] <= p for p in positions)
